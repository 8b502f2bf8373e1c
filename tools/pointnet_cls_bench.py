#!/usr/bin/env python
"""PointNet v1 (nets.PointNetClsBasic) and the whole-cloud max-pool layers behind it, timed.

Arms are timed alternately in one process with the method of tools/ragged_bench.py (L2 flushed before every launch, the
median of LAUNCHES launches per round, the median and [min, max] over ROUNDS rounds), float32 with TF32 off:
  steps   a cls_basic training step (forward, cls_loss, backward) at B 32 / N 1024, dense and with ModelNet's point
          dropout (each cloud keeps N * (1 - U[0, 0.875]) rows, the padding NaN): the fused route (masked_bn_relu_max)
          against the torch composition (conv5 through SharedMLP's masked layers, padding to -inf, first-row max),
          which this script calls directly;
  eval    cls_basic eval forwards under no_grad, default mode / inside batch_invariant(), dense and dropout;
  levels  the group_all levels of cls_ssg, cls_msg and part_seg and PointNet's conv5 + max: the whole-cloud entry
          (pn2_sa_mlp_max_all_typed, split over CTAs) against the one-CTA walk (pn2_sa_mlp_max_typed, called through
          _lib) and the torch layers (cuBLAS Linear, eval BatchNorm1d, ReLU, max), on the same inputs; the split and
          one-CTA outputs are checked to be bit-identical.
The card's name, power limit and maximum SM clock are printed in the same run.

    python tools/pointnet_cls_bench.py [--rounds 5] [--launches 10] [--json OUT]
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from pointnet2_b200 import _lib, batch_invariant, layers, nets  # noqa: E402
from pointnet2_b200 import workloads as W  # noqa: E402
from pointnet2_b200._tensor import DTYPE_CODES, ptr, stream_ptr  # noqa: E402
from ragged_bench import L2_FLUSH_BYTES, gpu_info  # noqa: E402
from sa_mlp_bench import timed  # noqa: E402

B, N = 32, 1024
# (name, B, rows per cloud, feature channels, widths): the group_all levels (after a 128-centroid level) and conv5
LEVELS = [
    ("cls_ssg.sa3", 32, 128, 256, [256, 512, 1024]),
    ("cls_msg.sa3", 16, 128, 640, [256, 512, 1024]),
    ("part_seg.sa3", 32, 128, 256, [256, 512, 1024]),
    ("cls_basic.conv5", 32, 1024, 128, [1024]),
]


def dropout_lengths(b, n, seed):
    rs = np.random.RandomState(seed)
    return np.maximum(1, (n * (1.0 - rs.uniform(0, 0.875, b))).astype(np.int64))


def step_arms(dev):
    torch.manual_seed(0)
    net = nets.PointNetClsBasic(40).to(dev).train()
    label = torch.randint(0, 40, (B,), device=dev)
    arms = {}
    for layout in ("dense", "dropout"):
        pts = W.cloud_uniform(B, N, 3)
        lengths = None
        if layout == "dropout":
            lens = dropout_lengths(B, N, 4)
            for i, l in enumerate(lens):
                pts[i, l:] = np.nan
            lengths = torch.from_numpy(lens.astype(np.int32)).to(dev)
        x = torch.from_numpy(pts).to(dev)

        def fused(x=x, lengths=lengths):
            net.zero_grad(set_to_none=True)
            nets.cls_loss(net(x, lengths)[0], label).backward()

        def composition(x=x, lengths=lengths):
            net.zero_grad(set_to_none=True)
            mask = torch.ones(B, N, dtype=torch.bool, device=dev) if lengths is None else layers.row_mask(lengths, N)
            y = net.conv5(net.feat(x, mask), mask)
            g = layers._first_max(torch.where(mask.unsqueeze(-1), y, float("-inf")))
            nets.cls_loss(net.fc3(net.dp1(net.fc2(net.fc1(g)))), label).backward()

        arms[f"{layout}.fused"] = fused
        arms[f"{layout}.composition"] = composition
    return arms


def eval_arms(dev):
    torch.manual_seed(0)
    net = nets.PointNetClsBasic(40).to(dev).eval()
    arms = {}
    for layout in ("dense", "dropout"):
        pts = W.cloud_uniform(B, N, 5)
        lengths = None
        if layout == "dropout":
            lens = dropout_lengths(B, N, 6)
            for i, l in enumerate(lens):
                pts[i, l:] = np.nan
            lengths = torch.from_numpy(lens.astype(np.int32)).to(dev)
        x = torch.from_numpy(pts).to(dev)

        def default(x=x, lengths=lengths):
            with torch.no_grad():
                net(x, lengths)

        def invariant(x=x, lengths=lengths):
            with torch.no_grad(), batch_invariant():
                net(x, lengths)

        arms[f"{layout}.default"] = default
        arms[f"{layout}.batch_invariant"] = invariant
    return arms


def level_arms(level, dev):
    name, b, n, c, widths = level
    torch.manual_seed(1)
    mlp = layers.SharedMLP(c, widths).to(dev).eval()
    points = torch.randn(b, n, c, device=dev)
    out_one = torch.empty((b, 1, mlp.out_channels), device=dev)
    args = layers._layer_args(layers._mlp_stack(mlp))
    lib = _lib.load()

    def split():
        with torch.no_grad():
            return layers.sa_mlp_max(None, None, points, None, mlp, True, False)

    def one_cta():
        rc = lib.pn2_sa_mlp_max_typed(DTYPE_CODES[torch.float32], b, n, c, 1, n, ptr(points), ptr(None), ptr(points),
                                      ptr(None), 1, 0, *args, ptr(out_one), out_one.stride(1), stream_ptr(dev))
        _lib.check(rc, "pn2_sa_mlp_max_typed")
        return out_one

    def torch_layers():
        with torch.no_grad():
            return mlp(points).amax(1)

    same = bool(torch.equal(split().view(torch.int32), one_cta().view(torch.int32)))
    return {"split": split, "one_cta": one_cta, "torch": torch_layers}, same


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--launches", type=int, default=10)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("pointnet_cls_bench.py needs a CUDA device")
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    dev = torch.device("cuda:0")
    flush = torch.empty(L2_FLUSH_BYTES, dtype=torch.uint8, device=dev)
    out = {"gpu": gpu_info(), "sms": torch.cuda.get_device_properties(dev).multi_processor_count, "rounds": args.rounds,
           "launches": args.launches, "unit": "ms"}
    print("# gpu (name, power limit, max SM clock):", out["gpu"], flush=True)
    med, rng = timed(step_arms(dev), flush, args.rounds, args.launches)
    out["steps"] = {"B": B, "N": N, "median": med, "range": rng}
    print("train step", json.dumps(out["steps"]), flush=True)
    med, rng = timed(eval_arms(dev), flush, args.rounds, args.launches)
    out["eval"] = {"B": B, "N": N, "median": med, "range": rng}
    print("eval forward", json.dumps(out["eval"]), flush=True)
    out["levels"] = []
    for level in LEVELS:
        arms, same = level_arms(level, dev)
        med, rng = timed(arms, flush, args.rounds, args.launches)
        row = {"level": level[0], "B": level[1], "rows": level[2], "cin": level[3], "widths": level[4],
               "split_equals_one_cta": same, "median": med, "range": rng}
        out["levels"].append(row)
        print("level", json.dumps(row), flush=True)
    if args.json:
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
