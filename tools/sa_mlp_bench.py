#!/usr/bin/env python
"""The inference tail of every set-abstraction level of the networks, two ways, and whole eval forwards.

Arms, timed alternately in one process with the method of tools/ragged_bench.py (L2 flushed before every launch, the
median of LAUNCHES launches per round, the median and [min, max] over ROUNDS rounds), on the same indices:
  (a) torch:  group_and_concat -> SharedMLP (cuBLAS Linear, eval BatchNorm1d, ReLU) -> max, what fused=False runs;
  (b) fused:  layers.sa_mlp_max (csrc/sa_mlp.cu).
float32 (TF32 off) and bfloat16 (arm (a) under autocast).  Levels: sem_seg at B 16 / N 8192, cls_ssg at B 32 / N 1024,
cls_msg at B 16 / N 1024, part_seg at B 32 / N 2048.  Per level the script computes, from the shapes alone, the FLOPs
(2 * rows * sum C_in * C_out) and the bytes the fused form needs (idx, the gathered rows, the weights once, the
output), the time each implies on the H100 SXM data sheet (67 TFLOP/s FP32, 989 dense BF16, 3.35 TB/s), which of the
two binds, and the share of that bound the kernel reaches.  Then eval forwards of the four networks under no_grad with
the set-abstraction tails routed as the modules route them (layers.sa_mlp_applies: the kernel up to
layers.SA_MLP_MAX_MACS multiply-adds per row; "modules_take" in each level's row) and all through the torch layers.

    python tools/sa_mlp_bench.py [--rounds 5] [--launches 10] [--json OUT]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from pointnet2_b200 import layers, nets, pointnet_util  # noqa: E402
from pointnet2_b200 import workloads as W  # noqa: E402
from pointnet2_b200.sa_layer import sample_group  # noqa: E402
from ragged_bench import L2_FLUSH_BYTES, gpu_info, launch_ms  # noqa: E402

# (name, B, N, S, radius, K, C, widths, xyz_first); S None: the one group of all N points
LEVELS = [
    ("sem_seg.sa1", 16, 8192, 1024, 0.1, 32, 0, [32, 32, 64], True),
    ("sem_seg.sa2", 16, 1024, 256, 0.2, 32, 64, [64, 64, 128], True),
    ("sem_seg.sa3", 16, 256, 64, 0.4, 32, 128, [128, 128, 256], True),
    ("sem_seg.sa4", 16, 64, 16, 0.8, 32, 256, [256, 256, 512], True),
    ("cls_ssg.sa1", 32, 1024, 512, 0.2, 32, 0, [64, 64, 128], True),
    ("cls_ssg.sa2", 32, 512, 128, 0.4, 64, 128, [128, 128, 256], True),
    ("cls_ssg.sa3", 32, 128, None, None, 128, 256, [256, 512, 1024], True),
    ("cls_msg.sa1a", 16, 1024, 512, 0.1, 16, 0, [32, 32, 64], False),
    ("cls_msg.sa1b", 16, 1024, 512, 0.2, 32, 0, [64, 64, 128], False),
    ("cls_msg.sa1c", 16, 1024, 512, 0.4, 128, 0, [64, 96, 128], False),
    ("cls_msg.sa2a", 16, 512, 128, 0.2, 32, 320, [64, 64, 128], False),
    ("cls_msg.sa2b", 16, 512, 128, 0.4, 64, 320, [128, 128, 256], False),
    ("cls_msg.sa2c", 16, 512, 128, 0.8, 128, 320, [128, 128, 256], False),
    ("cls_msg.sa3", 16, 128, None, None, 128, 640, [256, 512, 1024], True),
    ("part_seg.sa1", 32, 2048, 512, 0.2, 64, 3, [64, 64, 128], True),
    ("part_seg.sa2", 32, 512, 128, 0.4, 64, 128, [128, 128, 256], True),
    ("part_seg.sa3", 32, 128, None, None, 128, 256, [256, 512, 1024], True),
]
PEAK_FLOPS_PER_MS = {torch.float32: 67e9, torch.bfloat16: 989e9}
HBM_BYTES_PER_MS = 3.35e9


def level_counts(b, s, k, c, widths, dtype):
    """(flops, bytes) of the fused form, from the shapes"""
    cin, rows, e = c + 3, b * s * k, torch.tensor([], dtype=dtype).element_size()
    macs = sum(i * o for i, o in zip([cin] + widths[:-1], widths))
    params = 4 * (macs + sum(6 * w for w in widths))  # weights, bias and the four batch-norm vectors, float32, once
    return 2 * rows * macs, 4 * rows + rows * (12 + c * e) + params + b * s * widths[-1] * e


def level_arms(level, dtype, dev):
    name, b, n, s, radius, k, c, widths, xyz_first = level
    xyz = torch.from_numpy(W.cloud_uniform(b, n, 7)).to(dev)
    points = None if c == 0 else torch.from_numpy(W.features(b, n, c, 8)).to(dev).to(dtype)
    mlp = layers.SharedMLP(c + 3, widths).to(dev).eval()
    if s is None:
        new_xyz = idx = None
    else:
        _, new_xyz, idx, _, _ = sample_group(s, radius, k, xyz, want_grouped=False)

    def torch_arm():
        with torch.no_grad(), torch.autocast("cuda", dtype=dtype, enabled=dtype != torch.float32):
            if idx is None:
                rows = (xyz if points is None else torch.cat([xyz.to(points.dtype), points], dim=2)).unsqueeze(1)
            else:
                rows, _ = pointnet_util.group_and_concat(xyz, new_xyz, points, idx, xyz_first)
            return mlp(rows).max(dim=2).values

    def fused_arm():
        with torch.no_grad(), torch.autocast("cuda", dtype=dtype, enabled=dtype != torch.float32):
            return layers.sa_mlp_max(xyz, new_xyz, points, idx, mlp, xyz_first)

    a, f = torch_arm().float(), fused_arm().float()
    err = ((a - f).abs().max() / a.abs().max()).item()
    with torch.no_grad():
        routed = "fused" if layers.sa_mlp_applies(mlp, xyz, points) else "torch"  # the arm the modules take
    return {"torch": torch_arm, "fused": fused_arm}, err, routed


def net_arms(dev):
    cases = [("sem_seg", nets.PointNet2SemSeg(21), 16, 8192, 3), ("cls_ssg", nets.PointNet2ClsSSG(40), 32, 1024, 3),
             ("cls_msg", nets.PointNet2ClsMSG(40), 16, 1024, 3), ("part_seg", nets.PointNet2PartSeg(50), 32, 2048, 6)]
    applies = layers.sa_mlp_applies
    for name, net, b, n, ch in cases:
        net = net.to(dev).eval()
        x = torch.from_numpy(W.cloud_uniform(b, n, 3)).to(dev)
        if ch == 6:
            x = torch.cat([x, torch.nn.functional.normalize(x, dim=2)], dim=2)

        def run(kernel, net=net, x=x):
            layers.sa_mlp_applies = applies if kernel else (lambda *a, **k: False)
            try:
                with torch.no_grad():
                    net(x)
            finally:
                layers.sa_mlp_applies = applies

        yield name, b, n, {"torch": lambda run=run: run(False), "fused": lambda run=run: run(True)}


def timed(arms, flush, rounds, launches):
    for f in arms.values():
        f(), f(), f()
    times = {k: [] for k in arms}
    for _ in range(rounds):
        for k, f in arms.items():
            times[k].append(launch_ms(f, flush, launches))
    med = {k: round(statistics.median(v), 4) for k, v in times.items()}
    return med, {k: [round(min(v), 4), round(max(v), 4)] for k, v in times.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--launches", type=int, default=10)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("sa_mlp_bench.py needs a CUDA device")
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    dev = torch.device("cuda:0")
    flush = torch.empty(L2_FLUSH_BYTES, dtype=torch.uint8, device=dev)
    out = {"gpu": gpu_info(), "rounds": args.rounds, "launches": args.launches, "unit": "ms", "levels": [], "nets": []}
    print("# gpu (name, power limit, max SM clock):", out["gpu"], flush=True)
    for level in LEVELS:
        name, b, n, s, _, k, c, widths, _ = level
        for dtype in (torch.float32, torch.bfloat16):
            arms, err, routed = level_arms(level, dtype, dev)
            med, spread = timed(arms, flush, args.rounds, args.launches)
            flops, nbytes = level_counts(b, s or 1, k, c, widths, dtype)
            t_flop, t_byte = flops / PEAK_FLOPS_PER_MS[dtype], nbytes / HBM_BYTES_PER_MS
            bound = max(t_flop, t_byte)
            row = {"level": name, "b": b, "rows": b * (s or 1) * k, "dtype": str(dtype).replace("torch.", ""), **med,
                   "modules_take": routed, "spread": spread, "gflop": round(flops / 1e9, 3), "mbytes": round(nbytes / 1e6, 3),
                   "flop_bound": round(t_flop, 4), "byte_bound": round(t_byte, 4),
                   "binds": "flops" if t_flop >= t_byte else "bytes", "share_of_bound": round(bound / med["fused"], 3),
                   "fused_vs_torch_scaled_diff": float(f"{err:.3g}")}
            out["levels"].append(row)
            print(json.dumps(row), flush=True)
    for name, b, n, arms in net_arms(dev):
        med, spread = timed(arms, flush, args.rounds, args.launches)
        row = {"net": name, "b": b, "n": n, "dtype": "float32", **med, "spread": spread}
        out["nets"].append(row)
        print(json.dumps(row), flush=True)
    if args.json:
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
