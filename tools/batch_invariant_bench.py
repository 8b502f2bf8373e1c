#!/usr/bin/env python
"""What layers.batch_invariant() costs: every feature-propagation level and head two ways, whole eval forwards of the
five networks with the mode off and on, and predict_scene on a room of about 10^6 points.

Levels (arms timed alternately in one process with the method of tools/ragged_bench.py: L2 flushed before every
launch, the median of LAUNCHES launches per round, the median and [min, max] over ROUNDS rounds), on the same inputs:
  (a) torch:   fp_interpolate_concat -> SharedMLP (cuBLAS Linear, eval BatchNorm1d, ReLU), or the SharedMLP alone for
               a head: what the modules run outside the mode;
  (b) kernel:  layers.fp_mlp / layers.mlp_rows (csrc/fp_mlp.cu): what they run inside it.
float32 (TF32 off) and bfloat16 (arm (a) under autocast).  Sizes as in the README: sem_seg B 16 / N 8192, part_seg and
part_seg_msg B 32 / N 2048, the classifier head at B 32.  Nets: eval forwards under no_grad, default / batch-invariant,
float32 and bf16 autocast (cls_msg at B 16 / N 1024, cls_ssg at B 32 / N 1024).  Scene: predict_scene at batch size 16,
default / batch-invariant, CUDA-event time of the whole call, median of ROUNDS.

    python tools/batch_invariant_bench.py [--rounds 5] [--launches 10] [--scene-points 1000000] [--json OUT]
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
from pointnet2_b200 import batch_invariant, layers, nets, scene  # noqa: E402
from pointnet2_b200 import workloads as W  # noqa: E402
from pointnet2_b200.tf_interpolate import fp_interpolate_concat  # noqa: E402
from ragged_bench import L2_FLUSH_BYTES, gpu_info  # noqa: E402
from sa_mlp_bench import timed  # noqa: E402

# (name, B, N1, N2, C1, C2, widths, bn, last_activation); N2 = 0: a head on (B, N1, C2) rows
LEVELS = [
    ("sem_seg.fp1", 16, 64, 16, 256, 512, [256, 256], True, True),
    ("sem_seg.fp2", 16, 256, 64, 128, 256, [256, 256], True, True),
    ("sem_seg.fp3", 16, 1024, 256, 64, 256, [256, 128], True, True),
    ("sem_seg.fp4", 16, 8192, 1024, 0, 128, [128, 128, 128], True, True),
    ("sem_seg.fc1", 16, 8192, 0, 0, 128, [128], True, True),
    ("sem_seg.fc2", 16, 8192, 0, 0, 128, [21], False, False),
    ("part_seg.fp1", 32, 128, 1, 256, 1024, [256, 256], True, True),
    ("part_seg.fp2", 32, 512, 128, 128, 256, [256, 128], True, True),
    ("part_seg.fp3", 32, 2048, 512, 6, 128, [128, 128, 128], True, True),
    ("part_seg.fc1", 32, 2048, 0, 0, 128, [128], True, True),
    ("part_seg.fc2", 32, 2048, 0, 0, 128, [50], False, False),
    ("part_seg_msg.fp1", 32, 128, 1, 512, 1024, [256, 256], True, True),
    ("part_seg_msg.fp2", 32, 512, 128, 320, 256, [256, 128], True, True),
    ("part_seg_msg.fp3", 32, 2048, 512, 22, 128, [128, 128], True, True),
    ("cls.fc1", 32, 1, 0, 0, 1024, [512], True, True),
    ("cls.fc2", 32, 1, 0, 0, 512, [256], True, True),
    ("cls.fc3", 32, 1, 0, 0, 256, [40], False, False),
]


def level_arms(level, dtype, dev):
    name, b, n1, n2, c1, c2, widths, bn, last = level
    xyz1 = torch.from_numpy(W.cloud_uniform(b, n1, 7)).to(dev)
    xyz2 = torch.from_numpy(W.cloud_uniform(b, max(n2, 1), 8)).to(dev)
    points2 = torch.from_numpy(W.features(b, n2 if n2 else n1, c2, 9)).to(dev).to(dtype)
    points1 = None if c1 == 0 else torch.from_numpy(W.features(b, n1, c1, 10)).to(dev).to(dtype)
    mlp = layers.SharedMLP(c2 + c1, widths, bn=bn, last_activation=last).to(dev).eval()
    amp = dict(device_type="cuda", dtype=dtype, enabled=dtype != torch.float32)

    def torch_arm():
        with torch.no_grad(), torch.autocast(**amp):
            return mlp(fp_interpolate_concat(xyz1, xyz2, points1, points2) if n2 else points2)

    def kernel_arm():
        with torch.no_grad(), torch.autocast(**amp):
            return layers.fp_mlp(xyz1, xyz2, points1, points2, mlp) if n2 else layers.mlp_rows(points2, mlp)

    a, k = torch_arm().float(), kernel_arm().float()
    return {"torch": torch_arm, "kernel": kernel_arm}, ((a - k).abs().max() / a.abs().max()).item()


def net_arms(dev):
    cases = [("sem_seg", nets.PointNet2SemSeg(21), 16, 8192, 3), ("cls_ssg", nets.PointNet2ClsSSG(40), 32, 1024, 3),
             ("cls_msg", nets.PointNet2ClsMSG(40), 16, 1024, 3), ("part_seg", nets.PointNet2PartSeg(50), 32, 2048, 6),
             ("part_seg_msg", nets.PointNet2PartSegMSG(50), 32, 2048, 6)]
    for name, net, b, n, ch in cases:
        net = net.to(dev).eval()
        x = torch.from_numpy(W.cloud_uniform(b, n, 3)).to(dev)
        if ch == 6:
            x = torch.cat([x, torch.nn.functional.normalize(x, dim=2)], dim=2)
        args = (x, torch.arange(b, device=dev) % 16) if name == "part_seg_msg" else (x,)
        for dtype in (torch.float32, torch.bfloat16):
            def run(mode, net=net, args=args, dtype=dtype):
                with torch.no_grad(), torch.autocast("cuda", dtype=dtype, enabled=dtype != torch.float32), \
                        batch_invariant(mode):
                    net(*args)

            yield name, b, n, dtype, {"default": lambda run=run: run(False), "invariant": lambda run=run: run(True)}


def scene_ms(net, xyz, mode, rounds):
    times = []
    for _ in range(rounds + 1):
        start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        start.record()
        with batch_invariant(mode):
            scene.predict_scene(net, xyz, batch_size=16)
        end.record()
        torch.cuda.synchronize()
        times.append(start.elapsed_time(end))
    return times[1:]  # the first call warms up


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--launches", type=int, default=10)
    ap.add_argument("--scene-points", type=int, default=1_000_000)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("batch_invariant_bench.py needs a CUDA device")
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    dev = torch.device("cuda:0")
    flush = torch.empty(L2_FLUSH_BYTES, dtype=torch.uint8, device=dev)
    out = {"gpu": gpu_info(), "rounds": args.rounds, "launches": args.launches, "unit": "ms", "levels": [], "nets": []}
    print("# gpu (name, power limit, max SM clock):", out["gpu"], flush=True)
    for level in LEVELS:
        name, b, n1 = level[:3]
        for dtype in (torch.float32, torch.bfloat16):
            arms, err = level_arms(level, dtype, dev)
            med, spread = timed(arms, flush, args.rounds, args.launches)
            macs = sum(i * o for i, o in zip([level[4] + level[5]] + level[6][:-1], level[6]))
            row = {"level": name, "rows": b * n1, "dtype": str(dtype).replace("torch.", ""), **med, "spread": spread,
                   "gflop": round(2 * b * n1 * macs / 1e9, 3), "kernel_vs_torch_scaled_diff": float(f"{err:.3g}")}
            out["levels"].append(row)
            print(json.dumps(row), flush=True)
    for name, b, n, dtype, arms in net_arms(dev):
        med, spread = timed(arms, flush, args.rounds, args.launches)
        row = {"net": name, "b": b, "n": n, "dtype": str(dtype).replace("torch.", ""), **med, "spread": spread}
        out["nets"].append(row)
        print(json.dumps(row), flush=True)
    torch.manual_seed(0)
    net = nets.PointNet2SemSeg(21).to(dev).eval()
    xyz = torch.from_numpy(W.scene_room(args.scene_points, 1)[0]).to(dev)
    blocks = scene.scene_blocks(xyz)
    t = {}
    for _ in range(2):  # alternate the arms
        for mode in (False, True):
            t.setdefault(mode, []).extend(scene_ms(net, xyz, mode, max(1, args.rounds // 2)))
    out["scene"] = {"points": int(xyz.shape[0]), "blocks": int(blocks.lengths.shape[0]), "batch_size": 16,
                    "default": round(statistics.median(t[False]), 2), "invariant": round(statistics.median(t[True]), 2),
                    "spread": {"default": [round(min(t[False]), 2), round(max(t[False]), 2)],
                               "invariant": [round(min(t[True]), 2), round(max(t[True]), 2)]}}
    print(json.dumps(out["scene"]), flush=True)
    if args.json:
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
