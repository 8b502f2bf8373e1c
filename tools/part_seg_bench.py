#!/usr/bin/env python
"""One training step (forward, part_seg_loss, backward; no optimiser step) of the part segmentation nets on one GPU, for
three ways of feeding a batch of variable-size shapes.

Arms, timed alternately in one process with the method of tools/ragged_bench.py (L2 flushed before every launch, the
median of LAUNCHES launches per round, the median and [min, max] over ROUNDS rounds):
  (a) dense:    full shapes of N points, no lengths;
  (b) ragged:   the same shapes cut to lengths drawn uniformly from [N/2, N], NaN in the padding rows, with lengths=;
  (c) resample: the shapes of (b) resampled to N points with replacement (what the reference's ShapeNet loader does),
                labels alike, through the dense call.
Rows: PointNet2PartSeg and PointNet2PartSegMSG at B 16 and B 32, N 2048, on workloads.part_shapes.

    python tools/part_seg_bench.py [--rounds 5] [--launches 20] [--json OUT] [--only NAMES] [--profile]

--profile adds, per row and arm, a torch.profiler record of a few steps (after the timed rounds): the summed GPU kernel
time per step, the wall time per step with a device synchronise, and the kernels whose time differs most between the
dense and the ragged arm (with lengths, the batch norms of fp3 and fc1 are masked torch code).
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from pointnet2_b200 import nets, workloads as W  # noqa: E402
from ragged_bench import L2_FLUSH_BYTES, gpu_info, launch_ms, profile_arms  # noqa: E402

N = 2048
ROWS = [
    # name, net class, batch
    ("part_seg_b16", "PointNet2PartSeg", 16),
    ("part_seg_b32", "PointNet2PartSeg", 32),
    ("part_seg_msg_b16", "PointNet2PartSegMSG", 16),
    ("part_seg_msg_b32", "PointNet2PartSegMSG", 32),
]


def inputs(b, n, seed, dev):
    """dense, ragged and resampled (points, part labels), the categories, the device lengths and the host lengths"""
    rs = np.random.RandomState(seed)
    pts, cls, label = W.part_shapes(b, n, seed, nets.PART_OFFSETS)
    lengths = rs.randint(n // 2, n + 1, size=b)
    ragged = pts.copy()
    res_pts, res_label = np.empty_like(pts), np.empty_like(label)
    for i, l in enumerate(lengths):
        ragged[i, l:] = np.nan
        pick = rs.choice(l, n, replace=True)
        res_pts[i], res_label[i] = pts[i, pick], label[i, pick]
    t = lambda a: torch.from_numpy(a).to(dev)
    return ({"dense": (t(pts), t(label)), "ragged": (t(ragged), t(label)), "resample": (t(res_pts), t(res_label))},
            t(cls), t(lengths.astype(np.int32)), lengths)


def train_arms(net_name, b, dev):
    torch.manual_seed(0)
    net = getattr(nets, net_name)().to(dev).train()
    data, cls, lens, host_lengths = inputs(b, N, 100 + b, dev)

    def step(x, label, lengths=None):
        net.zero_grad(set_to_none=True)
        if isinstance(net, nets.PointNet2PartSegMSG):
            pred, _ = net(x, cls, lengths=lengths)
        else:
            pred, _ = net(x, lengths=lengths)
        nets.part_seg_loss(pred, label, lengths=lengths).backward()
    arms = {"dense": lambda: step(*data["dense"]), "ragged": lambda: step(*data["ragged"], lens),
            "resample": lambda: step(*data["resample"])}
    return arms, host_lengths


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--launches", type=int, default=20)
    ap.add_argument("--json", default=None)
    ap.add_argument("--only", default=None, help="comma-separated row names to run (default: all)")
    ap.add_argument("--profile", action="store_true", help="add a torch.profiler breakdown per row and arm")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("part_seg_bench.py needs a CUDA device")
    dev = torch.device("cuda:0")
    flush = torch.empty(L2_FLUSH_BYTES, dtype=torch.uint8, device=dev)
    out = {"gpu": gpu_info(), "rounds": args.rounds, "launches": args.launches, "unit": "ms per training step",
           "n": N, "rows": []}
    print("# gpu (name, power limit, max SM clock):", out["gpu"], flush=True)
    for name, net_name, b in ROWS:
        if args.only and name not in args.only.split(","):
            continue
        arms, host_lengths = train_arms(net_name, b, dev)
        for f in arms.values():  # warm-up: module load, cuBLAS heuristics, the allocator
            f(), f(), f()
        times = {k: [] for k in arms}
        for _ in range(args.rounds):
            for k, f in arms.items():
                times[k].append(launch_ms(f, flush, args.launches))
        row = {"row": name, "net": net_name, "b": b, "n": N, "mean_length": float(np.mean(host_lengths)),
               **{k: round(statistics.median(v), 3) for k, v in times.items()},
               "spread": {k: [round(min(v), 3), round(max(v), 3)] for k, v in times.items()}}
        if args.profile:
            prof = profile_arms(arms)
            d, r = prof["dense"]["per"], prof["ragged"]["per"]
            diff = sorted(set(d) | set(r), key=lambda k: -abs(r[k] - d[k]))[:12]
            row["profile"] = {k: {x: v[x] for x in ("kernel_ms", "wall_ms", "kernels")} for k, v in prof.items()}
            row["profile"]["ragged_minus_dense_ms"] = [[k[:90], round(r[k] - d[k], 4), round(d[k], 4)] for k in diff]
        out["rows"].append(row)
        print(json.dumps(row), flush=True)
    if args.json:
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
