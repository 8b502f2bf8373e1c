#!/usr/bin/env python
"""What a batch of variable-size clouds costs, on one GPU, against two ways of feeding it without lengths.

Arms, timed alternately in one process, the L2 flushed before every launch (as bench.py does):
  (a) dense:    today's call on full clouds of n points;
  (b) ragged:   the same call with `lengths` drawn uniformly from [n/2, n] and NaN in the padding rows;
  (c) resample: the clouds of (b) resampled to n points with replacement (what a loader does without lengths,
                e.g. a ScanNet crop), through the dense call.
Shapes: cfg2 (B 32, N 4096 -> 1024, S 32, r 0.1) and the first sem-seg level (B 16, N 8192 -> 1024) through the fused
sampling+grouping layer, cfg2 and a cluster plan (B 8, N 65 536 -> 16 384) through FPS + gather alone.  Each number is the
median over ROUNDS rounds of the median of LAUNCHES launches.

    python tools/ragged_bench.py [--rounds 5] [--launches 20] [--json OUT]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from pointnet2_b200 import workloads as W  # noqa: E402
from pointnet2_b200.sa_layer import sample_group  # noqa: E402
from pointnet2_b200.tf_sampling import farthest_point_sample_and_gather  # noqa: E402

L2_FLUSH_BYTES = 256 << 20  # > the 50 MB L2 of the H100
SHAPES = [
    # name, b, n, npoint, radius, nsample (radius None: FPS + gather only)
    ("cfg2", 32, 4096, 1024, 0.1, 32),
    ("cfg2_fps", 32, 4096, 1024, None, None),
    ("semseg_l1", 16, 8192, 1024, 0.1, 32),
    ("fps_cluster", 8, 65536, 16384, None, None),
]


def gpu_info() -> str:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name()


def inputs(b, n, seed, dev):
    rs = np.random.RandomState(seed)
    full = W.cloud_uniform(b, n, seed)
    lengths = rs.randint(n // 2, n + 1, size=b)
    ragged = full.copy()
    resampled = np.empty_like(full)
    for i, l in enumerate(lengths):
        ragged[i, l:] = np.nan
        resampled[i] = full[i, rs.choice(l, n, replace=True)]
    t = lambda a: torch.from_numpy(a).to(dev)
    return t(full), t(ragged), torch.from_numpy(lengths.astype(np.int32)).to(dev), t(resampled), lengths


def launch_ms(fn, flush, launches):
    st = torch.cuda.current_stream()
    ts = []
    for _ in range(launches):
        flush.zero_()
        a, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(st)
        fn()
        e.record(st)
        e.synchronize()
        ts.append(a.elapsed_time(e))
    return statistics.median(ts)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--launches", type=int, default=20)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("ragged_bench.py needs a CUDA device")
    dev = torch.device("cuda:0")
    flush = torch.empty(L2_FLUSH_BYTES, dtype=torch.uint8, device=dev)
    out = {"gpu": gpu_info(), "rounds": args.rounds, "launches": args.launches, "unit": "ms per call", "shapes": []}
    print("# gpu (name, power limit, max SM clock):", out["gpu"], flush=True)
    for name, b, n, m, r, s in SHAPES:
        full, ragged, lens, resampled, host_lengths = inputs(b, n, 100, dev)
        if r is None:
            call = lambda x, lengths=None: farthest_point_sample_and_gather(m, x, lengths=lengths)
        else:
            call = lambda x, lengths=None: sample_group(m, r, s, x, center=True, lengths=lengths)
        arms = {"dense": lambda: call(full), "ragged": lambda: call(ragged, lens), "resample": lambda: call(resampled)}
        for f in arms.values():  # warm-up: module load, function attributes
            f(), f()
        times = {k: [] for k in arms}
        for _ in range(args.rounds):
            for k, f in arms.items():
                times[k].append(launch_ms(f, flush, args.launches))
        row = {"shape": name, "b": b, "n": n, "npoint": m, "radius": r, "nsample": s,
               "mean_length": float(np.mean(host_lengths)),
               **{k: round(statistics.median(v), 4) for k, v in times.items()},
               "spread": {k: [round(min(v), 4), round(max(v), 4)] for k, v in times.items()}}
        out["shapes"].append(row)
        print(json.dumps(row), flush=True)
    if args.json:
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
