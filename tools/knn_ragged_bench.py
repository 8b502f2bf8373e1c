#!/usr/bin/env python
"""Time the kNN set-abstraction layer on batches of variable-size clouds (B 32, capacity N 4096 -> 1024, k 32) three
ways, alternating in one process:

  ragged   sample_knn(..., lengths=L): one call on the padded batch, each cloud sampled and searched alone;
  padded   the same clouds padded to N rows by repeating their points (what a loader that must fill a dense batch
           does today) through sample_knn without lengths — note that this changes the answer (DESIGN.md §6.8);
  loop     sample_knn on each cloud alone (b = 1, n = its length), one call per cloud.

Both layer paths are forced in turn with pn2_set_sa_knn_path (1 = overlapped, 2 = sequential); the loop takes each
cloud's own choice.  knn_point(k, xyz, new_xyz, lengths=L) is also timed alone against the dense call on the padded
clouds.  Lengths are drawn from a seeded U[lo, hi] per batch, for the rows U[N/2, N] and U[N/4, N/2], on uniform and
duplicate-heavy clouds.  Times are CUDA events around `--iters` calls after a warm-up, median over `--rounds` rounds
(variants in alternating order).  The card's name and power limit are read in the same run.

    python tools/knn_ragged_bench.py --out DIR [--rounds 5] [--iters 20]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from pointnet2_b200 import _lib, workloads as W  # noqa: E402
from pointnet2_b200.sa_layer import sample_knn  # noqa: E402
from pointnet2_b200.tf_grouping import knn_point  # noqa: E402

B, N, M, K = 32, 4096, 1024, 32
ROWS = [("U[N/2, N]", N // 2, N), ("U[N/4, N/2]", N // 4, N // 2)]
CLOUDS = {"uniform": W.cloud_uniform, "duplicates": W.cloud_duplicates}


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = "nvidia-smi unavailable"
    return {"torch_name": name, "nvidia_smi": q}


def timed(fn, iters):
    fn()  # warm-up (and the first-call attribute setup)
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--iters", type=int, default=20)
    args = ap.parse_args()
    os.makedirs(args.out, exist_ok=True)
    dev = torch.device("cuda:0")
    lib = _lib.load()
    results = {"card": card(), "shape": dict(B=B, N=N, M=M, k=K), "rows": []}
    for cname, gen in CLOUDS.items():
        pool = gen(B, N, 11)
        for label, lo, hi in ROWS:
            lens = np.random.default_rng(lo).integers(lo, hi + 1, B)
            ragged = pool.copy()
            for i, ln in enumerate(lens):  # padding a kernel must never read
                ragged[i, ln:] = np.nan
            padded = pool.copy()
            for i, ln in enumerate(lens):
                padded[i, ln:] = pool[i, np.arange(ln, N) % ln]
            xr, xp = torch.from_numpy(ragged).to(dev), torch.from_numpy(padded).to(dev)
            clouds = [torch.from_numpy(np.ascontiguousarray(pool[i:i + 1, :ln])).to(dev) for i, ln in enumerate(lens)]
            lt = torch.from_numpy(lens.astype(np.int32)).to(dev)
            _, new_xyz, _, _, _ = sample_knn(M, K, xr, lengths=lt, want_grouped=False)
            variants = {}
            for path, pname in ((1, "overlapped"), (2, "sequential")):
                variants[f"ragged/{pname}"] = (path, lambda: sample_knn(M, K, xr, lengths=lt))
                variants[f"padded/{pname}"] = (path, lambda: sample_knn(M, K, xp))
            variants["loop/auto"] = (0, lambda: [sample_knn(M, K, c) for c in clouds])
            variants["knn_point/ragged"] = (0, lambda: knn_point(K, xr, new_xyz, lengths=lt))
            variants["knn_point/padded"] = (0, lambda: knn_point(K, xp, new_xyz))
            times = {v: [] for v in variants}
            names = list(variants)
            for r in range(args.rounds):
                for v in (names if r % 2 == 0 else names[::-1]):
                    path, fn = variants[v]
                    try:
                        lib.pn2_set_sa_knn_path(path)
                        times[v].append(timed(fn, args.iters))
                    finally:
                        lib.pn2_set_sa_knn_path(0)
            row = {"clouds": cname, "lengths": label, "mean_length": float(lens.mean()),
                   "ms": {v: round(statistics.median(t), 4) for v, t in times.items()},
                   "ms_min": {v: round(min(t), 4) for v, t in times.items()},
                   "ms_max": {v: round(max(t), 4) for v, t in times.items()}}
            results["rows"].append(row)
            print(json.dumps(row), flush=True)
    with open(os.path.join(args.out, "knn_ragged_bench.json"), "w") as f:
        json.dump(results, f, indent=1)
    print(json.dumps(results["card"]))


if __name__ == "__main__":
    main()
