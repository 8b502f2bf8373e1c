#!/usr/bin/env python
"""Time a stream of variable-size batches through the host-buffer set-abstraction layer (the cfg2 layer: B 32,
capacity N 4096 -> 1024, r 0.1, S 32) two ways, alternating in one process:

  ragged   SetAbstractionPipeline(..., ragged=True): the clouds are packed into the pinned input, only their rows
           are copied in, and the layer runs at the stride of the batch's longest cloud;
  padded   each cloud padded on the host to N rows (its points repeated, as a loader that must fill a dense batch
           would) in the pinned input of today's SetAbstractionPipeline.

Each batch's lengths are drawn from a seeded U[lo, hi]; row "U[N/2, N]" is the mixed case and row "U[N/4, N/2]"
the one where every cloud is at most half the capacity.  A round times `--batches` batches through each variant
(order alternating by round), wall clock from the first submit to the last collect, packing and padding included;
the JSON has the median, minimum and maximum over the rounds.  The card's name and power limit are read in the same
run.

    python tools/ragged_host_bench.py --out DIR [--rounds 7] [--batches 100]
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from pointnet2_b200 import _lib, workloads as W  # noqa: E402
from pointnet2_b200.host import SetAbstractionPipeline  # noqa: E402

B, N, M, R, S, DEPTH = 32, 4096, 1024, 0.1, 32, 2
ROWS = [("U[N/2, N]", N // 2, N), ("U[N/4, N/2]", N // 4, N // 2)]


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = "nvidia-smi unavailable"
    return {"torch_name": name, "nvidia_smi": q}


def fps_plan(lib, b, n):
    t, p, c = ctypes.c_int(), ctypes.c_int(), ctypes.c_int()
    assert lib.pn2_fps_plan(b, n, ctypes.byref(t), ctypes.byref(p), ctypes.byref(c)) == 0
    return f"threads {t.value}, points/thread {p.value}, cluster {c.value}"


def stream(lo, hi, batches, seed):
    rng = np.random.default_rng(seed)
    pool = W.cloud_uniform(B, N, seed)
    out = []
    for _ in range(batches):
        lens = rng.integers(lo, hi + 1, B)
        out.append([np.ascontiguousarray(pool[i, :l]) for i, l in enumerate(lens)])
    return out


def run_ragged(pipe, batches):
    h2d = 0
    for clouds in batches:
        if pipe.full():
            pipe.collect()
        pipe.submit(clouds)
        h2d += pipe.h2d_bytes
    while pipe.pending():
        pipe.collect()
    return h2d


def run_padded(pipe, batches):
    h2d = 0
    for clouds in batches:
        if pipe.full():
            pipe.collect()
        buf = pipe.input_buffer()
        for i, c in enumerate(clouds):
            buf[i] = c[np.arange(N) % len(c)]
        pipe.submit()
        h2d += pipe.h2d_bytes
    while pipe.pending():
        pipe.collect()
    return h2d


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True, help="directory for ragged_host_bench.json")
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--batches", type=int, default=100)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("ragged_host_bench needs a CUDA device")
    dev = torch.device("cuda:0")
    lib = _lib.load()
    info = card()
    print(info, flush=True)
    pipes = {"ragged": SetAbstractionPipeline(B, N, M, R, S, depth=DEPTH, device=dev, ragged=True),
             "padded": SetAbstractionPipeline(B, N, M, R, S, depth=DEPTH, device=dev)}
    runners = {"ragged": run_ragged, "padded": run_padded}
    rows = []
    for label, lo, hi in ROWS:
        batches = stream(lo, hi, a.batches, 400 + lo)
        points = sum(len(c) for clouds in batches for c in clouds)
        strides = sorted({max(len(c) for c in clouds) for clouds in batches})
        for name in runners:  # warm-up: module loads, function attributes, pinned pages
            runners[name](pipes[name], batches[:4])
        torch.cuda.synchronize(dev)
        times = {name: [] for name in runners}
        h2d = {}
        names = list(runners)
        for r in range(a.rounds):
            for name in (names if r % 2 == 0 else names[::-1]):
                t0 = time.perf_counter()
                h2d[name] = runners[name](pipes[name], batches)
                torch.cuda.synchronize(dev)
                times[name].append((time.perf_counter() - t0) * 1e3 / a.batches)
        row = dict(lengths=label, b=B, capacity=N, npoint=M, radius=R, nsample=S, depth=DEPTH, batches=a.batches,
                   rounds=a.rounds, mean_length=round(points / (B * a.batches), 1),
                   stride_min=strides[0], stride_max=strides[-1])
        for name, ts in times.items():
            med = float(np.median(ts))
            row[name] = dict(median_ms_per_batch=round(med, 4), min_ms=round(min(ts), 4), max_ms=round(max(ts), 4),
                             real_points_per_s=round(points / a.batches / (med * 1e-3)),
                             h2d_bytes_per_batch=round(h2d[name] / a.batches))
        row["ragged"]["fps_plan"] = {str(s): fps_plan(lib, B, s) for s in sorted({strides[0], strides[-1]})}
        row["padded"]["fps_plan"] = {str(N): fps_plan(lib, B, N)}
        rows.append(row)
        print(json.dumps(row), flush=True)
    os.makedirs(a.out, exist_ok=True)
    with open(os.path.join(a.out, "ragged_host_bench.json"), "w") as f:
        json.dump({"card": info, "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
