#!/usr/bin/env python
"""What a batch of variable-size clouds costs, on one GPU, against two ways of feeding it without lengths.

Arms, timed alternately in one process, the L2 flushed before every launch (as bench.py does):
  (a) dense:    today's call on full clouds of n points;
  (b) ragged:   the same call with `lengths` drawn uniformly from [n/2, n] and NaN in the padding rows;
  (c) resample: the clouds of (b) resampled to n points with replacement (what a loader does without lengths,
                e.g. a ScanNet crop), through the dense call.
Shapes: cfg2 (B 32, N 4096 -> 1024, S 32, r 0.1) and the first sem-seg level (B 16, N 8192 -> 1024) through the fused
sampling+grouping layer, cfg2 and a cluster plan (B 8, N 65 536 -> 16 384) through FPS + gather alone.  Feature
propagation at the last sem-seg level (B 16, 8192 <- 1024 known points, C 128 + 0): the fused front end
(fp_interpolate_concat, also at B 64) and the deterministic three_interpolate gradient; and one PointNet2SemSeg training step (forward,
sem_seg_loss, backward; B 8, N 8192).  Each number is the median over ROUNDS rounds of the median of LAUNCHES launches.

    python tools/ragged_bench.py [--rounds 5] [--launches 20] [--json OUT] [--only NAMES] [--profile]

--profile adds, per row and arm, a torch.profiler record of a few calls (after the timed rounds): the summed GPU kernel
time per call, the wall time per call with a device synchronise, and the kernels whose time differs most between the
dense and the ragged arm.  The difference between wall time and kernel time is time the GPU waits for the host.
"""
from __future__ import annotations

import argparse
import collections
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from pointnet2_b200 import _lib, workloads as W  # noqa: E402
from pointnet2_b200._tensor import ptr, stream_ptr  # noqa: E402
from pointnet2_b200.nets import PointNet2SemSeg, sem_seg_loss  # noqa: E402
from pointnet2_b200.sa_layer import sample_group  # noqa: E402
from pointnet2_b200.tf_interpolate import fp_interpolate_concat, three_nn_interpolate  # noqa: E402
from pointnet2_b200.tf_sampling import farthest_point_sample_and_gather  # noqa: E402

L2_FLUSH_BYTES = 256 << 20  # > the 50 MB L2 of the H100
SHAPES = [
    # name, b, n, npoint, radius, nsample (radius None: FPS + gather only)
    ("cfg2", 32, 4096, 1024, 0.1, 32),
    ("cfg2_fps", 32, 4096, 1024, None, None),
    ("semseg_l1", 16, 8192, 1024, 0.1, 32),
    ("fps_cluster", 8, 65536, 16384, None, None),
    # feature propagation rows: radius / nsample hold the row kind
    ("fp4_front", 16, 8192, 1024, "fp_front", 128),
    ("fp4_front_b64", 64, 8192, 1024, "fp_front", 128),  # four waves of CTAs instead of one
    ("fp4_det_grad", 16, 8192, 1024, "det_grad", 128),
    ("semseg_train_step", 8, 8192, None, "train", 13),
]


def fp_arms(kind, b, n, m, c, full, ragged, lens, resampled, dev):
    """the three arms of a feature-propagation row; the known level is dense (the first m points of every full cloud)"""
    known = full[:, :m].contiguous()
    g = torch.Generator(device="cpu").manual_seed(7)
    feats = torch.randn(b, m, c, generator=g).to(dev)
    if kind == "fp_front":
        call = lambda x, lengths=None: fp_interpolate_concat(x, known, None, feats, lengths=lengths)
        return {"dense": lambda: call(full), "ragged": lambda: call(ragged, lens), "resample": lambda: call(resampled)}
    # the deterministic gradient of three_interpolate, through the C entry (grad_out's padding rows are NaN when ragged)
    lib = _lib.load()
    wsb = int(lib.pn2_three_interpolate_grad_det_workspace_bytes(b, n, m))
    ws = torch.empty(wsb, dtype=torch.uint8, device=dev)
    gp = torch.empty(b, m, c, device=dev)
    arms = {}
    for name, x, lg in (("dense", full, None), ("ragged", ragged, lens), ("resample", resampled, None)):
        _, _, idx, w = three_nn_interpolate(x, known, feats, return_aux=True, lengths=lg)
        go = torch.randn(b, n, c, generator=g).to(dev)
        if lg is not None:
            go[torch.isnan(x[..., 0])] = float("nan")

        def run(idx=idx, w=w, go=go, lg=lg):
            if lg is None:
                rc = lib.pn2_three_interpolate_grad_det(b, n, c, m, ptr(go), ptr(idx), ptr(w), ptr(gp), ptr(ws), wsb, stream_ptr(dev))
            else:
                rc = lib.pn2_three_interpolate_grad_det_ragged_typed(0, b, n, c, m, ptr(go), ptr(idx), ptr(w), ptr(lg), ptr(gp),
                                                                     ptr(ws), wsb, stream_ptr(dev))
            _lib.check(rc, "three_interpolate grad det")
        arms[name] = run
    return arms


def train_arms(b, n, num_class, full, ragged, lens, resampled, dev):
    """one PointNet2SemSeg training step per arm (no optimiser step, so every launch sees the same weights)"""
    torch.manual_seed(0)
    net = PointNet2SemSeg(num_class=num_class).to(dev).train()
    rs = np.random.RandomState(9)
    label = torch.from_numpy(rs.randint(0, num_class, (b, n))).to(dev)
    smpw = torch.ones(b, n, device=dev)

    def step(x, lengths=None):
        net.zero_grad(set_to_none=True)
        pred, _ = net(x, lengths=lengths)
        sem_seg_loss(pred, label, smpw, lengths=lengths).backward()
    return {"dense": lambda: step(full), "ragged": lambda: step(ragged, lens), "resample": lambda: step(resampled)}


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


def profile_arms(arms, calls=5):
    """per arm: kernel ms per call, wall ms per call, and per-kernel ms per call"""
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile
    res = {}
    for k, f in arms.items():
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
            t0 = time.perf_counter()
            for _ in range(calls):
                f()
            torch.cuda.synchronize()
            wall = (time.perf_counter() - t0) * 1e3 / calls
        per = collections.Counter()
        for e in prof.key_averages():
            if e.device_type == DeviceType.CUDA:
                per[e.key] += e.self_device_time_total / 1e3 / calls
        res[k] = {"kernel_ms": round(sum(per.values()), 4), "wall_ms": round(wall, 4), "kernels": len(per), "per": per}
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--launches", type=int, default=20)
    ap.add_argument("--json", default=None)
    ap.add_argument("--only", default=None, help="comma-separated shape names to run (default: all)")
    ap.add_argument("--profile", action="store_true", help="add a torch.profiler breakdown per row and arm")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("ragged_bench.py needs a CUDA device")
    dev = torch.device("cuda:0")
    flush = torch.empty(L2_FLUSH_BYTES, dtype=torch.uint8, device=dev)
    out = {"gpu": gpu_info(), "rounds": args.rounds, "launches": args.launches, "unit": "ms per call", "shapes": []}
    print("# gpu (name, power limit, max SM clock):", out["gpu"], flush=True)
    for name, b, n, m, r, s in SHAPES:
        if args.only and name not in args.only.split(","):
            continue
        full, ragged, lens, resampled, host_lengths = inputs(b, n, 100, dev)
        if r in ("fp_front", "det_grad"):
            arms = fp_arms(r, b, n, m, s, full, ragged, lens, resampled, dev)
        elif r == "train":
            arms = train_arms(b, n, s, full, ragged, lens, resampled, dev)
        else:
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
        if args.profile:
            prof = profile_arms(arms)
            d, r_ = prof["dense"]["per"], prof["ragged"]["per"]
            diff = sorted(set(d) | set(r_), key=lambda name: -abs(r_[name] - d[name]))[:12]
            row["profile"] = {k: {x: v[x] for x in ("kernel_ms", "wall_ms", "kernels")} for k, v in prof.items()}
            row["profile"]["ragged_minus_dense_ms"] = [[name[:90], round(r_[name] - d[name], 4), round(d[name], 4)] for name in diff]
        out["shapes"].append(row)
        print(json.dumps(row), flush=True)
    if args.json:
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
