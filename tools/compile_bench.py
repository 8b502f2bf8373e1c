"""Eager against torch.compile for the networks' training step and eval forward.

Arms, run alternately in every round of one process:
  eager       the library's ctypes launches and the torch layers, as they run without compile;
  cudagraphs  torch.compile(backend="cudagraphs"): dynamo + AOTAutograd, the step replayed as CUDA graphs, no
              generated kernels;
  inductor    torch.compile(mode="reduce-overhead"): inductor's kernels for the torch layers, plus CUDA graphs.
The compiled region is the forward and the loss (AOTAutograd compiles their backward); the SGD step runs after it.
Per row and arm: the median CUDA-event time per step over the rounds with [min, max], the GPU kernel time per step
from a separate torch.profiler run, and the wall time of the first (compiling) call.  The card's name and power limit
are read in the same run.

    python tools/compile_bench.py --out /tmp/compile_bench.json
"""
from __future__ import annotations

import argparse
import copy
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from pointnet2_b200 import nets, workloads as W  # noqa: E402

ROWS = {  # name: (net, batch, points, ragged)
    "sem_seg": (nets.PointNet2SemSeg, 8, 8192, False),
    "sem_seg_ragged": (nets.PointNet2SemSeg, 8, 8192, True),
    "cls_ssg": (nets.PointNet2ClsSSG, 32, 1024, False),
    "part_seg": (nets.PointNet2PartSeg, 16, 2048, False),
    "cls_basic": (nets.PointNetClsBasic, 32, 1024, False),
}
ARMS = ("eager", "cudagraphs", "inductor")


def card():
    name = torch.cuda.get_device_name(0)
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        power = r.stdout.strip() or "unknown"
    except (OSError, subprocess.SubprocessError):
        power = "unknown"
    return name, power


def inputs(row, dev):
    cls, b, n, ragged = ROWS[row]
    xyz = torch.from_numpy(W.cloud_uniform(b, n, 3)).to(dev)
    if cls is nets.PointNet2PartSeg:
        xyz = torch.cat([xyz, torch.nn.functional.normalize(torch.randn(b, n, 3, device=dev), dim=-1)], -1).contiguous()
    lens = None
    if ragged:
        lens = torch.randint(n // 2, n + 1, (b,), device=dev, generator=torch.Generator(dev).manual_seed(1)).to(torch.int32)
    return xyz, lens


def loss_fn(row, pred, lens):
    b = pred.shape[0]
    if pred.dim() == 2:
        return nets.cls_loss(pred, torch.arange(b, device=pred.device) % pred.shape[-1])
    label = (torch.arange(pred.shape[1], device=pred.device) % pred.shape[-1]).expand(b, -1)
    if row.startswith("sem_seg"):
        return nets.sem_seg_loss(pred, label, torch.ones(label.shape, device=pred.device), lengths=lens)
    return nets.part_seg_loss(pred, label, lengths=lens)


def make_arm(row, arm, base, kind):
    net = copy.deepcopy(base)
    if kind == "train":
        net.train()

        def fn(x, lens):
            return loss_fn(row, net(x, lengths=lens)[0], lens)
    else:
        net.eval()

        def fn(x, lens):
            with torch.no_grad():
                return net(x, lengths=lens)[0]
    if arm == "cudagraphs":
        fn = torch.compile(fn, backend="cudagraphs", fullgraph=True)
    elif arm == "inductor":
        fn = torch.compile(fn, mode="reduce-overhead", fullgraph=True)
    opt = torch.optim.SGD(net.parameters(), lr=1e-4) if kind == "train" else None

    def step(x, lens):
        out = fn(x, lens)
        if opt is not None:
            out.backward()
            opt.step()
            opt.zero_grad(set_to_none=True)
        return out
    return step


def run_row(row, kind, args, dev):
    torch._dynamo.reset()
    torch.manual_seed(0)
    base = ROWS[row][0]().to(dev)
    for m in base.modules():
        if isinstance(m, torch.nn.Dropout):
            m.p = 0.0
    x, lens = inputs(row, dev)
    steps, res = {}, {}
    for arm in args.arms:
        steps[arm] = make_arm(row, arm, base, kind)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        steps[arm](x, lens)
        torch.cuda.synchronize()
        first = time.perf_counter() - t0
        for _ in range(args.warmup):
            steps[arm](x, lens)
        torch.cuda.synchronize()
        res[arm] = {"first_call_s": first, "rounds_ms": []}
    for _ in range(args.rounds):
        for arm in args.arms:
            start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            start.record()
            for _ in range(args.steps):
                steps[arm](x, lens)
            end.record()
            end.synchronize()
            res[arm]["rounds_ms"].append(start.elapsed_time(end) / args.steps)
    for arm in args.arms:  # kernel time: a separate, profiled run
        n_prof = 5
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            for _ in range(n_prof):
                steps[arm](x, lens)
            torch.cuda.synchronize()
        kern = sum(e.self_device_time_total for e in prof.key_averages() if e.self_device_time_total > 0)
        r = res[arm]
        r["kernel_ms"] = kern / 1e3 / n_prof
        r["median_ms"] = float(np.median(r["rounds_ms"]))
        r["min_ms"], r["max_ms"] = float(min(r["rounds_ms"])), float(max(r["rounds_ms"]))
    return res


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--rows", nargs="+", default=list(ROWS), choices=list(ROWS))
    ap.add_argument("--arms", nargs="+", default=list(ARMS), choices=list(ARMS))
    ap.add_argument("--kinds", nargs="+", default=["train", "eval"], choices=["train", "eval"])
    ap.add_argument("--steps", type=int, default=20, help="steps per timed round")
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--out", default=None, help="JSON file for every row")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("compile_bench needs a CUDA device")
    dev = torch.device("cuda:0")
    name, power = card()
    rows = []
    for row in args.rows:
        for kind in args.kinds:
            res = run_row(row, kind, args, dev)
            for arm, r in res.items():
                rec = {"row": row, "kind": kind, "arm": arm, "batch": ROWS[row][1], "points": ROWS[row][2],
                       "median_ms": round(r["median_ms"], 3), "min_ms": round(r["min_ms"], 3),
                       "max_ms": round(r["max_ms"], 3), "kernel_ms": round(r["kernel_ms"], 3),
                       "first_call_s": round(r["first_call_s"], 2), "gpu": name, "power_limit": power}
                rows.append(rec)
                print(json.dumps(rec), flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
