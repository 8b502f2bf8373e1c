#!/usr/bin/env python
"""Whole-scene segmentation timings on synthetic rooms (workloads.scene_room): scene_blocks wall time (both read-backs
included) next to the host numpy restatements, the merge kernel's time against its bytes bound at 3.35 TB/s, and a
predict_scene breakdown (partition, net, merge) with a random-weight PointNet2SemSeg in eval mode at batch 16.
Prints the card's name and power limit from the same run.

    python tools/scene_bench.py [--points 150000 1000000 4000000] [--strides 1.5 0.5] [--out FILE.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import scene_oracle as SO  # noqa: E402

from pointnet2_b200 import scene, workloads as W  # noqa: E402
from pointnet2_b200.nets import PointNet2SemSeg  # noqa: E402

HBM_BPS = 3.35e12  # H100 SXM data sheet
NUM_CLASS = 21


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[torch.cuda.current_device()] if q.returncode == 0 else torch.cuda.get_device_name()


def wall(fn, reps):
    ts = []
    for _ in range(reps):
        torch.cuda.synchronize()
        t = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ts.append(time.perf_counter() - t)
    return float(np.median(ts))


def events(fn, reps):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    fn()
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / 1e3 / reps


def merge_bytes(blocks, c):
    """Each tensor the merge touches, once: point_idx and core of every row, the occ lists of the core rows' points,
    the core rows' logits, accum read and written once per point."""
    rows = blocks.point_idx.numel()
    occ = blocks.occ_row.numel()
    p = blocks.occ_off.numel() - 1
    return rows * 5 + occ * 4 * 2 + 8 * p + occ * c * 4 + p * c * 8


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--points", type=int, nargs="+", default=[150000, 1000000, 4000000])
    ap.add_argument("--strides", type=float, nargs="+", default=[1.5, 0.5])
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "scene_bench measures on a CUDA device"
    dev = torch.device("cuda:0")
    print("card:", card(), flush=True)
    torch.manual_seed(0)
    net = PointNet2SemSeg(NUM_CLASS).to(dev).eval()
    with torch.no_grad():  # library loads and GEMM algorithm choices before any timed window
        net(torch.rand(16, 8192, 3, device=dev), torch.full((16,), 8192, dtype=torch.int32, device=dev))
    rows = []
    for p in args.points:
        xyz_np, _ = W.scene_room(p, 0)
        xyz = torch.from_numpy(xyz_np).to(dev)
        for stride in args.strides:
            r = {"points": p, "stride": stride}
            blocks = scene.scene_blocks(xyz, stride=stride)
            b, n = blocks.point_idx.shape
            r.update(blocks=b, rows=n, members=int(blocks.lengths.sum()), core_rows=int(blocks.occ_row.numel()))
            r["partition_ms"] = 1e3 * wall(lambda: scene.scene_blocks(xyz, stride=stride), 5)
            t = time.perf_counter()
            SO.oracle_scene_blocks(xyz_np, stride=stride)
            r["host_oracle_ms"] = 1e3 * (time.perf_counter() - t)
            if stride == 1.5:
                t = time.perf_counter()
                SO.reference_blocks(xyz_np)
                r["host_reference_loop_ms"] = 1e3 * (time.perf_counter() - t)
            logits = torch.randn(b, n, NUM_CLASS, device=dev)
            accum = torch.zeros(p, NUM_CLASS, device=dev)
            r["merge_ms"] = 1e3 * events(lambda: scene.merge_block_logits(blocks, logits, accum), 20)
            r["merge_bytes"] = merge_bytes(blocks, NUM_CLASS)
            r["merge_bound_ms"] = 1e3 * r["merge_bytes"] / HBM_BPS
            del logits, accum
            # predict_scene, phase by phase (the loop of scene.predict_scene with events between phases)
            net_s = merge_s = 0.0
            ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            blk = scene.scene_blocks(xyz, stride=stride)
            torch.cuda.synchronize()
            part_s = time.perf_counter() - t0
            acc = torch.zeros(p, NUM_CLASS, device=dev)
            with torch.no_grad():
                for b0 in range(0, b, 16):
                    ev[0].record()
                    out = net(blk.xyz[b0:b0 + 16], blk.lengths[b0:b0 + 16])[0]
                    ev[1].record()
                    scene.merge_block_logits(blk, out, acc, row_begin=b0 * n)
                    ev[2].record()
                    ev[2].synchronize()
                    net_s += ev[0].elapsed_time(ev[1]) / 1e3
                    merge_s += ev[1].elapsed_time(ev[2]) / 1e3
            r.update(predict_partition_ms=1e3 * part_s, predict_net_ms=1e3 * net_s, predict_merge_ms=1e3 * merge_s)
            r["predict_scene_ms"] = 1e3 * wall(lambda: scene.predict_scene(net, xyz, batch_size=16, stride=stride), 1)
            rows.append(r)
            print(json.dumps(r), flush=True)
    hdr = ("points", "stride", "blocks", "rows", "partition_ms", "host_oracle_ms", "host_reference_loop_ms", "merge_ms",
           "merge_bound_ms", "predict_partition_ms", "predict_net_ms", "predict_merge_ms", "predict_scene_ms")
    print("| " + " | ".join(hdr) + " |")
    for r in rows:
        print("| " + " | ".join(f"{r[h]:.3f}" if isinstance(r.get(h), float) and h.endswith("ms") else str(r.get(h, "-"))
                                for h in hdr) + " |")
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump({"card": card(), "results": rows}, f, indent=1)


if __name__ == "__main__":
    main()
