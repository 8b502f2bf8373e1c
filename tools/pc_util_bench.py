#!/usr/bin/env python
"""Voxel and pillar grouping timings (pointnet2_b200.pc_util, csrc/voxel.cu) on the reference's own sizes: a batch of
32 ModelNet-size clouds (workloads.cloud_surface, 4096 points, in the unit sphere) converted by

  volume_v2: point_cloud_to_volume_v2_batch, V 12, num_sample 128  -> (32, 12, 12, 12, 128, 3) float64
  image:     point_cloud_to_image_batch, I 32, num_sample 128      -> (32, 32, 32, 128, 3) float64
  volume:    point_cloud_to_volume_batch, V 12                     -> (32, 1728) float64

For each: GPU time by CUDA events after warm-up, the bytes the outputs take and the rate that makes; the reference's
own function (utils/pc_util.py, through oracle/pcutil_ref.py, where it is present) on one host core over the same
batch, and whether the two results are equal (no cell here holds more than 128 points, so no draw is involved); and
the card's name and power limit read in the same run.

    python tools/pc_util_bench.py [--reps 50] [--out FILE.json]
"""
import os

for _v in ("OMP_NUM_THREADS", "OPENBLAS_NUM_THREADS", "MKL_NUM_THREADS"):  # the host side on one core
    os.environ[_v] = "1"

import argparse  # noqa: E402
import json  # noqa: E402
import subprocess  # noqa: E402
import sys  # noqa: E402
import time  # noqa: E402

import numpy as np  # noqa: E402
import torch  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import pcutil_ref as PR  # noqa: E402
from pointnet2_b200 import pc_util, workloads as W  # noqa: E402

B, N, S = 32, 4096, 128


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[torch.cuda.current_device()] if q.returncode == 0 else torch.cuda.get_device_name()


def events(fn, reps):
    for _ in range(3):
        fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / reps


def host(fn):
    if fn is None:
        return None, None
    t = time.perf_counter()
    out = fn()
    return 1e3 * (time.perf_counter() - t), out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    torch.set_num_threads(1)
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    res = {"card": card(), "rows": []}
    print(res["card"], flush=True)
    pts = W.cloud_surface(B, N, 1)
    x = torch.from_numpy(pts).to(dev)
    ref = PR.load_pc_util()
    cases = [
        ("volume_v2", 12, lambda: pc_util.point_cloud_to_volume_v2_batch(x, 12, 1.0, S),
         None if ref is None else (lambda: ref.point_cloud_to_volume_v2_batch(pts, 12, 1.0, S)), B * 12 ** 3 * S),
        ("image", 32, lambda: pc_util.point_cloud_to_image_batch(x, 32, 1.0, S),
         None if ref is None else (lambda: ref.point_cloud_to_image_batch(pts, 32, 1.0, S)), B * 32 ** 2 * S),
        ("volume", 12, lambda: pc_util.point_cloud_to_volume_batch(x, 12, 1.0),
         None if ref is None else (lambda: ref.point_cloud_to_volume_batch(pts, 12, 1.0)), 0),
    ]
    for name, grid, gpu, cpu, slots in cases:
        row = {"workload": name, "clouds": B, "points": N, "grid": grid, "nsample": S if slots else None}
        row["gpu_ms"] = events(gpu, args.reps)
        cells = B * grid ** (2 if name == "image" else 3)
        # outputs: count (4 B per cell), idx (4 B) and grouped (24 B) per slot, and the returned tensor
        row["output_bytes"] = cells * 4 + slots * 28 if slots else cells * (4 + 4 + 28 + 8)
        row["output_GBps"] = row["output_bytes"] / row["gpu_ms"] / 1e6
        row["reference_host_ms"], want = host(cpu)
        if want is not None:
            row["speedup"] = row["reference_host_ms"] / row["gpu_ms"]
            row["equal_to_reference"] = bool(np.array_equal(gpu().cpu().numpy(), want))
        print(json.dumps(row), flush=True)
        res["rows"].append(row)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
