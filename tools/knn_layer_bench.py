#!/usr/bin/env python
"""Time the kNN set-abstraction layer (FPS + gather + knn_point + centred xyz grouping) on the GPU: the op sequence
against the one-call layer (sa_layer.sample_knn) on the path its rule picks, and on each path forced
(pn2_set_sa_knn_path), next to the sampling kernel alone and knn_point alone.  `c_over_t` is the ratio the rule
bounds: knn_point's SM time per query over one sampling step.  Each round flushes L2 and runs every variant once,
in alternating order; the JSON has the median, minimum and maximum over the rounds.

    python tools/knn_layer_bench.py --out DIR [--rounds 15]
"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from pointnet2_b200 import _lib, workloads as W  # noqa: E402
from pointnet2_b200.sa_layer import sample_knn  # noqa: E402
from pointnet2_b200.tf_grouping import group_point, knn_point  # noqa: E402
from pointnet2_b200.tf_sampling import farthest_point_sample_and_gather  # noqa: E402

# (label, cloud, b, n, npoint, k)
SHAPES = [("cfg2", "U", 32, 4096, 1024, 32), ("cfg2 duplicates", "D", 32, 4096, 1024, 32),
          ("b40", "U", 40, 4096, 1024, 32), ("b40 duplicates", "D", 40, 4096, 1024, 32),
          ("b64", "U", 64, 4096, 1024, 32), ("b64 duplicates", "D", 64, 4096, 1024, 32),
          ("n4096 k64 b16 duplicates", "D", 16, 4096, 1024, 64), ("n4096 k64 b26", "U", 26, 4096, 1024, 64),
          ("n4096 k64 b32", "U", 32, 4096, 1024, 64), ("n4096 k64 b32 duplicates", "D", 32, 4096, 1024, 64),
          ("n1024 k32", "U", 16, 1024, 512, 32), ("n1024 k64", "U", 16, 1024, 512, 64),
          ("n1024 k64 duplicates", "D", 16, 1024, 512, 64), ("n1024 k128", "U", 16, 1024, 512, 128),
          ("n4096 k8 b44", "U", 44, 4096, 1024, 8), ("n8192", "U", 8, 8192, 1024, 32), ("b80", "U", 80, 1024, 512, 32)]


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = "nvidia-smi unavailable"
    return {"torch_name": name, "nvidia_smi": q}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True, help="directory for knn_layer_bench.json")
    ap.add_argument("--rounds", type=int, default=11)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("knn_layer_bench needs a CUDA device")
    dev = torch.device("cuda:0")
    lib = _lib.load()
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    info = card()
    print(info, flush=True)
    rows = []
    for label, gen, b, n, m, k in SHAPES:
        x = torch.from_numpy(W.DISTRIBUTIONS[gen](b, n, 300)).to(dev)
        _, nx = farthest_point_sample_and_gather(m, x)

        def sequential():
            _, q = farthest_point_sample_and_gather(m, x)
            _, idx = knn_point(k, x, q)
            return group_point(x, idx) - q.unsqueeze(2)

        def path(mode):
            def f():
                lib.pn2_set_sa_knn_path(mode)
                sample_knn(m, k, x, center=True)
            return f

        variants = {"sampling alone": lambda: farthest_point_sample_and_gather(m, x),
                    "knn_point alone": lambda: knn_point(k, x, nx),
                    "sequential ops": sequential,
                    "layer": path(0), "layer, overlapped": path(1), "layer, sequential": path(2)}
        for f in variants.values():  # warm-up: module loads, function attributes
            f()
        lib.pn2_set_sa_knn_path(0)
        before = _lib.launch_count()
        want = sequential()
        got = sample_knn(m, k, x, center=True)[4]
        assert torch.equal(got, want), label
        rule = "overlapped" if _lib.launch_count() - before == 5 else "sequential"  # 3 sequential ops, then 2 or 3
        times = {name: [] for name in variants}
        names = list(variants)
        for r in range(a.rounds):
            for name in (names if r % 2 == 0 else names[::-1]):
                flush.zero_()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                variants[name]()
                e1.record()
                e1.synchronize()
                times[name].append(e0.elapsed_time(e1))
        lib.pn2_set_sa_knn_path(0)
        row = dict(shape=label, cloud=gen, b=b, n=n, npoint=m, k=k, fits=int(lib.pn2_sa_knn_layer_fits(n, k)), rule=rule)
        for name, ts in times.items():
            row[name] = dict(median_ms=round(float(np.median(ts)), 4), min_ms=round(min(ts), 4), max_ms=round(max(ts), 4))
        sms = torch.cuda.get_device_properties(0).multi_processor_count
        c = row["knn_point alone"]["median_ms"] * sms / (b * m)
        row["c_over_t"] = round(c / (row["sampling alone"]["median_ms"] / m), 2)
        rows.append(row)
        print(json.dumps(row), flush=True)
    os.makedirs(a.out, exist_ok=True)
    with open(os.path.join(a.out, "knn_layer_bench.json"), "w") as f:
        json.dump({"card": info, "rounds": a.rounds, "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
