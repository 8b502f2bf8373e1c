#!/usr/bin/env python
"""One batch norm + ReLU layer of the segmentation nets' ragged tail, three ways, forward and forward + backward.

Arms, timed alternately in one process with the method of tools/ragged_bench.py (L2 flushed before every launch, the
median of LAUNCHES launches per round, the median and [min, max] over ROUNDS rounds):
  (a) cudnn:  torch's BatchNorm1d + ReLU on the real rows alone, packed densely (no mask: the cost to aim for);
  (b) torch:  layers.masked_batch_norm + ReLU + torch.where on the padded rows (the route without the fused op);
  (c) fused:  layers.masked_batch_norm_relu (csrc/masked_bn.cu).
Rows: (R, C) = (32 768, 128) (part seg, B 16), (65 536, 128) (sem seg, B 8), (262 144, 128) (sem seg, B 32), in float32
and bfloat16, 75 % real rows.  The bytes-bound column is the HBM traffic the fused op needs at 3.35 TB/s (the H100 SXM
data sheet): forward reads x twice and writes y; forward + backward adds reading dy, y and x twice and writing dx.

    python tools/masked_bn_bench.py [--rounds 7] [--launches 20] [--json OUT]
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
from pointnet2_b200 import layers  # noqa: E402
from ragged_bench import L2_FLUSH_BYTES, gpu_info, launch_ms  # noqa: E402

ROWS = [(32768, 128), (65536, 128), (262144, 128)]
HBM_BYTES_PER_MS = 3.35e9  # 3.35 TB/s


def bytes_bound_ms(r, c, dtype, backward):
    e = torch.tensor([], dtype=dtype).element_size() * r * c
    fwd = 3 * e  # x twice, y once
    return (fwd + (6 * e if backward else 0)) / HBM_BYTES_PER_MS  # dy, y, x twice; dx once


def arms_for(r, c, dtype, backward, dev):
    g = torch.Generator(device=dev).manual_seed(r + c)
    x = (torch.randn(r, c, device=dev, generator=g) * 2 + 1).to(dtype)
    keep = torch.arange(r, device=dev) % 4 != 3
    x[~keep] = float("nan")
    dense = x[keep].contiguous()
    dy = torch.randn(r, c, device=dev, generator=g).to(dtype)
    dy_dense = dy[keep].contiguous()
    bn = torch.nn.BatchNorm1d(c).to(dev).train()
    k1 = keep.unsqueeze(1)

    def run(f, inp, grad):
        if backward:
            xx = inp.detach().requires_grad_(True)
            f(xx).backward(grad)
        else:
            with torch.no_grad():
                f(inp)

    cudnn = lambda t: torch.relu(bn(t))
    masked = lambda t: torch.where(k1, torch.relu(layers.masked_batch_norm(bn, torch.where(k1, t, 0), k1)), 0)
    fused = lambda t: layers.masked_batch_norm_relu(bn, t, keep)
    return {"cudnn": lambda: run(cudnn, dense, dy_dense), "torch": lambda: run(masked, x, dy), "fused": lambda: run(fused, x, dy)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--launches", type=int, default=20)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("masked_bn_bench.py needs a CUDA device")
    dev = torch.device("cuda:0")
    flush = torch.empty(L2_FLUSH_BYTES, dtype=torch.uint8, device=dev)
    out = {"gpu": gpu_info(), "rounds": args.rounds, "launches": args.launches, "unit": "ms per layer", "rows": []}
    print("# gpu (name, power limit, max SM clock):", out["gpu"], flush=True)
    for r, c in ROWS:
        for dtype in (torch.float32, torch.bfloat16):
            for backward in (False, True):
                arms = arms_for(r, c, dtype, backward, dev)
                for f in arms.values():  # warm-up
                    f(), f(), f()
                times = {k: [] for k in arms}
                for _ in range(args.rounds):
                    for k, f in arms.items():
                        times[k].append(launch_ms(f, flush, args.launches))
                row = {"r": r, "c": c, "dtype": str(dtype).replace("torch.", ""), "pass": "fwd+bwd" if backward else "fwd",
                       **{k: round(statistics.median(v), 4) for k, v in times.items()},
                       "spread": {k: [round(min(v), 4), round(max(v), 4)] for k, v in times.items()},
                       "bytes_bound": round(bytes_bound_ms(r, c, dtype, backward), 4)}
                out["rows"].append(row)
                print(json.dumps(row), flush=True)
    if args.json:
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
