#!/usr/bin/env python
"""Point-cloud rendering timings (render.show_points, csrc/render.cu) on the two workloads a user of the viewer runs:

  shapes: 64 ShapeNet-size clouds (workloads.cloud_surface, 2048 points) drawn twice, with ground-truth and predicted
          part colours (part_seg/test.py:83-85), ball radius 8 on 800 x 800: one call of 128 images;
  scene:  one workloads.scene_room scene of 10^6 points coloured by label, radius 8, at 800^2 and 1600^2, 1 and 8 views.

For each: GPU time by CUDA events after warm-up (show_points end to end, and render_balls alone on the projected
points), the pixel atomics issued and skipped in one counted call, the (point, pattern entry) pairs that land on the
canvas, the reference's render_ball on one host core (oracle/_ref/libref_render.so, where it is present) over the same
images, and the card's name and power limit read in the same run.

    python tools/render_bench.py [--reps 20] [--out FILE.json]
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import render_ref as RR  # noqa: E402
from pointnet2_b200 import _lib, render, workloads as W  # noqa: E402
from pointnet2_b200._tensor import ptr, stream_ptr  # noqa: E402

RADIUS = 8


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


def counted(ixyz, colors, size, lengths=None):
    """(issued, skipped) pixel atomics of one render_balls call on (B, N, 3) int32 points."""
    lib = _lib.load()
    b, n, _ = ixyz.shape
    wsb = int(lib.pn2_render_balls_workspace_bytes(b, size, size))
    ws = torch.empty(wsb, dtype=torch.uint8, device=ixyz.device)
    out = torch.empty((b, size, size, 3), dtype=torch.uint8, device=ixyz.device)
    cnt = torch.zeros(2, dtype=torch.int64, device=ixyz.device)
    bg = (ctypes.c_ubyte * 3)(0, 0, 0)
    rc = lib.pn2_render_balls_counted(b, n, size, size, ptr(ixyz), ptr(colors), ptr(lengths), RADIUS, bg, ptr(ws), wsb,
                                      ptr(out), ptr(cnt), stream_ptr(ixyz.device))
    _lib.check(rc, "pn2_render_balls_counted")
    issued, skipped = cnt.tolist()
    return issued, skipped


def candidates(ixyz, size):
    """(point, pattern entry) pairs on the canvas, from the shapes: per pattern row dx, the run of columns it covers."""
    pat = [(dx, int(np.sqrt(RADIUS * RADIUS - dx * dx - 1))) for dx in range(-RADIUS + 1, RADIUS)]  # dy^2 < r^2 - dx^2
    x, y = ixyz[..., 0].long(), ixyz[..., 1].long()
    total = 0
    for dx, half in pat:
        row_ok = ((x + dx) >= 0) & ((x + dx) < size)
        lo, hi = torch.clamp(y - half, min=0), torch.clamp(y + half, max=size - 1)
        total += int((row_ok * torch.clamp(hi - lo + 1, min=0)).sum())
    return total


def host_reference(ixyz, colors, size):
    """render_ball on one host core over every image; None without oracle/_ref/libref_render.so."""
    if not RR.have_refrender():
        return None
    ix = ixyz.cpu().numpy()
    col = None if colors is None else colors.cpu().numpy()
    t = time.perf_counter()
    for i in range(ix.shape[0]):
        RR.refrender_ball(ix[i], None if col is None else col[i], size, size, RADIUS)
    return 1e3 * (time.perf_counter() - t)


def measure(name, xyz, colors, size, views, reps):
    xa = list(np.linspace(-0.6, 0.6, views)) if views > 1 else 0.3
    ixyz = render.project_points(xyz, size, xa, 0.2).reshape(-1, xyz.shape[1], 3)
    v = ixyz.shape[0] // xyz.shape[0]
    cols = None
    if colors is not None:
        c = colors.double()
        c = (c / ((c.amax(dim=1, keepdim=True) + 1e-14) / 255.0)).float()
        cols = c[:, None].expand(-1, v, -1, -1).reshape(-1, xyz.shape[1], 3).contiguous()
    row = {"workload": name, "images": ixyz.shape[0], "points": xyz.shape[1], "size": size, "views": views,
           "radius": RADIUS}
    row["show_points_ms"] = events(lambda: render.show_points(xyz, colors, size=size, xangle=xa, yangle=0.2,
                                                              ballradius=RADIUS), reps)
    row["render_balls_ms"] = events(lambda: render.render_balls(ixyz, cols, size, size, RADIUS), reps)
    row["project_points_ms"] = events(lambda: render.project_points(xyz, size, xa, 0.2), reps)
    row["atomics_issued"], row["atomics_skipped"] = counted(ixyz, cols, size)
    row["pairs_on_canvas"] = candidates(ixyz, size)
    row["reference_host_ms"] = host_reference(ixyz, cols, size)
    if row["reference_host_ms"] is not None:
        row["speedup_render_balls"] = row["reference_host_ms"] / row["render_balls_ms"]
    print(json.dumps(row), flush=True)
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    res = {"card": card(), "rows": []}
    print(res["card"], flush=True)
    rng = np.random.RandomState(0)
    palette = torch.from_numpy(rng.rand(50, 3)).to(dev)  # float64 colour-map rows
    shapes = torch.from_numpy(W.cloud_surface(64, 2048, 1)).to(dev)
    gt = torch.from_numpy(rng.randint(0, 50, (64, 2048))).to(dev)
    pred = torch.where(torch.from_numpy(rng.rand(64, 2048) < 0.1).to(dev), (gt + 1) % 50, gt)
    xyz = torch.cat([shapes, shapes]).double()
    res["rows"].append(measure("shapes_gt_pred", xyz, torch.cat([palette[gt], palette[pred]]), 800, 1, args.reps))
    pts, label = W.scene_room(1_000_000, 7)
    scene = torch.from_numpy(pts[None]).to(dev).double()
    lab = torch.from_numpy(label[None]).to(dev)
    for size in (800, 1600):
        for views in (1, 8):
            res["rows"].append(measure("scene_1e6", scene, palette[lab], size, views, max(3, args.reps // views)))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
