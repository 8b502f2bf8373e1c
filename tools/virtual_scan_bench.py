#!/usr/bin/env python
"""Virtual-scan timings on synthetic rooms (workloads.scene_room): scene.sample_virtual_scans with device events at
B 8 (the 8 fixed views of one room), B 32 (the 8 fixed views of four rooms) and B 32 random views, npoints 8192, next to
one run of a host numpy restatement of scene_util.virtual_scan (scipy kd-tree) over the 8 views of one room, and the
call's share of a ragged PointNet2SemSeg training step (forward, backward, Adam) on 32 fixed-view scans.  Prints the
card's name and power limit from the same run.

    python tools/virtual_scan_bench.py [--points 150000 1000000 4000000] [--out FILE.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch
from scipy.spatial import cKDTree

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from pointnet2_b200 import nets, scene, workloads as W  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[torch.cuda.current_device()] if q.returncode == 0 else torch.cuda.get_device_name()


def events(fn, reps):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    fn()
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / reps


def _sph(v):
    xy = v[:, 0] ** 2 + v[:, 1] ** 2
    return np.arctan2(v[:, 1], v[:, 0]), np.arctan2(v[:, 2], np.sqrt(xy)), np.sqrt(xy + v[:, 2] ** 2)


def host_scan(xyz, mode):
    """One fixed view as the reference computes it on the host: rays, a kd-tree over their (az, el), the nearest ray
    of every point and the z-buffer."""
    cam = np.mean(xyz, axis=0)
    cam[2] = 1.5
    phi = np.pi / 4 * mode
    cam[:2] -= np.array([np.cos(phi), np.sin(phi)])
    ct = np.array([np.cos(phi), np.sin(phi), 0.0])
    hr = np.cross(ct, [0.0, 0.0, 1.0])
    hr /= np.linalg.norm(hr)
    vt = np.cross(hr, ct)
    vt /= np.linalg.norm(vt)
    xx, yy = np.meshgrid(np.linspace(-0.6, 0.6, 200), np.linspace(-0.45, 0.45, 150))
    rays = xx.reshape(-1, 1) * hr + yy.reshape(-1, 1) * vt + ct
    raz, rel, _ = _sph(rays)
    az, el, r = _sph(xyz - cam)
    d, k = cKDTree(np.stack([raz, rel], 1)).query(np.stack([az, el], 1))
    near = d < 0.01
    if near.sum() < 100:
        return np.zeros(0, np.int64)
    zbuf = np.full(len(rays), np.inf)
    np.minimum.at(zbuf, k[near], r[near])
    return np.nonzero(near & (r == zbuf[k]))[0]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--points", type=int, nargs="+", default=[150000, 1000000, 4000000])
    ap.add_argument("--npoints", type=int, default=8192)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    res = {"card": card(), "npoints": args.npoints, "rows": []}
    print(res["card"], flush=True)
    views = torch.arange(scene.SCAN_VIEWS, device=dev)
    for p in args.points:
        rooms = [W.scene_room(p, 200 + k) for k in range(4)]
        ss = scene.SceneSet([r[0] for r in rooms], [r[1] for r in rooms], device=dev)
        lw = ss.train_label_weights()
        seed = torch.zeros(1, dtype=torch.int64, device=dev)
        cases = [("fixed", torch.zeros(8, dtype=torch.int64, device=dev), views),
                 ("fixed", torch.arange(32, device=dev) // 8, views.repeat(4)),
                 ("random", torch.arange(32, device=dev) % 4, torch.full((32,), -1, device=dev))]
        for kind, cs, cm in cases:
            def call():
                seed.add_(1)
                return scene.sample_virtual_scans(ss, cs, cm, seed, lw, npoints=args.npoints)
            ms = events(call, 10)
            out = call()
            row = {"points": p, "batch": len(cs), "views": kind, "sample_virtual_scans_ms": ms,
                   "mean_visible": float(out.visible.float().mean()), "valid": float(out.valid.float().mean())}
            if kind == "fixed" and len(cs) == 8:
                xyz = rooms[0][0]
                t = time.perf_counter()
                vis = [len(host_scan(xyz, m)) for m in range(8)]
                row["host_numpy_ms"] = 1e3 * (time.perf_counter() - t)
                row["host_visible_mean"] = float(np.mean(vis))
            res["rows"].append(row)
            print(json.dumps(row), flush=True)
    # the call's share of a ragged training step on the 32 fixed views of four rooms of the first size
    p = args.points[0]
    rooms = [W.scene_room(p, 200 + k) for k in range(4)]
    ss = scene.SceneSet([r[0] for r in rooms], [r[1] for r in rooms], device=dev)
    lw = ss.train_label_weights()
    seed = torch.zeros(1, dtype=torch.int64, device=dev)
    cs, cm = torch.arange(32, device=dev) // 8, views.repeat(4)
    torch.manual_seed(0)
    net = nets.PointNet2SemSeg(21).to(dev).train()
    opt = torch.optim.Adam(net.parameters(), lr=1e-3)

    def scans_only():
        seed.add_(1)
        return scene.sample_virtual_scans(ss, cs, cm, seed, lw, npoints=args.npoints)

    def step():
        s = scans_only()
        pred, _ = net(s.xyz, s.lengths)
        loss = nets.sem_seg_loss(pred, s.label, s.weight, lengths=s.lengths)
        opt.zero_grad(set_to_none=True)
        loss.backward()
        opt.step()
    for _ in range(3):
        step()
    step_ms = events(step, 10)
    scan_ms = events(scans_only, 20)
    res["train_step"] = {"points": p, "batch": 32, "step_ms": step_ms, "sample_virtual_scans_ms": scan_ms,
                         "share": scan_ms / step_ms}
    print(json.dumps(res["train_step"]), flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
