#!/usr/bin/env python
"""Training-crop timings on synthetic rooms (workloads.scene_room): scene.sample_crops with device events at B 8 / 16 / 32
and npoints 8192, next to a host numpy restatement of ScannetDataset.__getitem__ + get_batch_wdp +
rotate_point_cloud_z (resampling with replacement, as the reference does), and the crop call's share of a ragged
PointNet2SemSeg training step (forward, backward, Adam) at B 32.  Prints the card's name and power limit from the same
run.

    python tools/scene_crop_bench.py [--points 150000 1000000 4000000] [--rooms 2] [--out FILE.json]
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


def host_crop(point_set, semantic_seg, labelweights, npoints, rs):
    """One training crop on the host as the reference draws it: ten attempted 1.5 m columns, the first with >= 70 %
    labelled points and >= 2 % occupied voxels, resampled to npoints with replacement."""
    coordmax, coordmin = point_set.max(0), point_set.min(0)
    for _ in range(10):
        centre = point_set[rs.randint(len(point_set))].astype(np.float64)
        lo = np.array([centre[0] - 0.75, centre[1] - 0.75, coordmin[2]])
        hi = np.array([centre[0] + 0.75, centre[1] + 0.75, coordmax[2]])
        inside = np.all((point_set >= lo - 0.2) & (point_set <= hi + 0.2), axis=1)
        pts, seg = point_set[inside], semantic_seg[inside]
        core = np.all((pts >= lo - 0.01) & (pts <= hi + 0.01), axis=1)
        v = np.ceil((pts[core] - lo) / (hi - lo) * [31.0, 31.0, 62.0])
        nvox = len(np.unique(v[:, 0] * 31.0 * 62.0 + v[:, 1] * 62.0 + v[:, 2]))
        if np.mean(seg > 0) >= 0.7 and nvox / 31.0 / 31.0 / 62.0 >= 0.02:
            break
    choice = rs.randint(0, len(seg), npoints)
    return pts[choice], seg[choice], labelweights[seg[choice]] * core[choice]


def host_batch(scenes, labels, idx, labelweights, npoints, rs):
    """get_batch_wdp (dropout onto row 0) + rotate_point_cloud_z for the crops of scenes idx."""
    data = np.zeros((len(idx), npoints, 3))
    lab = np.zeros((len(idx), npoints), np.int32)
    smpw = np.zeros((len(idx), npoints), np.float32)
    for i, s in enumerate(idx):
        data[i], lab[i], smpw[i] = host_crop(scenes[s], labels[s], labelweights, npoints, rs)
        drop = np.nonzero(rs.random_sample(npoints) <= rs.random_sample() * 0.875)[0]
        data[i, drop], lab[i, drop] = data[i, 0], lab[i, 0]
        smpw[i, drop] = 0
    out = np.zeros(data.shape, np.float32)
    for i in range(len(idx)):
        a = rs.uniform() * 2 * np.pi
        c, s = np.cos(a), np.sin(a)
        out[i] = data[i] @ np.array([[c, s, 0], [-s, c, 0], [0, 0, 1]])
    return out, lab, smpw


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--points", type=int, nargs="+", default=[150000, 1000000, 4000000])
    ap.add_argument("--rooms", type=int, default=2, help="rooms per scene set")
    ap.add_argument("--batches", type=int, nargs="+", default=[8, 16, 32])
    ap.add_argument("--npoints", type=int, default=8192)
    ap.add_argument("--host-batch", type=int, default=8, help="crops per host-timed batch (the host loop is slow)")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    res = {"card": card(), "npoints": args.npoints, "rows": []}
    print(res["card"], flush=True)
    for p in args.points:
        rooms = [W.scene_room(p, 100 + k) for k in range(args.rooms)]
        ss = scene.SceneSet([r[0] for r in rooms], [r[1] for r in rooms], device=dev)
        lw = ss.train_label_weights()
        seed = torch.zeros(1, dtype=torch.int64, device=dev)
        for b in args.batches:
            cs = torch.arange(b, device=dev) % args.rooms

            def call():
                seed.add_(1)
                return scene.sample_crops(ss, cs, seed, lw, npoints=args.npoints)
            ms = events(call, 20)
            crops = call()
            row = {"points": p, "batch": b, "sample_crops_ms": ms,
                   "mean_length": float(crops.lengths.float().mean()), "valid": float(crops.valid.float().mean())}
            if b == args.host_batch:
                rs = np.random.RandomState(0)
                idx = np.arange(b) % args.rooms
                t = time.perf_counter()
                host_batch([r[0] for r in rooms], [r[1] for r in rooms], idx, lw.cpu().numpy(), args.npoints, rs)
                row["host_numpy_ms"] = 1e3 * (time.perf_counter() - t)
            res["rows"].append(row)
            print(json.dumps(row), flush=True)
    # the crop call's share of a ragged training step at B 32 on the first set
    p = args.points[0]
    rooms = [W.scene_room(p, 100 + k) for k in range(args.rooms)]
    ss = scene.SceneSet([r[0] for r in rooms], [r[1] for r in rooms], device=dev)
    lw = ss.train_label_weights()
    seed = torch.zeros(1, dtype=torch.int64, device=dev)
    cs = torch.arange(32, device=dev) % args.rooms
    torch.manual_seed(0)
    net = nets.PointNet2SemSeg(21).to(dev).train()
    opt = torch.optim.Adam(net.parameters(), lr=1e-3)

    def crops_only():
        seed.add_(1)
        return scene.sample_crops(ss, cs, seed, lw, npoints=args.npoints)

    def step():
        c = crops_only()
        pred, _ = net(c.xyz, c.lengths)
        loss = nets.sem_seg_loss(pred, c.label, c.weight, lengths=c.lengths)
        opt.zero_grad(set_to_none=True)
        loss.backward()
        opt.step()
    for _ in range(3):
        step()
    step_ms = events(step, 10)
    crop_ms = events(crops_only, 20)
    res["train_step"] = {"points": p, "batch": 32, "step_ms": step_ms, "sample_crops_ms": crop_ms,
                         "share": crop_ms / step_ms}
    print(json.dumps(res["train_step"]), flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
