#!/usr/bin/env python
"""Shape-batch timings on a synthetic shape set (512 shapes of 10,000 points with normals, ModelNet's resampled size):
shapes.sample_shapes with device events at B 16 / 32 / 64 x npoints 1024 / 2048, and at npoints 10,000 with normals,
for both row subsets; a host numpy restatement of ModelNetDataset.next_batch(augment=True) (first npoints rows, the five
provider.py steps, shuffle_points) and of the part loader (resampling with replacement, jitter) at the same sizes; a
PointNet2ClsSSG training step (forward, backward, Adam) at B 32 on device batches against one on host batches; and
classify_votes at V = 12 over a 2468-shape synthetic test set.  Prints the card's name and power limit from the same run.

    python tools/shape_batch_bench.py [--shapes 512] [--test-shapes 2468] [--out FILE.json]
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

from pointnet2_b200 import nets, shapes as SH  # noqa: E402


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


def synthetic_set(n_shapes, n_points, num_class, seed):
    """Ellipsoid-like point sets with unit normals and a class each (the shapes only need to be distinct)."""
    rs = np.random.RandomState(seed)
    xyz, nrm = [], []
    for k in range(n_shapes):
        d = rs.standard_normal((n_points, 3))
        d /= np.linalg.norm(d, axis=1, keepdims=True)
        xyz.append((d * (1 + 0.5 * rs.random_sample(3)) + 0.01 * rs.standard_normal((n_points, 3))).astype(np.float32))
        nrm.append(d.astype(np.float32))
    return xyz, nrm, rs.randint(0, num_class, n_shapes)


def rot_y(a):
    c, s = np.cos(a), np.sin(a)
    return np.array([[c, 0, s], [0, 1, 0], [-s, 0, c]])


def host_modelnet_batch(cache, idx, npoints, normals, rs):
    """next_batch(augment=True) of modelnet_dataset.py:60-72,84 on the cached (normalised) shapes."""
    ch = 6 if normals else 3
    data = np.zeros((len(idx), npoints, ch))
    for i, s in enumerate(idx):
        data[i] = cache[s][:npoints, :ch]
    for k in range(len(data)):                      # rotate_point_cloud[_with_normal]
        r = rot_y(rs.uniform() * 2 * np.pi)
        data[k, :, 0:3] = data[k, :, 0:3] @ r
        if normals:
            data[k, :, 3:6] = data[k, :, 3:6] @ r
    for k in range(len(data)):                      # rotate_perturbation_point_cloud[_with_normal]
        a = np.clip(0.06 * rs.randn(3), -0.18, 0.18)
        rx = np.array([[1, 0, 0], [0, np.cos(a[0]), -np.sin(a[0])], [0, np.sin(a[0]), np.cos(a[0])]])
        rz = np.array([[np.cos(a[2]), -np.sin(a[2]), 0], [np.sin(a[2]), np.cos(a[2]), 0], [0, 0, 1]])
        r = rz @ (rot_y(a[1]) @ rx)
        data[k, :, 0:3] = data[k, :, 0:3] @ r
        if normals:
            data[k, :, 3:6] = data[k, :, 3:6] @ r
    xyz = data[:, :, 0:3]
    xyz *= rs.uniform(0.8, 1.25, len(data))[:, None, None]
    xyz += rs.uniform(-0.1, 0.1, (len(data), 3))[:, None, :]
    xyz += np.clip(0.01 * rs.randn(*xyz.shape), -0.05, 0.05)
    perm = np.arange(npoints)
    rs.shuffle(perm)
    return data[:, perm].astype(np.float32)


def host_part_batch(cache, idx, npoints, rs):
    """part_dataset_all_normal.py:103-107 (npoints rows with replacement) + part_seg/train.py:200 (jitter)."""
    data = np.zeros((len(idx), npoints, 6), np.float32)
    for i, s in enumerate(idx):
        data[i] = cache[s][rs.choice(len(cache[s]), npoints, replace=True)]
    data[:, :, 0:3] += np.clip(0.01 * rs.randn(len(idx), npoints, 3), -0.05, 0.05)
    return data


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", type=int, default=512)
    ap.add_argument("--points", type=int, default=10000)
    ap.add_argument("--test-shapes", type=int, default=2468)
    ap.add_argument("--votes", type=int, default=12)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    res = {"card": card(), "rows": []}
    print(res["card"], flush=True)
    xyz, nrm, lab = synthetic_set(args.shapes, args.points, 40, 0)
    ss = SH.ShapeSet(xyz, lab, nrm, num_class=40, device=dev)
    cache = np.concatenate([ss.xyz.cpu().numpy(), ss.normals.cpu().numpy()], 1)
    cache = np.split(cache, ss.offsets.cpu().numpy()[1:-1])
    seed = torch.zeros(1, dtype=torch.int64, device=dev)
    part_kw = dict(subset="random", rotate=False, perturb=False, scale=None, shift=0, with_normals=True)
    sizes = [(b, n, False) for b in (16, 32, 64) for n in (1024, 2048)] + [(b, args.points, True) for b in (16, 32, 64)]
    for subset in ("first", "random"):
        for b, n, normals in sizes:
            idx_np = np.random.RandomState(b).randint(0, args.shapes, b)
            idx = torch.from_numpy(idx_np).to(dev)
            kw = dict(with_normals=normals) if subset == "first" else part_kw

            def call():
                seed.add_(1)
                return SH.sample_shapes(ss, idx, seed, npoints=n, **kw)
            ms = events(call, 50)
            rs = np.random.RandomState(0)
            t = time.perf_counter()
            reps = 3
            for _ in range(reps):
                if subset == "first":
                    host_modelnet_batch(cache, idx_np, n, normals, rs)
                else:
                    host_part_batch(cache, idx_np, n, rs)
            host_ms = 1e3 * (time.perf_counter() - t) / reps
            row = {"subset": subset, "batch": b, "npoints": n, "normals": normals or subset == "random",
                   "sample_shapes_ms": ms, "host_numpy_ms": host_ms}
            res["rows"].append(row)
            print(json.dumps(row), flush=True)

    # a cls_ssg training step at B 32, npoints 1024: device batches against host batches (numpy + copy)
    torch.manual_seed(0)
    net = nets.PointNet2ClsSSG(40).to(dev).train()
    opt = torch.optim.Adam(net.parameters(), lr=1e-3)
    rs = np.random.RandomState(1)
    idx_np = rs.randint(0, args.shapes, 32)
    idx = torch.from_numpy(idx_np).to(dev)
    label_h = torch.from_numpy(lab[idx_np].astype(np.int64)).to(dev)

    def train(points, label, lengths=None):
        pred, _ = net(points, lengths)
        loss = nets.cls_loss(pred, label)
        opt.zero_grad(set_to_none=True)
        loss.backward()
        opt.step()

    def step_device():
        seed.add_(1)
        bt = SH.sample_shapes(ss, idx, seed)
        train(bt.points, bt.label, bt.lengths)

    def step_host():
        pts = torch.from_numpy(host_modelnet_batch(cache, idx_np, 1024, False, rs)).pin_memory().to(dev, non_blocking=True)
        train(pts, label_h)
    for fn in (step_device, step_host):
        for _ in range(3):
            fn()
    torch.cuda.synchronize()
    out = {}
    for name, fn in (("device_batches", step_device), ("host_batches", step_host)):
        t = time.perf_counter()
        for _ in range(20):
            fn()
        torch.cuda.synchronize()
        out[name + "_step_ms"] = 1e3 * (time.perf_counter() - t) / 20
    res["train_step"] = {"batch": 32, "npoints": 1024, **out}
    print(json.dumps(res["train_step"]), flush=True)

    # classify_votes over a ModelNet40-sized test set, 16 shapes per call as evaluate.py's BATCH_SIZE
    txyz, _, tlab = synthetic_set(args.test_shapes, args.points, 40, 1)
    ts = SH.ShapeSet(txyz, tlab, num_class=40, device=dev)
    net.eval()
    order = torch.arange(args.test_shapes, device=dev)

    def evaluate():
        preds = []
        for b0 in range(0, args.test_shapes, 16):
            logits = SH.classify_votes(net, ts, order[b0:b0 + 16], args.votes, b0)
            preds.append(logits.argmax(1))
        return SH.cls_accuracy(torch.cat(preds), ts.label.long(), 40)
    evaluate()
    torch.cuda.synchronize()
    t = time.perf_counter()
    acc, _ = evaluate()
    torch.cuda.synchronize()
    res["votes"] = {"shapes": args.test_shapes, "votes": args.votes, "seconds": time.perf_counter() - t,
                    "accuracy_untrained": float(acc)}
    print(json.dumps(res["votes"]), flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
