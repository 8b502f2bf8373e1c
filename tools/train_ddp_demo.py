#!/usr/bin/env python
"""Data-parallel training-step demo (SURVEY §8f n4; NOT the measured path, not bench.py).

Mirrors the structure of the reference's train_multi_gpu.py: the global batch is cut into
contiguous per-device slices (:185-188), every device runs the same network on its slice, and the
weight gradients are averaged across devices (:91-126, there on the CPU; here one NCCL all-reduce
issued by DistributedDataParallel over NVLink).  Optimiser and schedules follow :127-147,163-169:
Adam, lr 1e-3 decayed 0.7x every 200000 samples (floored at 1e-5), batch-norm decay
min(0.99, 1 - 0.5 * 0.5^(samples/200000)).

    python tools/train_ddp_demo.py --steps 20                                   # one GPU
    python tools/train_ddp_demo.py --steps 30 --amp bf16                        # bf16 autocast
    python tools/train_ddp_demo.py --steps 5 --deterministic                    # reproducible: prints a weights hash
    python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 \
        tools/train_ddp_demo.py --steps 20                                      # one rank per GPU

Data is synthetic (no dataset in this image): each cloud is one of `num_class` parametric shapes
(sphere, box, cylinder, cone, torus ... scaled/rotated/jittered like utils/provider.py), so the
loss has something to learn and the demo can assert that it goes down.
"""
from __future__ import annotations

import argparse
import hashlib
import json
import os
import sys
import time

import numpy as np
import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from pointnet2_b200 import nets  # noqa: E402
from pointnet2_b200.parallel import shard_batch  # noqa: E402


def synthetic_shapes(batch: int, num_point: int, num_class: int, rs: np.random.RandomState):
    """(batch, num_point, 3) float32 clouds in the unit sphere + (batch,) int64 labels."""
    xyz = np.empty((batch, num_point, 3), np.float32)
    labels = rs.randint(0, num_class, batch)
    for i, lab in enumerate(labels):
        u, v = rs.rand(num_point), rs.rand(num_point)
        th, z = 2 * np.pi * u, 2 * v - 1
        kind = lab % 5
        if kind == 0:    # sphere
            r = np.sqrt(1 - z * z)
            p = np.stack([r * np.cos(th), r * np.sin(th), z], 1)
        elif kind == 1:  # box surface
            p = rs.uniform(-1, 1, (num_point, 3))
            ax = rs.randint(0, 3, num_point)
            p[np.arange(num_point), ax] = rs.choice([-1.0, 1.0], num_point)
        elif kind == 2:  # cylinder
            p = np.stack([np.cos(th), np.sin(th), z], 1)
        elif kind == 3:  # cone
            h = (z + 1) / 2
            p = np.stack([(1 - h) * np.cos(th), (1 - h) * np.sin(th), z], 1)
        else:            # torus
            ph = 2 * np.pi * v
            p = np.stack([(1 + 0.35 * np.cos(ph)) * np.cos(th), (1 + 0.35 * np.cos(ph)) * np.sin(th), 0.35 * np.sin(ph)], 1)
        p = p * (1.0 + 0.15 * (lab // 5))  # classes beyond 5: same shapes, different aspect
        p[:, 2] *= 1.0 / (1.0 + 0.3 * (lab // 5))
        a = rs.uniform(0, 2 * np.pi)       # rotate about the up axis, scale, jitter (provider.py)
        rot = np.array([[np.cos(a), -np.sin(a), 0], [np.sin(a), np.cos(a), 0], [0, 0, 1]])
        p = (p @ rot.T) * rs.uniform(0.8, 1.25) + np.clip(0.01 * rs.randn(num_point, 3), -0.05, 0.05)
        p -= p.mean(0)
        xyz[i] = (p / np.sqrt((p ** 2).sum(1)).max()).astype(np.float32)
    return xyz, labels.astype(np.int64)


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", choices=["cls_ssg", "cls_msg", "sem_seg"], default="cls_ssg")
    ap.add_argument("--batch", type=int, default=32, help="GLOBAL batch (split across ranks)")
    ap.add_argument("--num-point", type=int, default=1024)
    ap.add_argument("--num-class", type=int, default=10)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--lr", type=float, default=1e-3)
    ap.add_argument("--decay-step", type=float, default=200000)
    ap.add_argument("--json", type=str, default=None)
    ap.add_argument("--amp", choices=["none", "bf16", "fp16"], default="none",
                    help="mixed precision: torch.autocast in bfloat16, or float16 with a GradScaler")
    ap.add_argument("--deterministic", action="store_true",
                    help="torch.use_deterministic_algorithms(True): run-to-run identical weights; prints their SHA-256")
    args = ap.parse_args()
    if args.deterministic:
        os.environ.setdefault("CUBLAS_WORKSPACE_CONFIG", ":4096:8")  # read when cuBLAS starts: before the first matmul
        torch.use_deterministic_algorithms(True)

    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    if not torch.cuda.is_available():
        raise SystemExit("train_ddp_demo.py needs a CUDA device: pointnet2_b200 has no CPU path")
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    if world > 1:
        dist.init_process_group("nccl", device_id=dev)
    if args.batch % world:
        raise SystemExit("--batch must be divisible by the number of ranks (train_multi_gpu.py:81 asserts the same)")

    torch.manual_seed(0)  # identical initial weights on every rank
    if args.model == "cls_ssg":
        model = nets.PointNet2ClsSSG(args.num_class)
    elif args.model == "cls_msg":
        model = nets.PointNet2ClsMSG(args.num_class)
    else:
        model = nets.PointNet2SemSeg(args.num_class)
    model = model.to(dev)
    net = torch.nn.parallel.DistributedDataParallel(model, device_ids=[local]) if world > 1 else model
    opt = torch.optim.Adam(net.parameters(), lr=args.lr)
    amp_dtype = {"none": None, "bf16": torch.bfloat16, "fp16": torch.float16}[args.amp]
    scaler = torch.amp.GradScaler("cuda") if args.amp == "fp16" else None

    rs = np.random.RandomState(1234)  # the same global batch stream on every rank; each takes its slice
    losses, t_steps = [], []
    for step in range(args.steps):
        seen = step * args.batch
        lr = max(args.lr * 0.7 ** (seen // args.decay_step), 1e-5)
        for g in opt.param_groups:
            g["lr"] = lr
        nets.set_bn_momentum(model, min(0.99, 1 - 0.5 * 0.5 ** (seen // args.decay_step)))
        xyz_np, lab_np = synthetic_shapes(args.batch, args.num_point, args.num_class, rs)
        xyz = shard_batch(torch.from_numpy(xyz_np), world, rank).to(dev, non_blocking=True).contiguous()
        lab = shard_batch(torch.from_numpy(lab_np), world, rank).to(dev, non_blocking=True)
        torch.cuda.synchronize(dev)
        t0 = time.perf_counter()
        net.train()
        with torch.autocast(device_type="cuda", dtype=amp_dtype, enabled=amp_dtype is not None):
            pred, _ = net(xyz)
            if args.model == "sem_seg":  # per-point labels: the cloud's class everywhere, unit weights
                lab_pt = lab[:, None].expand(-1, args.num_point)
                loss = nets.sem_seg_loss(pred, lab_pt, torch.ones_like(lab_pt, dtype=torch.float32))
            else:
                loss = nets.cls_loss(pred, lab)
        opt.zero_grad(set_to_none=True)
        if scaler is not None:
            scaler.scale(loss).backward()  # DDP all-reduces (averages) the gradients over NCCL here
            scaler.step(opt)
            scaler.update()
        else:
            loss.backward()  # DDP all-reduces (averages) the gradients over NCCL here
            opt.step()
        torch.cuda.synchronize(dev)
        t_steps.append(time.perf_counter() - t0)
        lv = loss.detach()
        if world > 1:
            dist.all_reduce(lv, op=dist.ReduceOp.AVG)
        losses.append(float(lv))
        if rank == 0:
            print(f"step {step:3d}  loss {losses[-1]:.4f}  lr {lr:.2e}  {t_steps[-1] * 1e3:7.1f} ms", flush=True)

    # weights must be identical on every rank after data-parallel training
    flat = torch.cat([p.detach().reshape(-1) for p in model.parameters()])
    checksum = flat.double().sum()
    same = True
    if world > 1:
        lo, hi = checksum.clone(), checksum.clone()
        dist.all_reduce(lo, op=dist.ReduceOp.MIN)
        dist.all_reduce(hi, op=dist.ReduceOp.MAX)
        same = bool(lo == hi)
    if rank == 0:
        k = max(1, args.steps // 4)
        first, last = float(np.mean(losses[:k])), float(np.mean(losses[-k:]))
        steady = t_steps[min(3, len(t_steps) - 1):]
        out = {"model": args.model, "amp": args.amp, "world": world, "global_batch": args.batch, "num_point": args.num_point,
               "steps": args.steps, "loss_first": first, "loss_last": last, "loss_decreased": last < first,
               "weights_identical_across_ranks": same, "ms_per_step_wallclock": 1e3 * float(np.median(steady)),
               "clouds_per_s": args.batch / float(np.median(steady)), "data": "synthetic parametric shapes",
               "deterministic": args.deterministic}
        if args.deterministic:
            h = hashlib.sha256()
            for p in model.parameters():
                h.update(p.detach().cpu().numpy().tobytes())
            out["weights_sha256"] = h.hexdigest()
        print(json.dumps(out))
        if args.json:
            with open(args.json, "w") as f:
                json.dump(out, f, indent=1)
    if world > 1:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
