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
    python tools/train_ddp_demo.py --model part_seg_msg --ragged --steps 30     # part segmentation, variable sizes
    python tools/train_ddp_demo.py --model sem_seg --scene-crops --steps 30     # training crops of synthetic rooms
    python tools/train_ddp_demo.py --shape-set --votes 12 --steps 30            # augmented shape batches, voted accuracy
    python tools/train_ddp_demo.py --model cls_basic --shape-set --votes 12 --steps 30   # PointNet v1 on the same
    python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 \
        tools/train_ddp_demo.py --steps 20                                      # one rank per GPU

Data is synthetic unless a dataset flag below is given: each cloud is one of `num_class` parametric shapes
(sphere, box, cylinder, cone, torus ... scaled/rotated/jittered like utils/provider.py), so the
loss has something to learn and the demo can assert that it goes down.  The part segmentation models
(part_seg, part_seg_msg) train on workloads.part_shapes instead: (B, N, 6) points with normals, one
of the 16 ShapeNet categories each, its parts the height bands of the shape.  --ragged (segmentation
models) draws each cloud's length from U[N/2, N], fills the padding rows with NaN and passes lengths=.
--scene-crops (sem_seg) trains on scene.sample_crops of a SceneSet of synthetic rooms (workloads.scene_room, 21
classes): each step's scenes come from a seeded permutation of the set, each rank draws its crops on its own GPU with a
seed derived from (step, rank), with dropout and rotation, and passes the crops' lengths and sample weights.
--shape-set (cls_ssg, cls_msg, cls_basic, part_seg, part_seg_msg) builds one shapes.ShapeSet of synthetic shapes (--set-shapes of
--set-points points: the parametric shapes above, or workloads.part_shapes for the part models) and trains on
shapes.sample_shapes batches drawn on the GPU with a seed derived from (step, rank): ModelNet's augmentation for the
classification nets, the ShapeNet part recipe (random rows, jitter, normals) for the part nets.  --votes V then prints
the accuracy of shapes.classify_votes with V rotated votes on a held-out synthetic set (classification nets).
--modelnet ROOT (cls models), --shapenet-part ROOT (part models) and --scannet ROOT (sem_seg) train on the reference's
dataset files instead (datasets.load_modelnet / load_shapenet_part / load_scannet): each implies --shape-set or
--scene-crops, the train split replaces the synthetic set and the test split the held-out one.

    python tools/train_ddp_demo.py --model cls_ssg --modelnet data/modelnet40_normal_resampled --steps 30 --votes 12
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
from pointnet2_b200 import datasets, nets, scene, shapes, workloads as W  # noqa: E402
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
    ap.add_argument("--model", choices=["cls_ssg", "cls_msg", "cls_basic", "sem_seg", "part_seg", "part_seg_msg"],
                    default="cls_ssg")
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
    ap.add_argument("--compile", choices=["none", "cudagraphs", "inductor"], default="none",
                    help="torch.compile the forward: cudagraphs = dynamo + AOTAutograd + CUDA graphs, inductor = "
                         "mode='reduce-overhead' (the library's ops are pn2:: operators inside the graph)")
    ap.add_argument("--ragged", action="store_true", help="cloud lengths from U[N/2, N], NaN padding, passed as lengths=")
    ap.add_argument("--scene-crops", action="store_true",
                    help="sem_seg only: train on seeded crops of synthetic rooms drawn on the GPU by scene.sample_crops")
    ap.add_argument("--rooms", type=int, default=6, help="rooms in the --scene-crops set")
    ap.add_argument("--scan-eval", action="store_true",
                    help="with --scene-crops: after training, the voxel accuracy on the valid fixed-view virtual scans "
                         "(scene.sample_virtual_scans) of held-out synthetic rooms")
    ap.add_argument("--shape-set", action="store_true",
                    help="cls / part models: train on augmented batches of a synthetic ShapeSet drawn by shapes.sample_shapes")
    ap.add_argument("--set-shapes", type=int, default=256, help="shapes in the --shape-set set (and in its held-out set)")
    ap.add_argument("--set-points", type=int, default=2048, help="points per shape of the --shape-set sets")
    ap.add_argument("--votes", type=int, default=0,
                    help="with --shape-set (cls models): accuracy of shapes.classify_votes with this many votes")
    ap.add_argument("--modelnet", default=None, metavar="ROOT",
                    help="cls models: train on modelnet40_normal_resampled/ at ROOT (implies --shape-set)")
    ap.add_argument("--shapenet-part", default=None, metavar="ROOT",
                    help="part models: train on shapenetcore_partanno_segmentation_benchmark_v0_normal/ at ROOT "
                         "(implies --shape-set)")
    ap.add_argument("--scannet", default=None, metavar="ROOT",
                    help="sem_seg: train on scannet_{train,test}.pickle at ROOT (implies --scene-crops)")
    args = ap.parse_args()
    if args.modelnet and args.model not in ("cls_ssg", "cls_msg", "cls_basic"):
        raise SystemExit("--modelnet trains a classification model")
    if args.shapenet_part and args.model not in ("part_seg", "part_seg_msg"):
        raise SystemExit("--shapenet-part trains a part segmentation model")
    args.shape_set = args.shape_set or bool(args.modelnet or args.shapenet_part)
    args.scene_crops = args.scene_crops or bool(args.scannet)
    if args.modelnet:
        args.num_class = len(datasets.modelnet_files(args.modelnet, "train")[2])
    if args.shape_set and (args.model == "sem_seg" or args.ragged or args.scene_crops):
        raise SystemExit("--shape-set trains the cls / part models on their own ragged batches (no --ragged)")
    if args.votes and (not args.shape_set or args.model not in ("cls_ssg", "cls_msg", "cls_basic")):
        raise SystemExit("--votes scores a classification model trained with --shape-set")
    if args.scene_crops and (args.model != "sem_seg" or args.ragged):
        raise SystemExit("--scene-crops trains the sem_seg model on its own ragged crops (no --ragged)")
    if args.scan_eval and not args.scene_crops:
        raise SystemExit("--scan-eval scores a sem_seg model trained with --scene-crops")
    if args.scene_crops:
        args.num_class = 21  # the rooms' labels
    part = args.model in ("part_seg", "part_seg_msg")
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
    elif args.model == "cls_basic":  # PointNet v1, the reference's baseline classifier
        model = nets.PointNetClsBasic(args.num_class)
    elif args.model == "part_seg":  # 50 ShapeNet parts: --num-class does not apply
        model = nets.PointNet2PartSeg()
    elif args.model == "part_seg_msg":
        model = nets.PointNet2PartSegMSG()
    else:
        model = nets.PointNet2SemSeg(args.num_class)
    model = model.to(dev)
    net = torch.nn.parallel.DistributedDataParallel(model, device_ids=[local]) if world > 1 else model
    opt = torch.optim.Adam(net.parameters(), lr=args.lr)
    if args.compile == "cudagraphs":
        fwd = torch.compile(net, backend="cudagraphs")
    elif args.compile == "inductor":
        fwd = torch.compile(net, mode="reduce-overhead")
    else:
        fwd = net
    amp_dtype = {"none": None, "bf16": torch.bfloat16, "fp16": torch.float16}[args.amp]
    scaler = torch.amp.GradScaler("cuda") if args.amp == "fp16" else None

    rs = np.random.RandomState(1234)  # the same global batch stream on every rank; each takes its slice
    if args.scene_crops:  # every rank builds the same set; only the crops' seeds differ between ranks
        if args.scannet:
            scenes = datasets.load_scannet(args.scannet, "train", device=dev)
        else:
            rooms = [W.scene_room(60000 + 20000 * k, 500 + k) for k in range(args.rooms)]
            scenes = scene.SceneSet([r[0] for r in rooms], [r[1] for r in rooms], num_class=21, device=dev)
        label_w = scenes.train_label_weights()
        order = np.zeros(0, np.int64)
    if args.shape_set:  # every rank builds the same set; only the batches' seeds differ between ranks
        if args.shapenet_part:
            shape_set = datasets.load_shapenet_part(args.shapenet_part, "trainval", device=dev)[0]
            recipe = dict(subset="random", rotate=False, perturb=False, scale=None, shift=0, with_normals=True)
        elif args.modelnet:
            shape_set = datasets.load_modelnet(args.modelnet, "train", npoints=args.num_point, device=dev)[0]
            recipe = {}
        elif part:
            pts6, cat, parts = W.part_shapes(args.set_shapes, args.set_points, 77, nets.PART_OFFSETS)
            shape_set = shapes.ShapeSet(list(pts6[:, :, :3]), cat, list(pts6[:, :, 3:]), list(parts), num_class=16,
                                        normalize=False, device=dev)
            recipe = dict(subset="random", rotate=False, perturb=False, scale=None, shift=0, with_normals=True)
        else:
            pts, cat = synthetic_shapes(args.set_shapes, args.set_points, args.num_class, np.random.RandomState(77))
            shape_set = shapes.ShapeSet(list(pts), cat, num_class=args.num_class, device=dev)
            recipe = {}
        order = np.zeros(0, np.int64)
    device_data = args.scene_crops or args.shape_set
    losses, t_steps = [], []
    for step in range(args.steps):
        seen = step * args.batch
        lr = max(args.lr * 0.7 ** (seen // args.decay_step), 1e-5)
        for g in opt.param_groups:
            g["lr"] = lr
        nets.set_bn_momentum(model, min(0.99, 1 - 0.5 * 0.5 ** (seen // args.decay_step)))
        if args.scene_crops:
            while len(order) < args.batch:  # the scenes of the global batch: a seeded permutation per epoch of the set
                order = np.concatenate([order, rs.permutation(len(scenes))])
            crop_scene = shard_batch(torch.from_numpy(order[:args.batch]), world, rank).to(dev, non_blocking=True)
            order = order[args.batch:]
            crops = scene.sample_crops(scenes, crop_scene, step * 65536 + rank, label_w, npoints=args.num_point)
            xyz, lab, lengths = crops.xyz, crops.label, crops.lengths
        elif args.shape_set:
            while len(order) < args.batch:  # the shapes of the global batch: a seeded permutation per epoch of the set
                order = np.concatenate([order, rs.permutation(len(shape_set))])
            shape_idx = shard_batch(torch.from_numpy(order[:args.batch]), world, rank).to(dev, non_blocking=True)
            order = order[args.batch:]
            batch = shapes.sample_shapes(shape_set, shape_idx, step * 65536 + rank, npoints=args.num_point, **recipe)
            xyz, lab, lengths = batch.points, batch.label, batch.lengths
            if part:
                lab_part = batch.part
        elif part:  # (B, N, 6) points with normals, per-point part labels, and the category
            xyz_np, lab_np, part_np = W.part_shapes(args.batch, args.num_point, int(rs.randint(1 << 30)), nets.PART_OFFSETS)
        else:
            xyz_np, lab_np = synthetic_shapes(args.batch, args.num_point, args.num_class, rs)
        if not device_data:
            lengths = None
        if args.ragged:
            len_np = rs.randint(args.num_point // 2, args.num_point + 1, args.batch)
            for i, l in enumerate(len_np):
                xyz_np[i, l:] = np.nan  # never read: only the first lengths[i] rows of cloud i are real
            lengths = shard_batch(torch.from_numpy(len_np.astype(np.int32)), world, rank).to(dev, non_blocking=True)
        if not device_data:
            xyz = shard_batch(torch.from_numpy(xyz_np), world, rank).to(dev, non_blocking=True).contiguous()
            lab = shard_batch(torch.from_numpy(lab_np), world, rank).to(dev, non_blocking=True)
        if part and not args.shape_set:
            lab_part = shard_batch(torch.from_numpy(part_np), world, rank).to(dev, non_blocking=True)
        torch.cuda.synchronize(dev)
        t0 = time.perf_counter()
        net.train()
        with torch.autocast(device_type="cuda", dtype=amp_dtype, enabled=amp_dtype is not None):
            if args.model == "part_seg_msg":
                pred, _ = fwd(xyz, lab, lengths=lengths)
            else:
                pred, _ = fwd(xyz, lengths=lengths)
            if part:
                loss = nets.part_seg_loss(pred, lab_part, lengths=lengths)
            elif args.scene_crops:  # the crops' labels and sample weights (label weight on core rows)
                loss = nets.sem_seg_loss(pred, lab, crops.weight, lengths=lengths)
            elif args.model == "sem_seg":  # per-point labels: the cloud's class everywhere, unit weights
                lab_pt = lab[:, None].expand(-1, args.num_point)
                loss = nets.sem_seg_loss(pred, lab_pt, torch.ones_like(lab_pt, dtype=torch.float32), lengths=lengths)
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

    voted = None
    if args.votes:  # a held-out set of the same kinds of shapes, 16 shapes per call as evaluate.py's BATCH_SIZE
        if args.modelnet:
            test_set = datasets.load_modelnet(args.modelnet, "test", npoints=args.num_point, device=dev)[0]
        else:
            pts, cat = synthetic_shapes(args.set_shapes, args.set_points, args.num_class, np.random.RandomState(99))
            test_set = shapes.ShapeSet(list(pts), cat, num_class=args.num_class, device=dev)
        model.eval()
        preds = []
        for b0 in range(0, len(test_set), 16):
            idx = torch.arange(b0, min(len(test_set), b0 + 16), device=dev)
            preds.append(shapes.classify_votes(model, test_set, idx, args.votes, 1 << 40, npoints=args.num_point).argmax(1))
        acc, class_acc = shapes.cls_accuracy(torch.cat(preds), test_set.label.long(), args.num_class)
        voted = {"votes": args.votes, "shapes": len(test_set), "accuracy": float(acc), "class_accuracy": float(class_acc)}
        if rank == 0:
            print(f"voted accuracy ({args.votes} votes, {len(test_set)} held-out shapes): {voted['accuracy']:.4f}  "
                  f"mean class accuracy {voted['class_accuracy']:.4f}", flush=True)

    scanned = None
    if args.scan_eval:  # train on crops of whole rooms, test on virtual scans (the paper's ScanNet robustness check)
        if args.scannet:
            test_scenes = datasets.load_scannet(args.scannet, "test", device=dev)
            held = range(len(test_scenes))
        else:
            held = [W.scene_room(60000 + 20000 * k, 900 + k) for k in range(3)]
            test_scenes = scene.SceneSet([r[0] for r in held], [r[1] for r in held], num_class=21, device=dev)
        views = scene.SCAN_VIEWS
        scans = scene.sample_virtual_scans(test_scenes, torch.arange(len(held) * views, device=dev) // views,
                                           torch.arange(views, device=dev).repeat(len(held)), 1 << 41,
                                           torch.ones(21, device=dev), npoints=args.num_point)
        model.eval()
        metric = scene.VoxelAccuracy(21, device=dev)
        valid = scans.valid.cpu().tolist()
        lengths_h = scans.lengths.cpu().tolist()
        with torch.no_grad():
            for b0 in range(0, len(valid), 8):
                pred, _ = model(scans.xyz[b0:b0 + 8], scans.lengths[b0:b0 + 8])
                for i in range(b0, min(b0 + 8, len(valid))):
                    if valid[i]:
                        n = lengths_h[i]
                        metric.update(scans.xyz[i, :n], scans.label[i, :n], pred[i - b0, :n].argmax(-1))
        r = metric.results()
        scanned = {"rooms": len(held), "scans": len(valid), "valid_scans": int(sum(valid)),
                   "accuracy": r["accuracy"], "class_accuracy": r["class_accuracy"],
                   "calibrated_accuracy": r["calibrated_accuracy"]}
        if rank == 0:
            print(f"virtual-scan voxel accuracy ({scanned['valid_scans']} valid scans of {len(held)} held-out rooms): "
                  f"{scanned['accuracy']:.4f}  mean class accuracy {scanned['class_accuracy']:.4f}", flush=True)

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
               "clouds_per_s": args.batch / float(np.median(steady)),
               "data": (f"ModelNet at {args.modelnet}" if args.modelnet else
                        f"ShapeNet-part at {args.shapenet_part}" if args.shapenet_part else
                        f"ScanNet at {args.scannet}" if args.scannet else
                        "synthetic room crops" if args.scene_crops else
                        "synthetic part shapes" if part else "synthetic parametric shapes"),
               "deterministic": args.deterministic, "compile": args.compile, "ragged": args.ragged, "scene_crops": args.scene_crops,
               "shape_set": args.shape_set}
        if voted is not None:
            out["voted"] = voted
        if scanned is not None:
            out["virtual_scans"] = scanned
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
