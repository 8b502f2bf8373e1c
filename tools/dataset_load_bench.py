#!/usr/bin/env python
"""Dataset load timings on a seeded synthetic tree in the reference's two text formats, about 1.1 GB of text:
ModelNet40 (--modelnet files of 10,000 rows x 6 comma-separated %.6f values) and ShapeNet-part (--shapenet files of
2,800 rows x 7 blank-separated values).  The tree is read once to warm the page cache, then the reference's way
(sequential np.loadtxt, ModelNet's first 1024 rows, the same ShapeSet) and datasets.load_modelnet /
load_shapenet_part run alternately, --rounds times each.  Reports files/s and MB/s of both, the device loader's split
between waiting on reads, the host-to-device copy, the parse kernels and the host fallback, the number of fallback
files (0 on this tree), whether both ways built the same sets bit for bit, and the card's name and power limit.

    python tools/dataset_load_bench.py [--modelnet 1200] [--shapenet 2400] [--rounds 2] [--out FILE.json]
"""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle.dataset_ref import PART_CATEGORIES  # noqa: E402
from pointnet2_b200 import datasets, shapes as SH  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[torch.cuda.current_device()] if q.returncode == 0 else torch.cuda.get_device_name()


def _line_pool(rng, n, ncol, sep, last_int=None):
    a = rng.uniform(-1, 1, (n, ncol))
    if last_int is not None:
        a[:, -1] = rng.integers(0, last_int, n)
    return [sep.join("%.6f" % v for v in row).encode() + b"\n" for row in a]


def write_tree(root, n_modelnet, n_shapenet, seed=0):
    """Files assembled from pools of formatted lines: the formats' byte statistics without formatting 1 GB."""
    rng = np.random.default_rng(seed)
    mn, sn = os.path.join(root, "modelnet"), os.path.join(root, "shapenet")
    classes = [f"class{k:02d}" for k in range(40)]
    os.makedirs(mn)
    with open(os.path.join(mn, "shape_names.txt"), "w") as f:
        f.write("\n".join(classes) + "\n")
    pool = _line_pool(rng, 1 << 16, 6, ",")
    ids = []
    for k in range(n_modelnet):
        c = classes[k % 40]
        os.makedirs(os.path.join(mn, c), exist_ok=True)
        sid = f"{c}_{k:05d}"
        with open(os.path.join(mn, c, sid + ".txt"), "wb") as f:
            f.write(b"".join(pool[i] for i in rng.integers(0, len(pool), 10000)))
        ids.append(sid)
    for split, lst in (("train", ids), ("test", ids[:1])):
        with open(os.path.join(mn, f"modelnet40_{split}.txt"), "w") as f:
            f.write("\n".join(lst) + "\n")
    os.makedirs(os.path.join(sn, "train_test_split"))
    with open(os.path.join(sn, "synsetoffset2category.txt"), "w") as f:
        f.write("".join(f"{n}\t{s}\n" for n, s in PART_CATEGORIES))
    pool = _line_pool(rng, 1 << 16, 7, " ", last_int=50)
    listed = []
    for k in range(n_shapenet):
        syn = PART_CATEGORIES[k % 16][1]
        os.makedirs(os.path.join(sn, syn), exist_ok=True)
        tok = f"{k:032x}"
        with open(os.path.join(sn, syn, tok + ".txt"), "wb") as f:
            f.write(b"".join(pool[i] for i in rng.integers(0, len(pool), 2800)))
        listed.append(f"shape_data/{syn}/{tok}")
    for split, lst in (("train", listed), ("val", []), ("test", [])):
        with open(os.path.join(sn, "train_test_split", f"shuffled_{split}_file_list.json"), "w") as f:
            json.dump(lst, f)
    return mn, sn


def reference_modelnet(root, dev):
    paths, labels, names = datasets.modelnet_files(root, "train")
    pts = [np.loadtxt(p, delimiter=",").astype(np.float32)[0:1024, :] for p in paths]
    return SH.ShapeSet([p[:, 0:3] for p in pts], labels, num_class=len(names), device=dev)


def reference_shapenet(root, dev):
    paths, labels, names = datasets.shapenet_part_files(root, "trainval")
    data = [np.loadtxt(p).astype(np.float32) for p in paths]
    return SH.ShapeSet([d[:, 0:3] for d in data], labels, [d[:, 3:6] for d in data],
                       [d[:, -1].astype(np.int32) for d in data], num_class=len(names), device=dev)


def same_set(a, b):
    def eq(x, y):
        return (x is None and y is None) or torch.equal(x.view(torch.int32) if x.dtype == torch.float32 else x,
                                                       y.view(torch.int32) if y.dtype == torch.float32 else y)
    return all(eq(getattr(a, k), getattr(b, k)) for k in ("xyz", "normals", "part", "label", "offsets"))


def timed(fn):
    torch.cuda.synchronize()
    t = time.perf_counter()
    r = fn()
    torch.cuda.synchronize()
    return r, time.perf_counter() - t


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--modelnet", type=int, default=1200)
    ap.add_argument("--shapenet", type=int, default=2400)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("dataset_load_bench.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    tmp = tempfile.mkdtemp(prefix="pn2_dataset_bench_")
    try:
        t = time.perf_counter()
        mn, sn = write_tree(tmp, args.modelnet, args.shapenet)
        out = {"gpu": card(), "write_s": time.perf_counter() - t}
        for name, root, fmt in (("modelnet", mn, (6, datasets.DELIM_COMMA, 1024)),
                                ("shapenet", sn, (7, datasets.DELIM_WHITESPACE, 1 << 62))):
            paths = (datasets.modelnet_files(root, "train")[0] if name == "modelnet"
                     else datasets.shapenet_part_files(root, "trainval")[0])
            mb = sum(os.path.getsize(p) for p in paths) / 1e6
            for p in paths:  # warm the page cache
                with open(p, "rb") as f:
                    f.read()
            ref_fn = (lambda: reference_modelnet(root, dev)) if name == "modelnet" else (lambda: reference_shapenet(root, dev))
            dev_fn = ((lambda: datasets.load_modelnet(root, "train", 1024, device=dev)[0]) if name == "modelnet"
                      else (lambda: datasets.load_shapenet_part(root, "trainval", device=dev)[0]))
            dev_fn()  # module load and first-launch costs
            ref_t, dev_t, same = [], [], True
            for _ in range(args.rounds):
                a, ta = timed(ref_fn)
                b, tb = timed(dev_fn)
                ref_t.append(ta)
                dev_t.append(tb)
                same = same and same_set(a, b)
                del a, b
            stats = {}
            timed(lambda: datasets._read_tables(paths, fmt[0], fmt[1], keep=fmt[2], device=dev, stats=stats))
            r, d = min(ref_t), min(dev_t)
            out[name] = {"files": len(paths), "MB": round(mb, 1), "same_sets": bool(same),
                         "reference_s": [round(x, 3) for x in ref_t], "device_s": [round(x, 3) for x in dev_t],
                         "reference_files_per_s": round(len(paths) / r, 1), "device_files_per_s": round(len(paths) / d, 1),
                         "reference_MB_per_s": round(mb / r, 1), "device_MB_per_s": round(mb / d, 1),
                         "speedup": round(r / d, 2),
                         "split_s": {k: round(stats[k], 4) for k in ("read_wait_s", "copy_s", "parse_s", "host_s")},
                         "chunks": stats["chunks"], "fallback_files": stats["fallback"]}
            print(name, json.dumps(out[name]), flush=True)
        print("# gpu (name, power limit, max SM clock):", out["gpu"], flush=True)
        if args.out:
            with open(args.out, "w") as f:
                json.dump(out, f, indent=1)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


if __name__ == "__main__":
    main()
