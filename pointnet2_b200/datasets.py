"""The reference's dataset files as shape and scene sets (DESIGN.md §6.18).

``load_modelnet`` and ``load_shapenet_part`` read the same files, in the same order, as the reference's
``ModelNetDataset`` (modelnet_dataset.py:23-46, 74-90) and ``PartNormalDataset`` (part_seg/part_dataset_all_normal.py:
19-97), and build a ``ShapeSet`` from exactly the rows those readers cache.  The point text is parsed on the GPU
(pn2_text_rows_scan / pn2_text_rows_parse): files are read into pinned chunks by a thread pool while the previous
chunk is parsed, and a file outside the device grammar is parsed with the reference's own ``np.loadtxt`` call.
``load_scannet`` reads the reference's ScanNet pickles (scannet/scannet_dataset.py:13-16) into a ``SceneSet`` through
an unpickler that admits numpy arrays and nothing else.
"""
from __future__ import annotations

import concurrent.futures as cf
import json
import os
import pickle
import time

import numpy as np
import torch

from . import _lib
from ._tensor import ptr, stream_ptr
from .scene import SceneSet
from .shapes import ShapeSet

DELIM_WHITESPACE, DELIM_COMMA = 0, 1  # pn2_api.h PN2_DELIM_*
TEXT_REASONS = {1: "syntax", 2: "fields", 3: "blank", 4: "cr", 5: "comment", 6: "inexact"}  # pn2_api.h PN2_TEXT_*
_NO_CAP = 1 << 62
_READERS = 8


def _loadtxt(path: str, delim: int) -> np.ndarray:
    """The reference's own parse of one file (modelnet_dataset.py:84, part_dataset_all_normal.py:88)."""
    if delim == DELIM_COMMA:
        return np.loadtxt(path, delimiter=",").astype(np.float32)
    return np.loadtxt(path).astype(np.float32)


def _refuse_short(path: str, shape) -> None:
    raise ValueError(f"{path}: a point file needs at least two rows of values, it gives an array of shape "
                     f"{tuple(shape)} (the reference's readers fail on it too)")


def _read_into(path: str, buf: np.ndarray) -> None:
    with open(path, "rb", buffering=0) as f:
        view, got = memoryview(buf), 0
        while got < len(buf):
            n = f.readinto(view[got:])
            if not n:
                raise OSError(f"{path}: the file shrank while it was read")
            got += n


def _read_tables(paths, ncol: int, delim: int, keep: int = _NO_CAP, device=None, chunk_bytes: int = 256 << 20,
                 stats: dict | None = None) -> list:
    """One float32 table per file: np.loadtxt(path, ...).astype(np.float32)[:keep], bit for bit.

    Files go to the GPU in chunks of at most ``chunk_bytes`` (a larger file is a chunk of its own), two pinned host
    buffers deep: the readers fill one while the other is copied and parsed.  Each chunk is read back once.  A file
    the device marks is parsed with np.loadtxt on the host.  Empty and one-row files raise ValueError.  ``stats``,
    when given, receives the counts and the time spent waiting on reads, copying, parsing and in the host fallback."""
    paths = list(paths)
    dev = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
    sizes = [os.path.getsize(p) for p in paths]
    chunks, cur, cur_bytes = [], [], 0
    for i, s in enumerate(sizes):
        if cur and cur_bytes + s > chunk_bytes:
            chunks.append(cur)
            cur, cur_bytes = [], 0
        cur.append(i)
        cur_bytes += s
    if cur:
        chunks.append(cur)
    cap = max(sum(sizes[i] for i in c) for c in chunks) if chunks else 0
    st = dict(files=len(paths), bytes=int(sum(sizes)), chunks=len(chunks), fallback=0, reasons={}, read_wait_s=0.0,
              copy_s=0.0, parse_s=0.0, host_s=0.0)
    out = [None] * len(paths)
    if not paths:
        return out
    lib = _lib.load()
    host = [torch.empty(cap, dtype=torch.uint8, pin_memory=True) for _ in range(min(2, len(chunks)))]
    with torch.cuda.device(dev), cf.ThreadPoolExecutor(_READERS) as pool:
        text = torch.empty(cap, dtype=torch.uint8, device=dev)
        stream = stream_ptr(dev)

        def submit(k):
            buf, off, futs = host[k % 2].numpy(), 0, []
            for i in chunks[k]:
                futs.append(pool.submit(_read_into, paths[i], buf[off:off + sizes[i]]))
                off += sizes[i]
            return futs

        pending = submit(0)
        for k, files in enumerate(chunks):
            t = time.perf_counter()
            for fut in pending:
                fut.result()
            st["read_wait_s"] += time.perf_counter() - t
            nb = sum(sizes[i] for i in files)
            ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
            ev[0].record()
            text[:nb].copy_(host[k % 2][:nb], non_blocking=True)
            ev[1].record()
            pending = submit(k + 1) if k + 1 < len(chunks) else []  # overlaps the parse below
            off = np.zeros(len(files) + 1, np.int64)
            np.cumsum([sizes[i] for i in files], out=off[1:])
            file_off = torch.from_numpy(off).to(dev, non_blocking=False)
            rows = torch.empty(len(files), dtype=torch.int64, device=dev)
            status = torch.empty(len(files), dtype=torch.int32, device=dev)
            _lib.check(lib.pn2_text_rows_scan(len(files), ptr(text), ptr(file_off), nb, ncol, delim, ptr(rows),
                                              ptr(status), stream), "pn2_text_rows_scan")
            rows_h, status_h = rows.cpu().numpy(), status.cpu().numpy()  # the one sync of the chunk before its rows
            kept = np.where(status_h == 0, np.minimum(rows_h, keep), 0)
            row_off = np.zeros(len(files) + 1, np.int64)
            np.cumsum(kept, out=row_off[1:])
            table = torch.empty((int(row_off[-1]), ncol), dtype=torch.float32, device=dev)
            if row_off[-1]:  # else every file of the chunk is the host's
                _lib.check(lib.pn2_text_rows_parse(len(files), ptr(text), ptr(file_off), nb, ncol, delim, ptr(status),
                                                   keep, ptr(torch.from_numpy(row_off).to(dev)), ptr(table),
                                                   int(row_off[-1]), stream), "pn2_text_rows_parse")
            ev[2].record()
            table_h = table.cpu().numpy()
            st["copy_s"] += ev[0].elapsed_time(ev[1]) / 1e3
            st["parse_s"] += ev[1].elapsed_time(ev[2]) / 1e3
            t = time.perf_counter()
            for j, i in enumerate(files):
                if status_h[j] == 0:
                    if rows_h[j] < 2:
                        _refuse_short(paths[i], (int(rows_h[j]), ncol))
                    out[i] = table_h[row_off[j]:row_off[j + 1]]
                else:
                    st["fallback"] += 1
                    why = TEXT_REASONS.get(int(status_h[j]), str(int(status_h[j])))
                    st["reasons"][why] = st["reasons"].get(why, 0) + 1
                    a = _loadtxt(paths[i], delim)
                    if a.ndim != 2 or len(a) < 2:
                        _refuse_short(paths[i], a.shape)
                    out[i] = a[:keep]
            st["host_s"] += time.perf_counter() - t
    if stats is not None:
        stats.update(st)
    return out


def _lines(path: str) -> list:
    with open(path) as f:
        return [line.rstrip() for line in f]


def modelnet_files(root: str, split: str = "train", modelnet10: bool = False):
    """(paths, labels, class_names) of a ModelNet split in the reference's order (modelnet_dataset.py:29-46): the
    class list file, the split's id list, class = the id without its last '_' part, path = root/class/id.txt."""
    if split not in ("train", "test"):
        raise ValueError(f"load_modelnet: split must be 'train' or 'test', got {split!r}")
    tag = "modelnet10" if modelnet10 else "modelnet40"
    names = _lines(os.path.join(root, "modelnet10_shape_names.txt" if modelnet10 else "shape_names.txt"))
    classes = dict(zip(names, range(len(names))))
    ids = _lines(os.path.join(root, f"{tag}_{split}.txt"))
    cls = ["_".join(x.split("_")[0:-1]) for x in ids]
    return [os.path.join(root, c, i) + ".txt" for c, i in zip(cls, ids)], [classes[c] for c in cls], names


def load_modelnet(root: str, split: str = "train", npoints: int = 1024, normalize: bool = True,
                  normal_channel: bool = False, modelnet10: bool = False, device=None):
    """``modelnet40_normal_resampled/`` (or its ModelNet10 lists) as a ShapeSet and its class names.

    Shape k is what ModelNetDataset(root, npoints=npoints, split=split, normalize=normalize,
    normal_channel=normal_channel, modelnet10=modelnet10)._get_item(k) caches: the file's first npoints rows, xyz
    pc_normalize'd in float32 when ``normalize``, normals (columns 3-5) when ``normal_channel``; label its class."""
    if isinstance(npoints, bool) or not isinstance(npoints, int) or npoints < 1:
        raise ValueError(f"load_modelnet expects a positive integer npoints, got {npoints!r}")
    paths, labels, names = modelnet_files(root, split, modelnet10)
    tables = _read_tables(paths, 6, DELIM_COMMA, keep=npoints, device=device)
    if normal_channel:
        for p, t in zip(paths, tables):
            if t.shape[1] != 6:
                raise ValueError(f"{p}: normal_channel needs 6 columns (xyz, normal), the file has {t.shape[1]}")
    shapes = ShapeSet([t[:, 0:3] for t in tables], labels,
                      normal_list=[t[:, 3:6] for t in tables] if normal_channel else None, num_class=len(names),
                      normalize=normalize, device=device)
    return shapes, names


def shapenet_part_files(root: str, split: str = "trainval"):
    """(paths, labels, category_names) of a ShapeNet-part split in the reference's order
    (part_dataset_all_normal.py:29-67): categories in synsetoffset2category.txt line order, each category's
    directory listing sorted and filtered by the split's train_test_split lists."""
    if split not in ("trainval", "train", "val", "test"):
        raise ValueError(f"load_shapenet_part: split must be 'trainval', 'train', 'val' or 'test', got {split!r}")
    cat = {}
    with open(os.path.join(root, "synsetoffset2category.txt")) as f:
        for line in f:
            ls = line.strip().split()
            cat[ls[0]] = ls[1]
    ids = {}
    for s in ("train", "val", "test"):
        with open(os.path.join(root, "train_test_split", f"shuffled_{s}_file_list.json")) as f:
            ids[s] = set(str(d.split("/")[2]) for d in json.load(f))
    want = {"trainval": ids["train"] | ids["val"], "train": ids["train"], "val": ids["val"], "test": ids["test"]}[split]
    paths, labels = [], []
    for k, item in enumerate(cat):
        d = os.path.join(root, cat[item])
        for fn in sorted(os.listdir(d)):
            if fn[0:-4] in want:
                paths.append(os.path.join(d, os.path.splitext(os.path.basename(fn))[0] + ".txt"))
                labels.append(k)
    return paths, labels, list(cat)


def load_shapenet_part(root: str, split: str = "trainval", normalize: bool = True, device=None):
    """``shapenetcore_partanno_segmentation_benchmark_v0_normal/`` as a ShapeSet and its category names.

    Shape k is what PartNormalDataset(root, split=split, normalize=normalize) caches for index k: xyz (columns 0-2)
    pc_normalize'd in float32 when ``normalize``, normals (3-5), part = the last column cast to int32; label the
    category's line in synsetoffset2category.txt."""
    paths, labels, names = shapenet_part_files(root, split)
    tables = _read_tables(paths, 7, DELIM_WHITESPACE, device=device)
    shapes = ShapeSet([t[:, 0:3] for t in tables], labels, normal_list=[t[:, 3:6] for t in tables],
                      part_list=[t[:, -1].astype(np.int32) for t in tables], num_class=len(names),
                      normalize=normalize, device=device)
    return shapes, names


class _ArrayUnpickler(pickle.Unpickler):
    """Admits the globals a pickled numpy array names and refuses every other one before it can be called."""

    _ALLOWED = {
        ("numpy.core.multiarray", "_reconstruct"): np._core.multiarray._reconstruct,  # Python 2 / numpy 1 home
        ("numpy._core.multiarray", "_reconstruct"): np._core.multiarray._reconstruct,
        ("numpy", "ndarray"): np.ndarray,
        ("numpy", "dtype"): np.dtype,
    }

    def find_class(self, module, name):
        try:
            return self._ALLOWED[(module, name)]
        except KeyError:
            raise pickle.UnpicklingError(f"refusing the global {module}.{name}: a dataset pickle holds numpy arrays "
                                         "only") from None


def read_scannet_pickle(path: str):
    """(points list, labels list): the two successive pickles of scannet_{split}.pickle, latin-1 as Python 2 wrote
    them (scannet_dataset.py:13-16)."""
    with open(path, "rb") as fp:
        points = _ArrayUnpickler(fp, encoding="latin1").load()
        labels = _ArrayUnpickler(fp, encoding="latin1").load()
    return points, labels


def load_scannet(root: str, split: str = "train", num_class: int = 21, device=None) -> SceneSet:
    """``scannet_{split}.pickle`` as a SceneSet.  Its train_label_weights() are scannet_dataset.py:17-24's weights;
    the reference's test split uses ones."""
    points, labels = read_scannet_pickle(os.path.join(root, f"scannet_{split}.pickle"))
    return SceneSet(points, labels, num_class=num_class, device=device)
