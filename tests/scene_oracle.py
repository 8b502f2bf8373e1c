"""Plain numpy restatements for the whole-scene tests and tools/scene_bench.py (test infrastructure only).

oracle_scene_blocks   the block partition exactly as pointnet2_b200.scene defines it, one block at a time
reference_blocks      the reference's loop, scannet/scannet_dataset.py:94-103 (without the resampling at :104)
reference_voxel_labels  scannet/pc_util.py:39-51 (point_cloud_label_to_surface_voxel_label_fast)
"""
from __future__ import annotations

import numpy as np


def plan_axis(lo: float, hi: float, size: float, stride: float) -> int:
    """The smallest k >= 1 with lo + (k - 1) * stride + size >= hi, by counting up."""
    k = 1
    while not lo + (k - 1) * stride + size >= hi:
        k += 1
    return k


def oracle_scene_blocks(xyz: np.ndarray, block_size=1.5, stride=None, padding=0.2, max_points=8192) -> dict:
    """The outputs of scene_blocks as numpy arrays (keys: the SceneBlocks fields), one block at a time."""
    stride = block_size if stride is None else stride
    xyz = np.asarray(xyz, np.float32)
    p = len(xyz)
    x, y = xyz[:, 0].astype(np.float64), xyz[:, 1].astype(np.float64)
    lo = xyz.min(0).astype(np.float64)
    hi = xyz.max(0).astype(np.float64)
    nx, ny = plan_axis(lo[0], hi[0], block_size, stride), plan_axis(lo[1], hi[1], block_size, stride)
    subs = []  # (members, core mask, i, j, q)
    for i in range(nx):
        bx = lo[0] + i * stride
        colx = (x >= bx - padding) & (x <= bx + block_size + padding)
        corex = (x >= bx - 0.001) & (x <= bx + block_size + 0.001)
        for j in range(ny):
            by = lo[1] + j * stride
            members = np.nonzero(colx & (y >= by - padding) & (y <= by + block_size + padding))[0]
            core = (corex[members] & (y[members] >= by - 0.001) & (y[members] <= by + block_size + 0.001))
            if not core.any():
                continue
            k = -(-len(members) // max_points)
            for q in range(k):
                subs.append((members[q::k], core[q::k], i, j, q))
    b, n = len(subs), max(len(s[0]) for s in subs)
    out = {"xyz": np.zeros((b, n, 3), np.float32), "lengths": np.zeros(b, np.int32),
           "point_idx": np.full((b, n), -1, np.int32), "core": np.zeros((b, n), bool), "block": np.zeros((b, 3), np.int32)}
    for s, (members, core, i, j, q) in enumerate(subs):
        c = len(members)
        out["xyz"][s, :c] = xyz[members]
        out["lengths"][s] = c
        out["point_idx"][s, :c] = members
        out["core"][s, :c] = core
        out["block"][s] = (i, j, q)
    flat = np.nonzero(out["core"].reshape(-1))[0]
    pts = out["point_idx"].reshape(-1)[flat]
    order = np.lexsort((flat, pts))
    out["occ_off"] = np.concatenate([[0], np.cumsum(np.bincount(pts, minlength=p))]).astype(np.int32)
    out["occ_row"] = flat[order].astype(np.int32)
    return out


def reference_blocks(point_set_ini: np.ndarray):
    """scannet_dataset.py:86-103 as written (block 1.5, context 0.2, core 0.001), without the resampling: for every
    (i, j) the reference forms, the context members (ascending scene index) and their core mask."""
    coordmax = np.max(point_set_ini, axis=0)
    coordmin = np.min(point_set_ini, axis=0)
    nsubvolume_x = np.ceil((coordmax[0] - coordmin[0]) / 1.5).astype(np.int32)
    nsubvolume_y = np.ceil((coordmax[1] - coordmin[1]) / 1.5).astype(np.int32)
    out = {}
    for i in range(nsubvolume_x):
        for j in range(nsubvolume_y):
            curmin = coordmin + [i * 1.5, j * 1.5, 0]
            curmax = coordmin + [(i + 1) * 1.5, (j + 1) * 1.5, coordmax[2] - coordmin[2]]
            curchoice = np.sum((point_set_ini >= (curmin - 0.2)) * (point_set_ini <= (curmax + 0.2)), axis=1) == 3
            cur_point_set = point_set_ini[curchoice, :]
            if len(cur_point_set) == 0:
                continue
            mask = np.sum((cur_point_set >= (curmin - 0.001)) * (cur_point_set <= (curmax + 0.001)), axis=1) == 3
            out[(i, j)] = (np.nonzero(curchoice)[0], mask)
    return out


def reference_voxel_labels(point_cloud: np.ndarray, label: np.ndarray, res=0.0484):
    """pc_util.py:39-51 as written."""
    coordmax = np.max(point_cloud, axis=0)
    coordmin = np.min(point_cloud, axis=0)
    nvox = np.ceil((coordmax - coordmin) / res)
    vidx = np.ceil((point_cloud - coordmin) / res)
    vidx = vidx[:, 0] + vidx[:, 1] * nvox[0] + vidx[:, 2] * nvox[0] * nvox[1]
    uvidx, vpidx = np.unique(vidx, return_index=True)
    if label.ndim == 1:
        uvlabel = label[vpidx]
    else:
        assert label.ndim == 2
        uvlabel = label[vpidx, :]
    return uvidx, uvlabel, nvox


def sequential_merge(blocks: dict, logits: np.ndarray, accum: np.ndarray, row_begin: int = 0) -> np.ndarray:
    """The merge restated one add at a time in float32: for each point, its core rows in [row_begin, row_begin +
    logits rows) in ascending order."""
    acc = accum.astype(np.float32).copy()
    lg = logits.reshape(-1, logits.shape[-1]).astype(np.float32)
    row_end = row_begin + len(lg)
    off, rows = blocks["occ_off"].astype(np.int64), blocks["occ_row"].astype(np.int64)
    cnt = np.diff(off)
    # the e-th occurrence of every point at once: each point still receives its adds in ascending row order
    for e in range(int(cnt.max())):
        pts = np.nonzero(cnt > e)[0]
        r = rows[off[pts] + e]
        sel = (r >= row_begin) & (r < row_end)
        acc[pts[sel]] = acc[pts[sel]] + lg[r[sel] - row_begin]
    return acc
