"""Plain numpy restatement of voxel and pillar grouping (pointnet2_b200.pc_util.voxel_group, csrc/voxel.cu, DESIGN.md
§6.19) for the tests and tools/pc_util_bench.py (test infrastructure only), one cloud at a time.

cells_of         each point's cell, or -1: the quotient (p + radius) / voxel in float32, truncated toward zero
oracle_cloud     idx, count and grouped of one cloud
oracle_voxel_group  the same for a padded batch with lengths
"""
from __future__ import annotations

import numpy as np

from crop_oracle import M64, draw

STREAM_CELL = 9


def cells_of(pts: np.ndarray, vsize: int, radius: float, dims: int) -> np.ndarray:
    """(N,) int64 cell of each float32 point, i-major, or -1 for a point whose quotient on some axis is NaN, <= -1 or
    >= vsize.  numpy rounds radius and 2 * radius / vsize to float32 and divides in float32."""
    q = (np.asarray(pts, np.float32)[:, :dims] + np.float32(radius)) / np.float32(2 * radius / float(vsize))
    assert q.dtype == np.float32
    with np.errstate(invalid="ignore"):
        ok = np.all((q > -1) & (q < vsize), axis=1)
    c = np.where(ok[:, None], q, 0).astype(np.int64)
    cell = c[:, 0] * vsize + c[:, 1]
    if dims == 3:
        cell = cell * vsize + c[:, 2]
    return np.where(ok, cell, -1)


def order_keys(rows: np.ndarray, over: np.ndarray, seed: int, entry: np.ndarray) -> np.ndarray:
    """uint64 order key of each member row: the row itself in a cell of at most nsample rows (``over`` False), else
    (draw(seed, 9, entry, row) >> 32) << 32 | row, the device's rng_row_key."""
    rows = rows.astype(np.uint64)
    d = draw(seed, STREAM_CELL, entry.astype(np.uint64), rows) >> np.uint64(32) << np.uint64(32)
    return np.where(over, d | rows, rows)


def oracle_cloud(pts: np.ndarray, vsize: int, radius: float = 1.0, nsample: int = 128, seed: int = 0, dims: int = 3,
                 cloud: int = 0):
    """(idx (C, S) int32, count (C,) int32, grouped (C, S, 3) float64) of one cloud of float32 points, its cells' draw
    entries being cloud * C + cell."""
    pts = np.asarray(pts, np.float32)
    ncell = vsize ** dims
    idx = np.zeros((ncell, nsample), np.int32)
    grouped = np.zeros((ncell, nsample, 3), np.float64)
    cell = cells_of(pts, vsize, radius, dims)
    rows = np.nonzero(cell >= 0)[0]
    cell = cell[rows]
    count = np.bincount(cell, minlength=ncell).astype(np.int32)
    if len(rows) == 0:
        return idx, count, grouped
    over = count[cell] > nsample
    key = order_keys(rows, over, seed & M64, cloud * ncell + cell)
    order = np.lexsort((key, cell))
    rows, cell = rows[order], cell[order]
    start = np.concatenate([[0], np.cumsum(count)])[:-1]
    full = np.nonzero(count)[0]
    m = np.minimum(count[full], nsample)
    src = start[full][:, None] + np.minimum(np.arange(nsample)[None, :], (m - 1)[:, None])
    sel = rows[src]
    idx[full] = sel
    voxel = 2 * radius / float(vsize)
    coord = np.stack([full // vsize, full % vsize], 1) if dims == 2 else \
        np.stack([full // (vsize * vsize), (full // vsize) % vsize, full % vsize], 1)
    centre = (coord + 0.5) * voxel - radius                            # (cells, dims) float64
    p = pts[sel].astype(np.float64)                                    # (cells, S, 3)
    norm = (p[:, :, :dims] - centre[:, None, :]) / voxel
    if dims == 2:
        norm = norm.astype(np.float32).astype(np.float64)
    grouped[full, :, :dims] = norm
    if dims == 2:
        grouped[full, :, 2] = p[:, :, 2]
    return idx, count, grouped


def oracle_voxel_group(xyz: np.ndarray, vsize: int, radius: float = 1.0, nsample: int = 128, seed: int = 0,
                       dims: int = 3, lengths=None):
    """voxel_group's (idx, count, grouped) for a padded (B, N, 3) float32 batch; lengths clamped to [0, N]."""
    xyz = np.asarray(xyz, np.float32)
    b, n, _ = xyz.shape
    out = [oracle_cloud(xyz[i, :n if lengths is None else min(max(int(lengths[i]), 0), n)], vsize, radius, nsample,
                        seed, dims, i) for i in range(b)]
    return tuple(np.stack([o[k] for o in out]) for k in range(3))
