"""The reference's point-cloud / volume conversions (utils/pc_util.py, copied in scannet/pc_util.py) on the GPU, for
padded ragged batches.

The grid cells play the part of centroids: ``voxel_group`` returns, for every cell of a V^3 grid (or an I^2 grid of
xy pillars) over [-radius, radius], up to ``nsample`` member rows as an ``idx`` / ``count`` pair, the layout of
``query_ball_point``, and those rows normalised to the cell.  ``group_point(xyz, idx)``, ``group_and_concat`` and
``sa_mlp_max(idx=...)`` then give voxel- or pillar-level features:

    idx, count, grouped = voxel_group(xyz, 12, nsample=32)          # csrc/voxel.cu
    vol = point_cloud_to_volume_batch(xyz, 12)                       # (B, 1728) float64 occupancy
    vol = point_cloud_to_volume_v2_batch(xyz, 12, num_sample=128)    # (B, 12, 12, 12, 128, 3) float64
    img = point_cloud_to_image_batch(xyz, 32, num_sample=128)        # (B, 32, 32, 128, 3) float64

Bit for bit the reference's arithmetic (DESIGN.md §6.19): a point's cell is computed in float32, as numpy computes
(points + radius) / voxel for float32 points, and truncated toward zero; the normalised coordinates are computed in
float64 (x and y of a pillar rounded once to float32, as the reference's float32 array holds them).  A cell of at most
``nsample`` rows holds them in ascending row order with the last one repeated (np.pad 'edge'); a fuller cell holds
``nsample`` of its rows drawn without replacement by a seeded counter-based draw, where the reference calls the
unseeded np.random.choice.  The one deviation: a point outside the grid (quotient <= -1 or >= V, or NaN) is ignored
by all three conversions, where point_cloud_to_volume raises or wraps a negative index.

The reference's volume_to_point_cloud is ``torch.nonzero(vol == 1)`` on one (V, V, V) volume.
"""
from __future__ import annotations

import numpy as np
import torch

from . import _lib
from ._tensor import (I31, SELECT_MAX_ROWS, as_int as _int, device_lengths0, on_device, ptr, require_cuda, seed_args,
                      stream_ptr)

MAX_NSAMPLE = SELECT_MAX_ROWS  # rows per cell: an over-full cell's draw is sorted in shared memory


def voxel_group(xyz: torch.Tensor, vsize: int, radius: float = 1.0, nsample: int = 128, seed=0, *, dims: int = 3,
                lengths=None):
    """Group the rows of ``xyz`` (B, N, 3) float32 CUDA by the cells of a grid over [-radius, radius]: ``dims`` = 3,
    vsize^3 voxels, cell (i * vsize + j) * vsize + k; ``dims`` = 2, vsize^2 xy pillars, cell i * vsize + j.

    Returns (idx, count, grouped): idx (B, C, nsample) int32, each cell's member rows; count (B, C) int32, the
    number of rows in the cell (it may exceed nsample); grouped (B, C, nsample, 3) float64, the rows normalised to the
    cell, (p - ((c + 0.5) * voxel - radius)) / voxel with voxel = 2 * radius / vsize (pillars: z unchanged).  An empty
    cell is idx 0, grouped 0.  ``seed``: a Python int, or a (1,) int64 CUDA tensor read on the device (rewrite it in
    place to draw again from a captured CUDA graph); it only matters for cells of more than nsample rows.  ``lengths``
    (B,): rows past lengths[b] are never read; a CUDA tensor is clamped to [0, N] on the device.  Nothing is read back
    and the same seed gives the same bits."""
    op = "voxel_group"
    vsize, nsample, dims = _int(vsize, "vsize", op), _int(nsample, "nsample", op), _int(dims, "dims", op)
    if dims not in (2, 3):
        raise ValueError(f"{op} expects dims 2 (pillars) or 3 (voxels), got {dims}")
    if isinstance(radius, bool) or not isinstance(radius, (int, float, np.floating, np.integer)):
        raise TypeError(f"{op} expects a number for radius, got {type(radius).__name__}")
    radius = float(radius)
    if not (0 < radius <= float(np.finfo(np.float32).max) and np.float32(radius) > 0):
        raise ValueError(f"{op} expects a positive radius, finite in float32, got {radius}")
    if not 1 <= nsample <= MAX_NSAMPLE:
        raise ValueError(f"{op} expects 1 <= nsample <= {MAX_NSAMPLE}, got {nsample}")
    if not isinstance(xyz, torch.Tensor):
        raise TypeError(f"{op} expects a torch.Tensor xyz, got {type(xyz).__name__}")
    if xyz.dim() != 3 or xyz.shape[2] != 3:
        raise ValueError(f"{op} expects xyz of shape (B, N, 3), got {tuple(xyz.shape)}")
    b, n, _ = xyz.shape
    if vsize < 1 or vsize ** dims * max(b, 1) >= I31:
        raise ValueError(f"{op} expects vsize >= 1 and B * vsize^{dims} < 2^31, got vsize {vsize} for B {b}")
    if not np.float32(2 * radius / vsize) > 0:
        raise ValueError(f"{op}: the cell edge 2 * {radius} / {vsize} is 0 in float32")
    if b * n >= I31:
        raise ValueError(f"{op} expects B * N < 2^31, got {tuple(xyz.shape)}")
    xyz = require_cuda(xyz, "xyz", torch.float32)
    dev = xyz.device
    seed_val, seed_dev = seed_args(seed, op, dev)
    lens = device_lengths0(lengths, b, n, dev, op)
    cells = vsize ** dims
    idx = torch.empty((b, cells, nsample), dtype=torch.int32, device=dev)
    count = torch.empty((b, cells), dtype=torch.int32, device=dev)
    grouped = torch.empty((b, cells, nsample, 3), dtype=torch.float64, device=dev)
    if b == 0 or n == 0:
        return idx.zero_(), count.zero_(), grouped.zero_()
    lib = _lib.load()
    with on_device(xyz):
        wsb = int(lib.pn2_voxel_group_workspace_bytes(b, n, vsize, dims))
        ws = torch.empty(wsb, dtype=torch.uint8, device=dev)
        rc = lib.pn2_voxel_group(b, n, ptr(xyz), ptr(lens), vsize, dims, radius, nsample, seed_val, ptr(seed_dev),
                                 ptr(count), ptr(idx), ptr(grouped), ptr(ws), wsb, stream_ptr(dev))
    _lib.check(rc, "pn2_voxel_group")
    return idx, count, grouped


def point_cloud_to_volume_batch(xyz: torch.Tensor, vsize: int = 12, radius: float = 1.0, flatten: bool = True, *,
                                lengths=None) -> torch.Tensor:
    """pc_util.point_cloud_to_volume_batch: the (B, vsize^3) float64 occupancy (1.0 where a cell holds a point), or
    (B, vsize, vsize, vsize, 1) when not ``flatten``.  Points outside the grid are ignored."""
    _, count, _ = voxel_group(xyz, vsize, radius, 1, lengths=lengths)
    vol = (count > 0).to(torch.float64)
    return vol if flatten else vol.reshape(vol.shape[0], vsize, vsize, vsize, 1)


def point_cloud_to_volume_v2_batch(xyz: torch.Tensor, vsize: int = 12, radius: float = 1.0, num_sample: int = 128,
                                   seed=0, *, lengths=None) -> torch.Tensor:
    """pc_util.point_cloud_to_volume_v2_batch: (B, vsize, vsize, vsize, num_sample, 3) float64, each voxel's rows
    normalised to it (see voxel_group)."""
    _, _, grouped = voxel_group(xyz, vsize, radius, num_sample, seed, lengths=lengths)
    return grouped.reshape(grouped.shape[0], vsize, vsize, vsize, num_sample, 3)


def point_cloud_to_image_batch(xyz: torch.Tensor, imgsize: int, radius: float = 1.0, num_sample: int = 128, seed=0, *,
                               lengths=None) -> torch.Tensor:
    """pc_util.point_cloud_to_image_batch: (B, imgsize, imgsize, num_sample, 3) float64, each xy pillar's rows with x
    and y normalised to it and z unchanged (see voxel_group)."""
    _, _, grouped = voxel_group(xyz, imgsize, radius, num_sample, seed, dims=2, lengths=lengths)
    return grouped.reshape(grouped.shape[0], imgsize, imgsize, num_sample, 3)
