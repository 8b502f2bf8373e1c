"""Whole-scene semantic segmentation: a scene of any size in, one label per point out.

The reference evaluates a ScanNet scene by cutting it into 1.5 m x 1.5 m xy columns with 0.2 m of context, resampling
every column to 8192 points with replacement and scoring each resampled column on its own
(scannet/scannet_dataset.py:83-118, scannet/train.py:326-427).  Here the columns are a padded ragged batch with per-block
``lengths``, nothing is resampled, and the logits of every block are merged back onto the scene's points in a fixed
order, so every point gets one label and two runs give the same bits:

    blocks = scene_blocks(xyz)                              # csrc/scene.cu: partition on the GPU
    accum, count, label = predict_scene(model, xyz)         # blocks -> model -> ordered merge -> argmax

Block (i, j) spans bmin = (lo_x + i*stride, lo_y + j*stride), bmax = bmin + block_size (lo: the scene's minimum).
Context members lie within ``padding`` of it in x and y, core members within 0.001 (z is not tested); every test is
in double on the float32 coordinates, as numpy evaluates the reference's expressions.  A block without core members is
dropped; a block of c > max_points members becomes k = ceil(c / max_points) sub-blocks, member r (ascending scene index)
going to sub-block r mod k, row r div k.  DESIGN.md §6.9 has the details and the differences from the reference.
"""
from __future__ import annotations

import math
from typing import NamedTuple

import numpy as np
import torch

from . import _lib
from ._tensor import (DTYPE_CODES, FEATURE_DTYPES, I31, SELECT_MAX_ROWS, check_dropout, check_npoints, index_tensors,
                      on_device, on_set_device, pack_offsets, ptr, require_cuda, seed_args, stream_ptr, to_host)

CORE_MARGIN = 0.001   # scannet_dataset.py:103
MAX_BLOCKS = 16384    # blocks in one scene's grid (pn2_api.h)

# train.py:418: per-class weights (classes 1..20) of the calibrated voxel accuracy
CALIBRATION_WEIGHTS = (0.388, 0.357, 0.038, 0.033, 0.017, 0.02, 0.016, 0.025, 0.002, 0.002, 0.002, 0.007, 0.006, 0.022,
                       0.004, 0.0004, 0.003, 0.002, 0.024, 0.029)


class SceneBlocks(NamedTuple):
    """A scene as a padded ragged batch of B (sub-)blocks of N rows, all on the scene's device.

    xyz (B, N, 3) float32, padding rows 0; lengths (B,) int32; point_idx (B, N) int32, the scene index of each row, -1 on
    padding; core (B, N) bool, the rows that are scored; block (B, 3) int32, (i, j, sub-block); occ_off (P + 1,) and
    occ_row int32, the CSR of every point's core rows as flat indices b * N + row, ascending."""
    xyz: torch.Tensor
    lengths: torch.Tensor
    point_idx: torch.Tensor
    core: torch.Tensor
    block: torch.Tensor
    occ_off: torch.Tensor
    occ_row: torch.Tensor


def grid_size(lo: float, hi: float, block_size: float, stride: float) -> int:
    """The smallest k >= 1 with lo + (k - 1) * stride + block_size >= hi, in double."""
    k = max(1, int(math.floor((hi - lo - block_size) / stride)) + 1)
    while k > 1 and lo + (k - 2) * stride + block_size >= hi:
        k -= 1
    while not lo + (k - 1) * stride + block_size >= hi:
        k += 1
    return k


def split_plan(ctx: np.ndarray, core: np.ndarray, max_points: int):
    """Sub-block plan of the blocks with ``ctx`` members and ``core`` core members (numpy int arrays, block order):
    (sub_begin, sub_count, lengths, block) -- each block's first sub-block and number of sub-blocks (0: dropped, it has no
    core member), and per sub-block its length and (i-major block index, sub-block).  Sub-block q of a block of c members
    in k sub-blocks holds the members r = q, q + k, ... : ceil((c - q) / k) rows."""
    ctx = np.asarray(ctx, np.int64)
    k = np.where(np.asarray(core) > 0, -(-ctx // max_points), 0)
    sub_begin = np.concatenate([[0], np.cumsum(k)[:-1]]).astype(np.int64)
    blk = np.repeat(np.arange(len(ctx)), k)
    q = np.arange(int(k.sum())) - np.repeat(sub_begin, k)
    kk, c = np.repeat(k, k), np.repeat(ctx, k)
    lengths = -(-(c - q) // np.maximum(kk, 1))
    return sub_begin, k, lengths, np.stack([blk, q], 1)


def _scene_box(xyz: torch.Tensor):
    """Per-axis minimum and maximum as Python floats: the partition's first read-back.  Non-finite input is rejected
    here (the extrema of a scene with NaN or inf are not finite)."""
    mn, mx = torch.aminmax(xyz, dim=0)
    box = torch.stack([mn, mx]).cpu().numpy().astype(np.float64)
    if not np.isfinite(box).all():
        raise ValueError("scene_blocks expects finite coordinates (the scene holds NaN or inf)")
    return box[0], box[1]


def _check_params(block_size, stride, padding, max_points):
    for name, v in (("block_size", block_size), ("stride", stride), ("padding", padding)):
        if isinstance(v, bool) or not isinstance(v, (int, float)):
            raise TypeError(f"scene_blocks expects a number for {name}, got {type(v).__name__}")
        if not math.isfinite(v):
            raise ValueError(f"scene_blocks expects a finite {name}, got {v}")
    if isinstance(max_points, bool) or not isinstance(max_points, int):
        raise TypeError(f"scene_blocks expects an integer max_points, got {type(max_points).__name__}")
    if not block_size > 0:
        raise ValueError(f"scene_blocks expects a positive block_size, got {block_size}")
    if not 0 < stride <= block_size:
        raise ValueError(f"scene_blocks expects 0 < stride <= block_size (no gaps between blocks), got {stride}")
    if padding < 0:
        raise ValueError(f"scene_blocks expects padding >= 0, got {padding}")
    if max_points < 1:
        raise ValueError(f"scene_blocks expects max_points >= 1, got {max_points}")


def scene_blocks(xyz: torch.Tensor, block_size: float = 1.5, stride=None, padding: float = 0.2,
                 max_points: int = 8192) -> SceneBlocks:
    """Partition the scene ``xyz`` (P, 3) float32 on CUDA into blocks (see the module docstring).  ``stride`` defaults
    to ``block_size``, the reference's tiling.  Reads back two things: the scene's bounding box and the per-block
    counts, which size the batch.  Same bits on every run."""
    if stride is None:
        stride = block_size
    _check_params(block_size, stride, padding, max_points)
    if not isinstance(xyz, torch.Tensor):
        raise TypeError(f"scene_blocks expects a torch.Tensor, got {type(xyz).__name__}")
    if xyz.dim() != 2 or xyz.shape[1] != 3 or xyz.shape[0] < 1:
        raise ValueError(f"scene_blocks expects a (num_points, 3) scene with at least one point, got {tuple(xyz.shape)}")
    xyz = require_cuda(xyz, "xyz", torch.float32)
    p = xyz.shape[0]
    if p + 1 >= I31:
        raise ValueError(f"scene_blocks takes fewer than 2^31 - 1 points, got {p}")
    block_size, stride, padding = float(block_size), float(stride), float(padding)
    dev = xyz.device
    lo, hi = _scene_box(xyz)
    nx, ny = grid_size(lo[0], hi[0], block_size, stride), grid_size(lo[1], hi[1], block_size, stride)
    if nx * ny > MAX_BLOCKS:
        raise ValueError(f"scene_blocks: a grid of {nx} x {ny} blocks exceeds {MAX_BLOCKS}; use a larger stride")
    nblk = nx * ny
    lib = _lib.load()
    geo = (float(lo[0]), float(lo[1]), block_size, stride, padding, nx, ny)
    with on_device(xyz):
        wsb = int(lib.pn2_scene_blocks_workspace_bytes(p, nx, ny))
        ws = torch.empty(wsb, dtype=torch.uint8, device=dev)
        counts = torch.empty(2 * nblk, dtype=torch.int32, device=dev)
        rc = lib.pn2_scene_blocks_count(p, ptr(xyz), *geo, ptr(counts), ptr(ws), wsb, stream_ptr(dev))
        _lib.check(rc, "pn2_scene_blocks_count")
        host = counts.cpu().numpy().astype(np.int64)
        ctx, core = host[:nblk], host[nblk:]
        sub_begin, sub_count, lengths, sub = split_plan(ctx, core, max_points)
        b, n = len(lengths), int(lengths.max())
        if b * n * 3 >= I31 or int(core.sum()) >= I31:
            raise ValueError(f"scene_blocks: a batch of {b} x {n} rows ({int(core.sum())} core rows) passes 2^31 elements")
        tables = torch.from_numpy(np.concatenate([sub_begin, sub_count]).astype(np.int32)).to(dev)
        blk = sub[:, 0]
        block = torch.from_numpy(np.stack([blk // ny, blk % ny, sub[:, 1]], 1).astype(np.int32)).to(dev)
        out = SceneBlocks(
            xyz=torch.empty(b, n, 3, dtype=torch.float32, device=dev),
            lengths=torch.from_numpy(lengths.astype(np.int32)).to(dev),
            point_idx=torch.empty(b, n, dtype=torch.int32, device=dev),
            core=torch.empty(b, n, dtype=torch.bool, device=dev),
            block=block,
            occ_off=torch.empty(p + 1, dtype=torch.int32, device=dev),
            occ_row=torch.empty(int(core.sum()), dtype=torch.int32, device=dev))
        rc = lib.pn2_scene_blocks_fill(p, ptr(xyz), *geo, ptr(tables), ptr(tables[nblk:]), b, n, ptr(out.xyz),
                                       ptr(out.point_idx), ptr(out.core), ptr(out.occ_off), ptr(out.occ_row), ptr(ws), wsb,
                                       stream_ptr(dev))
        _lib.check(rc, "pn2_scene_blocks_fill")
    return out


def merge_block_logits(blocks: SceneBlocks, logits: torch.Tensor, accum: torch.Tensor, row_begin: int = 0) -> torch.Tensor:
    """Add the logits of blocks[row_begin // N : ...] onto ``accum`` (P, C) float32, in place, and return it.

    ``logits`` (Bc, N, C) float32 / bfloat16 / float16 are the model's outputs for the Bc blocks whose rows start at the
    flat row ``row_begin`` (a multiple of N).  For every point, its core rows among them are added one at a time in
    ascending row order, starting from the value already in accum (each add rounded in float32).  Merging chunk by chunk
    therefore gives the bits of one merge over every block.  Asynchronous: nothing is read back."""
    b, n = blocks.point_idx.shape
    p = blocks.occ_off.shape[0] - 1
    if not isinstance(logits, torch.Tensor) or not isinstance(accum, torch.Tensor):
        raise TypeError("merge_block_logits expects torch.Tensor logits and accum")
    if isinstance(row_begin, bool) or not isinstance(row_begin, int):
        raise TypeError(f"merge_block_logits expects an integer row_begin, got {type(row_begin).__name__}")
    if logits.dim() != 3 or logits.shape[1] != n or logits.shape[0] < 1:
        raise ValueError(f"merge_block_logits expects (blocks, {n}, num_class) logits, got {tuple(logits.shape)}")
    c = logits.shape[2]
    if tuple(accum.shape) != (p, c):
        raise ValueError(f"merge_block_logits expects a ({p}, {c}) accum, got {tuple(accum.shape)}")
    if row_begin < 0 or row_begin % n or row_begin // n + logits.shape[0] > b:
        raise ValueError(f"merge_block_logits: row_begin {row_begin} with {logits.shape[0]} blocks of {n} rows is not "
                         f"a range of the {b} blocks")
    if c < 1 or p * c >= I31 or logits.numel() >= I31:
        raise ValueError(f"merge_block_logits: ({p}, {c}) accum or {tuple(logits.shape)} logits pass 2^31 elements")
    logits = require_cuda(logits, "logits", FEATURE_DTYPES)
    if accum.dtype != torch.float32:
        raise TypeError(f"accum must be torch.float32, got {accum.dtype}")
    if not accum.is_cuda:
        raise RuntimeError(f"accum must be a CUDA tensor: pointnet2_b200 has no CPU path (got device {accum.device})")
    if not accum.is_contiguous():
        raise ValueError("merge_block_logits accumulates in place: accum must be contiguous")
    if logits.device != blocks.point_idx.device or accum.device != logits.device:
        raise RuntimeError(f"all tensors must be on the same device ({blocks.point_idx.device}, {logits.device}, {accum.device})")
    lib = _lib.load()
    with on_device(accum):
        rc = lib.pn2_scene_merge_typed(DTYPE_CODES[logits.dtype], p, c, b, n, row_begin, row_begin + logits.shape[0] * n,
                                       ptr(logits), ptr(blocks.point_idx), ptr(blocks.core), ptr(blocks.occ_off),
                                       ptr(blocks.occ_row), ptr(accum), stream_ptr(accum.device))
    _lib.check(rc, "pn2_scene_merge_typed")
    return accum


def predict_scene(model, xyz: torch.Tensor, batch_size: int = 16, **block_kw):
    """Labels for every point of a scene: scene_blocks(xyz, **block_kw), then ``model(xyz_chunk, lengths_chunk)`` on
    ``batch_size`` blocks at a time under torch.no_grad() (in whatever train / eval mode the caller set; the reference
    evaluates with is_training=False), each chunk's logits merged as it comes.

    Returns (accum, count, label): accum (P, C) float32, the sum of each point's core logits in ascending row order;
    count (P,) int32, its number of core occurrences (always >= 1); label (P,) int64, the argmax of accum over the
    classes, the lowest class on ties.  Inside layers.batch_invariant() (an eval-mode model of SharedMLP layers) the
    results do not depend on batch_size: every block's logits have the same bits whatever blocks share its batch."""
    if isinstance(batch_size, bool) or not isinstance(batch_size, int) or batch_size < 1:
        raise ValueError(f"predict_scene expects a positive integer batch_size, got {batch_size!r}")
    blocks = scene_blocks(xyz, **block_kw)
    b, n = blocks.point_idx.shape
    accum = None
    with torch.no_grad():
        for b0 in range(0, b, batch_size):
            b1 = min(b, b0 + batch_size)
            out = model(blocks.xyz[b0:b1], blocks.lengths[b0:b1])
            logits = out[0] if isinstance(out, (tuple, list)) else out
            if accum is None:
                accum = torch.zeros(blocks.occ_off.shape[0] - 1, logits.shape[-1], dtype=torch.float32, device=xyz.device)
            merge_block_logits(blocks, logits, accum, row_begin=b0 * n)
    count = blocks.occ_off[1:] - blocks.occ_off[:-1]
    return accum, count, accum.argmax(dim=1)


# ---- whole-scene voxel metrics (scannet/pc_util.py:39-51, scannet/train.py:391-420) -------------------------------
def surface_voxel_labels(xyz: torch.Tensor, label: torch.Tensor, res: float = 0.0484):
    """pc_util.point_cloud_label_to_surface_voxel_label_fast in torch, on the tensors' device.

    Voxel keys are computed in float32, as numpy computes them for float32 input: ceil((p - min) / res) per axis and
    x + y * nvox0 + z * nvox0 * nvox1, so keys above 2^24 can round together and a coordinate on the maximum (index ==
    nvox) aliases the next row, exactly as in the reference.  Each voxel takes the label (row) of its first point by
    index.  Returns (keys, labels, nvox): the distinct keys ascending, their labels ((V,) or (V, K) for (P, K) labels)
    and nvox (3,) float32."""
    if xyz.dim() != 2 or xyz.shape[1] != 3 or xyz.dtype != torch.float32:
        raise ValueError(f"surface_voxel_labels expects (num_points, 3) float32 coordinates, got {xyz.dtype} {tuple(xyz.shape)}")
    if label.shape[0] != xyz.shape[0] or label.dim() not in (1, 2):
        raise ValueError(f"surface_voxel_labels expects ({xyz.shape[0]},) or ({xyz.shape[0]}, K) labels, got {tuple(label.shape)}")
    # a float32 tensor divisor: CUDA divides a tensor by a host scalar as a multiply by its reciprocal, numpy does not
    r = torch.full((), res, dtype=torch.float32, device=xyz.device)
    mn, mx = torch.aminmax(xyz, dim=0)
    nvox = torch.ceil((mx - mn) / r)
    v = torch.ceil((xyz - mn) / r)
    key = v[:, 0] + v[:, 1] * nvox[0] + v[:, 2] * nvox[0] * nvox[1]
    keys, inv = torch.unique(key, sorted=True, return_inverse=True)
    first = torch.full((keys.shape[0],), xyz.shape[0], dtype=torch.int64, device=xyz.device)
    first.scatter_reduce_(0, inv, torch.arange(xyz.shape[0], device=xyz.device), reduce="amin")
    return keys, label[first], nvox


class VoxelAccuracy:
    """The whole-scene accumulation of train.py:391-420 over surface voxels (res 0.02), applied to whole scenes with
    their merged labels (the reference applies it per resampled block, to duplicated points): voxel accuracy over
    label > 0, per-class voxel accuracy and the calibrated accuracy with CALIBRATION_WEIGHTS.  Counts stay on the
    device until a result is asked for."""

    def __init__(self, num_class: int = 21, res: float = 0.02, device=None):
        self.num_class, self.res = num_class, res
        self.seen_class = torch.zeros(num_class, dtype=torch.int64, device=device)
        self.correct_class = torch.zeros(num_class, dtype=torch.int64, device=device)

    def update(self, xyz: torch.Tensor, label: torch.Tensor, pred: torch.Tensor) -> None:
        """One scene: xyz (P, 3) float32, label and pred (P,) integer classes."""
        _, uv, _ = surface_voxel_labels(xyz, torch.stack([label.long(), pred.long()], 1), self.res)
        t, pr = uv[:, 0], uv[:, 1]
        nc = self.num_class
        self.seen_class += torch.bincount(t.clamp(0, nc - 1), minlength=nc)[:nc].to(self.seen_class.device)
        self.correct_class += torch.bincount(t[t == pr].clamp(0, nc - 1), minlength=nc)[:nc].to(self.seen_class.device)

    def results(self) -> dict:
        """accuracy (label > 0), mean class accuracy and calibrated accuracy over classes 1.., as train.py:412-419."""
        seen = self.seen_class.cpu().numpy().astype(np.float64)
        correct = self.correct_class.cpu().numpy().astype(np.float64)
        per_class = correct[1:] / (seen[1:] + 1e-6)
        w = np.asarray(CALIBRATION_WEIGHTS[:len(per_class)], np.float64)
        return {"accuracy": float(correct[1:].sum() / max(seen[1:].sum(), 1.0)),
                "class_accuracy": float(per_class.mean()),
                "calibrated_accuracy": float(np.average(per_class, weights=w)),
                "per_class": per_class}


# ---- training crops (scannet/scannet_dataset.py:27-60, scannet/train.py:181-197, utils/provider.py:52-70) ----------
CROP_MAX_POINTS = SELECT_MAX_ROWS  # npoints cap of sample_crops and sample_virtual_scans: the shared-memory row sort
CROP_MAX_BATCH = 65535    # crops per call


class SceneSet:
    """S scenes packed into one set on the device, the training side's counterpart of a list of scene arrays.

    xyz (P, 3) float32, label (P,) int32, offsets (S + 1,) int64 (scene k holds rows offsets[k] .. offsets[k + 1] - 1),
    lo / hi (S, 3) float32, each scene's per-axis minimum and maximum as np.min / np.max give them, mean (S, 3) float64,
    each scene's np.mean(x.astype(np.float64), axis=0) (the virtual scans' room centre).  ``sizes`` (numpy
    int64) and ``label_hist`` (numpy int64, (num_class,)) stay on the host.  Construction validates everything on the
    host and is the only place anything is read back.  ``device`` defaults to the current CUDA device; sample_crops
    needs one."""

    def __init__(self, xyz_list, label_list, num_class: int = 21, device=None):
        if isinstance(num_class, bool) or not isinstance(num_class, int) or num_class < 1:
            raise ValueError(f"SceneSet expects a positive integer num_class, got {num_class!r}")
        xyz_list, label_list = list(xyz_list), list(label_list)
        if not xyz_list:
            raise ValueError("SceneSet expects at least one scene")
        if len(xyz_list) != len(label_list):
            raise ValueError(f"SceneSet expects one label array per scene, got {len(xyz_list)} scenes and "
                             f"{len(label_list)} label arrays")
        xyz_list, label_list = [to_host(x) for x in xyz_list], [to_host(lab) for lab in label_list]
        for k, (x, lab) in enumerate(zip(xyz_list, label_list)):
            if x.ndim != 2 or x.shape[1] != 3:
                raise ValueError(f"SceneSet: scene {k} must be (num_points, 3), got {x.shape}")
            if len(x) == 0:
                raise ValueError(f"SceneSet: scene {k} is empty")
            if lab.shape != (len(x),):
                raise ValueError(f"SceneSet: scene {k} has {len(x)} points but labels of shape {lab.shape}")
            if not np.issubdtype(lab.dtype, np.integer):
                raise TypeError(f"SceneSet: scene {k} has {lab.dtype} labels, expected integers")
        self.sizes, self.offsets = pack_offsets(xyz_list, "SceneSet", device)
        pts, labs, lo, hi, mean = [], [], [], [], []
        hist = np.zeros(num_class, np.int64)
        for k, (x, lab) in enumerate(zip(xyz_list, label_list)):
            x = x.astype(np.float32)
            if not np.isfinite(x).all():
                raise ValueError(f"SceneSet: scene {k} holds NaN or inf coordinates")
            if np.abs(x).max() > 1e9:  # DESIGN.md §6.10: keeps the crop box's double arithmetic away from its collapse
                raise ValueError(f"SceneSet: scene {k} has coordinates beyond 1e9 in magnitude (sample_crops' limit)")
            mn, mx = np.min(x, axis=0), np.max(x, axis=0)
            if not mx[2] > mn[2]:
                raise ValueError(f"SceneSet: scene {k} has zero z extent (the voxel test divides by it)")
            if lab.min() < 0 or lab.max() >= num_class:
                raise ValueError(f"SceneSet: scene {k} has labels outside [0, {num_class})")
            hist += np.bincount(lab.astype(np.int64), minlength=num_class)
            pts.append(x)
            labs.append(lab.astype(np.int32))
            lo.append(mn)
            hi.append(mx)
            mean.append(np.mean(x.astype(np.float64), axis=0))
        self.device = dev = self.offsets.device  # "cuda" resolved to the current index: compared against by the samplers
        self.num_class = num_class
        self.label_hist = hist
        self.xyz = torch.from_numpy(np.concatenate(pts)).to(dev)
        self.label = torch.from_numpy(np.concatenate(labs)).to(dev)
        self.lo = torch.from_numpy(np.stack(lo)).to(dev)
        self.hi = torch.from_numpy(np.stack(hi)).to(dev)
        self.mean = torch.from_numpy(np.stack(mean)).to(dev)

    def __len__(self) -> int:
        return len(self.sizes)

    def train_label_weights(self) -> torch.Tensor:
        """scannet_dataset.py:17-24 over the set's labels: 1 / log(1.2 + freq), with the reference's dtypes (float64
        counts, then float32 throughout), as a (num_class,) float32 tensor on the set's device.  The test split uses
        torch.ones(num_class) instead (:25-26)."""
        w = self.label_hist.astype(np.float64).astype(np.float32)
        w = w / np.sum(w)
        w = 1 / np.log(1.2 + w)
        return torch.from_numpy(np.asarray(w, np.float32)).to(self.device)


class SceneCrops(NamedTuple):
    """B training crops as a padded ragged batch of ``npoints`` rows, every field on the scene set's device.

    xyz (B, npoints, 3) float32; label (B, npoints) int64; weight (B, npoints) float32, label_weights[label] on core
    rows; lengths (B,) int32, >= 1 for every crop whose crop_scene value is in [0, S) and 0 for one outside it (the
    only way a bad index can show without a read-back); point_idx (B, npoints) int32, the row of the scene set, -1 on padding; core
    (B, npoints) bool; attempt (B,) int32, the attempt taken; valid (B,) bool, whether it passed the test.  Padding
    rows are 0 (-1 in point_idx)."""
    xyz: torch.Tensor
    label: torch.Tensor
    weight: torch.Tensor
    lengths: torch.Tensor
    point_idx: torch.Tensor
    core: torch.Tensor
    attempt: torch.Tensor
    valid: torch.Tensor


def _label_weights(label_weights, scenes: SceneSet, what: str) -> torch.Tensor:
    label_weights = require_cuda(label_weights, "label_weights", torch.float32)
    if tuple(label_weights.shape) != (scenes.num_class,):
        raise ValueError(f"{what} expects ({scenes.num_class},) label_weights, got {tuple(label_weights.shape)}")
    on_set_device(label_weights, "label_weights", scenes.device)
    return label_weights


def sample_crops(scenes: SceneSet, crop_scene: torch.Tensor, seed, label_weights: torch.Tensor, npoints: int = 8192,
                 max_dropout: float = 0.875, rotate: bool = True) -> SceneCrops:
    """B random training crops of ``scenes`` on the GPU (DESIGN.md §6.10): crop i is a 1.5 m column of scene
    crop_scene[i] with 0.2 m of context, taken from ten seeded attempts as ScannetDataset.__getitem__ takes it; its
    rows are up to ``npoints`` of the column's points in a seeded random order, without replacement; rows after the
    first are dropped with probability U[0, 1) * max_dropout (get_batch_wdp; max_dropout=0 is get_batch); x and y are
    rotated about the origin by a U[0, 2 pi) angle when ``rotate`` (rotate_point_cloud_z).

    ``crop_scene`` (B,) integer CUDA tensor: the scene of each crop.  ``seed``: a Python int, or a (1,) int64 CUDA tensor
    read on the device (rewrite it in place to draw new crops from a captured CUDA graph).  Give every step and rank its
    own seed.  ``label_weights`` (num_class,) float32 CUDA tensor, e.g. scenes.train_label_weights().  Nothing is read
    back and the same seed gives the same bits.  A crop_scene value outside [0, S) gives an empty crop (lengths 0,
    attempt -1): it cannot be reported without a read-back."""
    what = "sample_crops"
    if not isinstance(scenes, SceneSet):
        raise TypeError(f"{what} expects a SceneSet, got {type(scenes).__name__}")
    check_npoints(npoints, what)
    check_dropout(max_dropout, what)
    if not isinstance(rotate, bool):
        raise TypeError(f"{what} expects a bool rotate, got {type(rotate).__name__}")
    dev = scenes.device
    if dev.type != "cuda":
        raise RuntimeError(f"{what} needs a SceneSet on a CUDA device: pointnet2_b200 has no CPU path (got {dev})")
    crop_scene, = index_tensors(what, dev, CROP_MAX_BATCH, crop_scene=crop_scene)
    b = crop_scene.shape[0]
    if b * npoints * 3 >= I31:
        raise ValueError(f"{what}: {b} crops of {npoints} rows pass 2^31 elements")
    seed_val, seed_dev = seed_args(seed, what, dev)
    label_weights = _label_weights(label_weights, scenes, what)
    lib = _lib.load()
    with on_device(scenes.xyz):
        wsb = int(lib.pn2_scene_crops_workspace_bytes(b, npoints))
        ws = torch.empty(wsb, dtype=torch.uint8, device=dev)
        out = SceneCrops(
            xyz=torch.empty(b, npoints, 3, dtype=torch.float32, device=dev),
            label=torch.empty(b, npoints, dtype=torch.int64, device=dev),
            weight=torch.empty(b, npoints, dtype=torch.float32, device=dev),
            lengths=torch.empty(b, dtype=torch.int32, device=dev),
            point_idx=torch.empty(b, npoints, dtype=torch.int32, device=dev),
            core=torch.empty(b, npoints, dtype=torch.bool, device=dev),
            attempt=torch.empty(b, dtype=torch.int32, device=dev),
            valid=torch.empty(b, dtype=torch.bool, device=dev))
        rc = lib.pn2_scene_crops(len(scenes), int(scenes.sizes.sum()), int(scenes.sizes.max()), ptr(scenes.xyz),
                                 ptr(scenes.label), ptr(scenes.offsets), ptr(scenes.lo), ptr(scenes.hi), scenes.num_class,
                                 ptr(label_weights), b, ptr(crop_scene), seed_val, ptr(seed_dev), npoints,
                                 float(max_dropout), int(rotate), ptr(out.xyz), ptr(out.label), ptr(out.weight),
                                 ptr(out.lengths), ptr(out.point_idx), ptr(out.core), ptr(out.attempt), ptr(out.valid),
                                 ptr(ws), wsb, stream_ptr(dev))
    _lib.check(rc, "pn2_scene_crops")
    return out


# ---- virtual scans (scannet/scene_util.py virtual_scan, scannet/scannet_dataset.py:122-166) ------------------------
SCAN_MAX_BATCH = 4096     # entries per call of sample_virtual_scans: its workspace is about 1.7 MB per entry
SCAN_VIEWS = 8            # the dataset's fixed views: azimuth pi/4 m for m = 0..7


class SceneScans(NamedTuple):
    """B virtual scans as a padded ragged batch of ``npoints`` rows, every field on the scene set's device.

    xyz (B, npoints, 3) float32, the scene's own coordinates (not centred or rotated); label (B, npoints) int64; weight
    (B, npoints) float32, label_weights[label], 0 on every row of an invalid entry; lengths (B,) int32, min(visible,
    npoints); point_idx (B, npoints) int32, the row of the scene set, -1 on padding; visible (B,) int32, the number of
    points the scan sees (0 when fewer than 100 points are near a ray, -1 for a scan_scene value outside [0, S), the only
    way a bad index can show without a read-back); valid (B,) bool, visible >= min_points.  Padding rows are 0 (-1 in
    point_idx)."""
    xyz: torch.Tensor
    label: torch.Tensor
    weight: torch.Tensor
    lengths: torch.Tensor
    point_idx: torch.Tensor
    visible: torch.Tensor
    valid: torch.Tensor


def sample_virtual_scans(scenes: SceneSet, scan_scene: torch.Tensor, scan_mode: torch.Tensor, seed,
                         label_weights: torch.Tensor, npoints: int = 8192, min_points: int = 300) -> SceneScans:
    """B virtual scans of ``scenes`` on the GPU (DESIGN.md §6.12): entry i is what a camera 1.5 m high, behind the
    centre of scene scan_scene[i], sees through a 200 x 150 grid of rays, as scene_util.virtual_scan computes it; its
    rows are up to ``npoints`` of the visible points in a seeded random order, without replacement.

    ``scan_scene`` (B,) integer CUDA tensor: the scene of each entry.  ``scan_mode`` (B,) integer CUDA tensor: -1 draws
    a random view from the seed (virtual_scan(mode=-1)); any other m is the fixed view at azimuth pi/4 m (the dataset
    uses m = 0..7).  ``seed``: a Python int, or a (1,) int64 CUDA tensor read on the device (rewrite it in place to draw
    new scans from a captured CUDA graph).  ``label_weights`` (num_class,) float32 CUDA tensor:
    scenes.train_label_weights() for the train split, torch.ones(num_class) for the test split.  An entry with fewer
    than ``min_points`` visible points stays in the batch, flagged invalid with weight 0 (the reference drops it).
    Nothing is read back and the same seed gives the same bits."""
    what = "sample_virtual_scans"
    if not isinstance(scenes, SceneSet):
        raise TypeError(f"{what} expects a SceneSet, got {type(scenes).__name__}")
    check_npoints(npoints, what)
    if isinstance(min_points, bool) or not isinstance(min_points, int):
        raise TypeError(f"{what} expects an integer min_points, got {type(min_points).__name__}")
    if not 0 <= min_points < I31:
        raise ValueError(f"{what} expects 0 <= min_points < 2^31, got {min_points}")
    dev = scenes.device
    if dev.type != "cuda":
        raise RuntimeError(f"{what} needs a SceneSet on a CUDA device: pointnet2_b200 has no CPU path (got {dev})")
    scan_scene, scan_mode = index_tensors(what, dev, SCAN_MAX_BATCH, scan_scene=scan_scene, scan_mode=scan_mode)
    b = scan_scene.shape[0]
    if b * npoints * 3 >= I31:
        raise ValueError(f"{what}: {b} scans of {npoints} rows pass 2^31 elements")
    seed_val, seed_dev = seed_args(seed, what, dev)
    label_weights = _label_weights(label_weights, scenes, what)
    lib = _lib.load()
    max_scene = int(scenes.sizes.max())
    with on_device(scenes.xyz):
        wsb = int(lib.pn2_virtual_scans_workspace_bytes(b, max_scene, npoints))
        ws = torch.empty(wsb, dtype=torch.uint8, device=dev)
        out = SceneScans(
            xyz=torch.empty(b, npoints, 3, dtype=torch.float32, device=dev),
            label=torch.empty(b, npoints, dtype=torch.int64, device=dev),
            weight=torch.empty(b, npoints, dtype=torch.float32, device=dev),
            lengths=torch.empty(b, dtype=torch.int32, device=dev),
            point_idx=torch.empty(b, npoints, dtype=torch.int32, device=dev),
            visible=torch.empty(b, dtype=torch.int32, device=dev),
            valid=torch.empty(b, dtype=torch.bool, device=dev))
        rc = lib.pn2_virtual_scans(len(scenes), int(scenes.sizes.sum()), max_scene, ptr(scenes.xyz), ptr(scenes.label),
                                   ptr(scenes.offsets), ptr(scenes.mean), scenes.num_class, ptr(label_weights), b,
                                   ptr(scan_scene), ptr(scan_mode), seed_val, ptr(seed_dev), npoints, min_points,
                                   ptr(out.xyz), ptr(out.label), ptr(out.weight), ptr(out.lengths), ptr(out.point_idx),
                                   ptr(out.visible), ptr(out.valid), ptr(ws), wsb, stream_ptr(dev))
    _lib.check(rc, "pn2_virtual_scans")
    return out
