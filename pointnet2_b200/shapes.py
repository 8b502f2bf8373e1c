"""Shape batches on the GPU: ModelNet classification and ShapeNet part training batches from a packed shape set, and
rotation-vote classification (DESIGN.md §6.11).

The reference builds every training batch on the host: ModelNet's loaders take each shape's first npoints rows, apply
the five augmentation steps of utils/provider.py and shuffle the rows (modelnet_dataset.py:60-84,
modelnet_h5_dataset.py:72-114); the part loader resamples npoints rows with replacement and train.py jitters them
(part_seg/part_dataset_all_normal.py:83-112, part_seg/train.py:200); evaluate.py:117-158 scores each test shape over V
rotated votes.  Here one kernel draws the whole batch from a device-resident ShapeSet, seeded and without a read-back,
as a padded ragged batch with per-entry ``lengths``:

    shapes = ShapeSet(xyz_list, label_list)                      # once: validation, pc_normalize, packing
    batch = sample_shapes(shapes, shape_idx, seed)               # ModelNet's _augment_batch_data
    batch = sample_shapes(shapes, shape_idx, seed, subset="random", rotate=False, perturb=False, scale=None,
                          shift=0, with_normals=True)            # the ShapeNet part recipe
    logits = classify_votes(model, shapes, shape_idx, 12, seed)  # evaluate.py's votes, summed in vote order
"""
from __future__ import annotations

import math
from typing import NamedTuple, Optional

import numpy as np
import torch

from . import _lib
from ._tensor import (I31, SELECT_MAX_ROWS, check_dropout, check_npoints, index_tensors, on_device, pack_offsets, ptr,
                      seed_args, stream_ptr, to_host)

MAX_POINTS = SELECT_MAX_ROWS  # points per shape and npoints: the kernel's (key, row) sort is in shared memory


def pc_normalize(pc: np.ndarray) -> np.ndarray:
    """modelnet_dataset.py:15-21 on a (P, 3) array, in its dtype: centre on the mean, divide by the largest norm."""
    centroid = np.mean(pc, axis=0)
    pc = pc - centroid
    m = np.max(np.sqrt(np.sum(pc ** 2, axis=1)))
    return pc / m


class ShapeSet:
    """S shapes packed into one set on the device.

    xyz (P, 3) float32; normals (P, 3) float32 or None; label (S,) int32, each shape's class; part (P,) int32 or None,
    per-point part labels; offsets (S + 1,) int64 (shape k holds rows offsets[k] .. offsets[k + 1] - 1).  ``sizes``
    (numpy int64) stays on the host.  ``normalize`` applies pc_normalize to each whole shape's xyz in float32 once, as
    the loaders cache it.  Construction validates everything on the host and is the only place anything is read back.
    ``device`` defaults to the current CUDA device; sample_shapes needs one."""

    def __init__(self, xyz_list, label_list, normal_list=None, part_list=None, num_class: int = 40,
                 normalize: bool = True, device=None):
        if isinstance(num_class, bool) or not isinstance(num_class, int) or num_class < 1:
            raise ValueError(f"ShapeSet expects a positive integer num_class, got {num_class!r}")
        xyz_list, label_list = list(xyz_list), list(label_list)
        if not xyz_list:
            raise ValueError("ShapeSet expects at least one shape")
        if len(label_list) != len(xyz_list):
            raise ValueError(f"ShapeSet expects one label per shape, got {len(xyz_list)} shapes and {len(label_list)} labels")
        for name, lst in (("normal", normal_list), ("part", part_list)):
            if lst is not None and len(list(lst)) != len(xyz_list):
                raise ValueError(f"ShapeSet expects one {name} array per shape, got {len(list(lst))} for {len(xyz_list)} shapes")
        xyz_list = [to_host(x) for x in xyz_list]
        normal_list = None if normal_list is None else [to_host(n) for n in normal_list]
        part_list = None if part_list is None else [to_host(p) for p in part_list]
        for k, x in enumerate(xyz_list):
            if x.ndim != 2 or x.shape[1] != 3:
                raise ValueError(f"ShapeSet: shape {k} must be (num_points, 3), got {x.shape}")
            if not 1 <= len(x) <= MAX_POINTS:
                raise ValueError(f"ShapeSet: shape {k} has {len(x)} points; a shape has 1 to {MAX_POINTS}")
        self.sizes, self.offsets = pack_offsets(xyz_list, "ShapeSet", device)
        labels = []
        for k, lab in enumerate(label_list):
            lab = to_host(lab)
            if lab.size != 1 or not np.issubdtype(lab.dtype, np.integer):
                raise TypeError(f"ShapeSet: shape {k} has label {lab!r}; expected one integer")
            lab = int(lab.reshape(()))
            if not 0 <= lab < num_class:
                raise ValueError(f"ShapeSet: shape {k} has label {lab} outside [0, {num_class})")
            labels.append(lab)
        pts, nrms, parts = [], [], []
        for k, x in enumerate(xyz_list):
            x = x.astype(np.float32)
            if not np.isfinite(x).all():
                raise ValueError(f"ShapeSet: shape {k} holds NaN or inf coordinates")
            if normalize:
                with np.errstate(invalid="ignore", divide="ignore"):
                    x = pc_normalize(x)
                if not np.isfinite(x).all():
                    raise ValueError(f"ShapeSet: shape {k} has all its points equal: normalize divides by its radius 0")
            pts.append(x)
            if normal_list is not None:
                n = normal_list[k]
                if n.shape != x.shape:
                    raise ValueError(f"ShapeSet: shape {k} has {len(x)} points but normals of shape {n.shape}")
                n = n.astype(np.float32)
                if not np.isfinite(n).all():
                    raise ValueError(f"ShapeSet: shape {k} holds NaN or inf normals")
                nrms.append(n)
            if part_list is not None:
                p = part_list[k]
                if p.shape != (len(x),):
                    raise ValueError(f"ShapeSet: shape {k} has {len(x)} points but part labels of shape {p.shape}")
                if not np.issubdtype(p.dtype, np.integer):
                    raise TypeError(f"ShapeSet: shape {k} has {p.dtype} part labels, expected integers")
                if p.min() < 0 or p.max() >= I31:
                    raise ValueError(f"ShapeSet: shape {k} has part labels outside [0, 2^31)")
                parts.append(p.astype(np.int32))
        self.device = dev = self.offsets.device  # "cuda" resolved to the current index: compared against by the samplers
        self.num_class = num_class
        self.xyz = torch.from_numpy(np.concatenate(pts)).to(dev)
        self.normals = torch.from_numpy(np.concatenate(nrms)).to(dev) if normal_list is not None else None
        self.part = torch.from_numpy(np.concatenate(parts)).to(dev) if part_list is not None else None
        self.label = torch.tensor(labels, dtype=torch.int32).to(dev)

    def __len__(self) -> int:
        return len(self.sizes)


class ShapeBatch(NamedTuple):
    """E entries as a padded ragged batch of ``npoints`` rows, every field on the shape set's device.

    points (E, npoints, 3) float32, or (E, npoints, 6) with the normals after the coordinates; label (E,) int64, the
    shape's class; part (E, npoints) int64, or None when the set has no part labels; lengths (E,) int32, 0 for an entry
    whose shape index is outside [0, S); point_idx (E, npoints) int32, the row of the set, -1 on padding.  Padding rows
    are 0."""
    points: torch.Tensor
    label: torch.Tensor
    part: Optional[torch.Tensor]
    lengths: torch.Tensor
    point_idx: torch.Tensor


def _number(v, name, op):
    if isinstance(v, bool) or not isinstance(v, (int, float, np.integer, np.floating)):
        raise TypeError(f"{op} expects a number for {name}, got {type(v).__name__}")
    v = float(v)
    if not math.isfinite(v):
        raise ValueError(f"{op} expects a finite {name}, got {v}")
    return v


def _pair(v, name, op):
    if v is None:
        return None
    if not isinstance(v, (tuple, list)) or len(v) != 2:
        raise TypeError(f"{op} expects None or a pair of numbers for {name}, got {v!r}")
    return _number(v[0], name, op), _number(v[1], name, op)


def _check_call(shapes, shape_idx, npoints, with_normals, op):
    """shape_idx as the kernel reads it, once the arguments every shape batch takes are checked."""
    if not isinstance(shapes, ShapeSet):
        raise TypeError(f"{op} expects a ShapeSet, got {type(shapes).__name__}")
    check_npoints(npoints, op)
    if not isinstance(with_normals, bool):
        raise TypeError(f"{op} expects a bool with_normals, got {type(with_normals).__name__}")
    if with_normals and shapes.normals is None:
        raise ValueError(f"{op}: with_normals=True needs a ShapeSet built with normals")
    dev = shapes.device
    if dev.type != "cuda":
        raise RuntimeError(f"{op} needs a ShapeSet on a CUDA device: pointnet2_b200 has no CPU path (got {dev})")
    return index_tensors(op, dev, shape_idx=shape_idx)[0]


def _launch(shapes, shape_idx, seed_val, seed_dev, votes, npoints, subset_random, rotate, perturb, scale, shift, jitter,
            max_dropout, with_normals) -> ShapeBatch:
    dev = shapes.device
    b = shape_idx.shape[0]
    e = b * votes if votes else b
    ch = 6 if with_normals else 3
    if e * npoints * ch >= I31:
        raise ValueError(f"{e} entries of {npoints} rows x {ch} channels pass 2^31 elements")
    lib = _lib.load()
    with on_device(shapes.xyz):
        out = ShapeBatch(
            points=torch.empty(e, npoints, ch, dtype=torch.float32, device=dev),
            label=torch.empty(e, dtype=torch.int64, device=dev),
            part=torch.empty(e, npoints, dtype=torch.int64, device=dev) if shapes.part is not None else None,
            lengths=torch.empty(e, dtype=torch.int32, device=dev),
            point_idx=torch.empty(e, npoints, dtype=torch.int32, device=dev))
        sc = scale if scale is not None else (1.0, 1.0)
        jt = jitter if jitter is not None else (0.0, 1.0)
        rc = lib.pn2_shape_batch(len(shapes), int(shapes.sizes.sum()), int(shapes.sizes.max()), ptr(shapes.xyz),
                                 ptr(shapes.normals), ptr(shapes.label), ptr(shapes.part), ptr(shapes.offsets), b,
                                 ptr(shape_idx), seed_val, ptr(seed_dev), votes, npoints, int(subset_random), int(rotate),
                                 int(perturb), int(scale is not None), sc[0], sc[1], float(shift), int(jitter is not None),
                                 jt[0], jt[1], float(max_dropout), int(with_normals), ptr(out.points), ptr(out.label),
                                 ptr(out.part), ptr(out.lengths), ptr(out.point_idx), stream_ptr(dev))
    _lib.check(rc, "pn2_shape_batch")
    return out


def sample_shapes(shapes: ShapeSet, shape_idx: torch.Tensor, seed, npoints: int = 1024, subset: str = "first",
                  rotate: bool = True, perturb: bool = True, scale=(0.8, 1.25), shift: float = 0.1,
                  jitter=(0.01, 0.05), max_dropout: float = 0.0, with_normals: bool = False) -> ShapeBatch:
    """B training entries of ``shapes`` on the GPU (DESIGN.md §6.11), entry i from shape shape_idx[i].

    Rows: ``subset="first"`` takes the shape's first npoints rows in a seeded order (the ModelNet loaders' truncation
    and shuffle_points); ``"random"`` takes min(P, npoints) of all P rows without replacement, in a seeded order (the
    part loader, without its resampling).  Rows after the first are removed with probability U[0, 1) * max_dropout
    (random_point_dropout; 0 turns it off).  Then, in float64 rounded once to float32: a U[0, 2 pi) rotation about y
    (``rotate``), a small random rotation (``perturb``, angles clip(0.06 N(0, 1), +-0.18)), a per-entry scale drawn
    from U[scale) (None: off), a per-entry shift from U[-shift, shift) per axis (0: off) and a per-point jitter
    clip(sigma N(0, 1), +-clip) for jitter=(sigma, clip) (None: off).  Normals get the two rotations only.  The defaults
    are ModelNet's _augment_batch_data.

    ``shape_idx`` (B,) integer CUDA tensor.  ``seed``: a Python int, or a (1,) int64 CUDA tensor read on the device
    (rewrite it in place to draw new batches from a captured CUDA graph).  Give every step and rank its own seed.
    Nothing is read back and the same seed gives the same bits.  A shape_idx value outside [0, S) gives an empty entry
    (lengths 0): it cannot be reported without a read-back."""
    op = "sample_shapes"
    if subset not in ("first", "random"):
        raise ValueError(f"{op} expects subset 'first' or 'random', got {subset!r}")
    for name, v in (("rotate", rotate), ("perturb", perturb)):
        if not isinstance(v, bool):
            raise TypeError(f"{op} expects a bool {name}, got {type(v).__name__}")
    scale, jitter = _pair(scale, "scale", op), _pair(jitter, "jitter", op)
    if scale is not None and not scale[0] <= scale[1]:
        raise ValueError(f"{op} expects scale=(low, high) with low <= high, got {scale}")
    if jitter is not None and not (jitter[0] >= 0 and jitter[1] > 0):
        raise ValueError(f"{op} expects jitter=(sigma, clip) with sigma >= 0 and clip > 0, got {jitter}")
    shift = _number(shift, "shift", op)
    if shift < 0:
        raise ValueError(f"{op} expects shift >= 0, got {shift}")
    check_dropout(max_dropout, op)
    shape_idx = _check_call(shapes, shape_idx, npoints, with_normals, op)
    seed_val, seed_dev = seed_args(seed, op, shapes.device)
    return _launch(shapes, shape_idx, seed_val, seed_dev, 0, npoints, subset == "random", rotate, perturb, scale, shift,
                   jitter, max_dropout, with_normals)


def vote_batch(shapes: ShapeSet, shape_idx: torch.Tensor, num_votes: int, seed, npoints: int = 1024,
               with_normals: bool = False) -> ShapeBatch:
    """The V = num_votes votes of evaluate.py:126-135 for the B shapes of ``shape_idx``, vote-major: entry v * B + i is
    shape shape_idx[i]'s first npoints rows in a seeded order, rotated about y by v / V of a turn; nothing else is
    applied.  ``seed`` as for sample_shapes (it orders the rows)."""
    op = "vote_batch"
    if isinstance(num_votes, bool) or not isinstance(num_votes, int) or num_votes < 1:
        raise ValueError(f"{op} expects a positive integer num_votes, got {num_votes!r}")
    shape_idx = _check_call(shapes, shape_idx, npoints, with_normals, op)
    if shape_idx.shape[0] * num_votes >= I31:
        raise ValueError(f"{op}: {shape_idx.shape[0]} shapes x {num_votes} votes pass 2^31 entries")
    seed_val, seed_dev = seed_args(seed, op, shapes.device)
    return _launch(shapes, shape_idx, seed_val, seed_dev, num_votes, npoints, False, False, False, None, 0.0, None, 0.0,
                   with_normals)


def classify_votes(model, shapes: ShapeSet, shape_idx: torch.Tensor, num_votes: int, seed, npoints: int = 1024,
                   chunk: Optional[int] = None) -> torch.Tensor:
    """(B, num_class) float32 logits of ``model`` summed over the votes of vote_batch, in ascending v (evaluate.py:
    126-138), under torch.no_grad() and in whatever train / eval mode the caller set.  The model is called as
    ``model(points, lengths)`` on ``chunk`` votes of all B shapes at a time (default: every vote in one call).  Inside
    layers.batch_invariant() (an eval-mode model of SharedMLP layers) the logits do not depend on ``chunk``."""
    if isinstance(num_votes, bool) or not isinstance(num_votes, int) or num_votes < 1:
        raise ValueError(f"classify_votes expects a positive integer num_votes, got {num_votes!r}")
    if chunk is None:
        chunk = num_votes
    if isinstance(chunk, bool) or not isinstance(chunk, int) or chunk < 1:
        raise ValueError(f"classify_votes expects a positive integer chunk, got {chunk!r}")
    votes = vote_batch(shapes, shape_idx, num_votes, seed, npoints)
    b = shape_idx.shape[0]
    acc = None
    with torch.no_grad():
        for v0 in range(0, num_votes, chunk):
            v1 = min(num_votes, v0 + chunk)
            out = model(votes.points[v0 * b:v1 * b], votes.lengths[v0 * b:v1 * b])
            logits = (out[0] if isinstance(out, (tuple, list)) else out).float()
            if acc is None:
                acc = torch.zeros(b, logits.shape[-1], dtype=torch.float32, device=logits.device)
            for v in range(v1 - v0):
                acc += logits[v * b:(v + 1) * b]
    return acc


def cls_accuracy(pred_class: torch.Tensor, label: torch.Tensor, num_class: int):
    """(accuracy, mean class accuracy) of evaluate.py:141-158 as 0-d float64 tensors on the inputs' device, without a
    read-back: correct / seen over all shapes, and the mean over the num_class classes of correct / seen per class (a
    class with no shape gives NaN, as numpy's 0 / 0 does there)."""
    if isinstance(num_class, bool) or not isinstance(num_class, int) or num_class < 1:
        raise ValueError(f"cls_accuracy expects a positive integer num_class, got {num_class!r}")
    if pred_class.shape != label.shape or pred_class.dim() != 1:
        raise ValueError(f"cls_accuracy expects (B,) pred_class and label, got {tuple(pred_class.shape)} and "
                         f"{tuple(label.shape)}")
    pred_class, label = pred_class.long(), label.long()
    hit = (pred_class == label).double()
    # per-class counts by scatter_add (bincount and boolean indexing would read back); a label outside [0, num_class)
    # counts in the accuracy only
    inside = ((label >= 0) & (label < num_class)).double()
    idx = label.clamp(0, num_class - 1)
    seen = torch.zeros(num_class, dtype=torch.float64, device=label.device).scatter_add_(0, idx, inside)
    correct = torch.zeros(num_class, dtype=torch.float64, device=label.device).scatter_add_(0, idx, hit * inside)
    return hit.mean(), (correct / seen).mean()
