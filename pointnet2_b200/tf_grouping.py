"""Grouping ops — drop-in for the reference's tf_ops/grouping/tf_grouping.py.

Same function names, positional order and return tuples as tf_grouping.py:8-73 on contiguous CUDA
torch tensors.  group_point is differentiable w.r.t. ``points`` (tf_grouping.py:42-46);
query_ball_point / select_top_k have no gradient (ops.NoGradient, :21,:32).
"""
from __future__ import annotations

import torch

from . import _lib
from ._tensor import DTYPE_CODES, FEATURE_DTYPES, device_lengths, on_device, ptr, require_cuda, same_device, stream_ptr


def query_ball_point(radius: float, nsample: int, xyz1: torch.Tensor, xyz2: torch.Tensor, *, lengths=None):
    """For every query centre, the first ``nsample`` data points (ascending index) closer than ``radius``.

    Arguments: ``radius`` of the ball; ``nsample`` row length; ``xyz1`` float32 (B, N, 3), the cloud that is
    searched; ``xyz2`` float32 (B, M, 3), the ball centres.
    Returns ``idx`` int32 (B, M, nsample) — positions in ``xyz1``, short rows padded with their first hit — and
    ``pts_cnt`` int32 (B, M), how many distinct hits each row holds.
    ``lengths`` (B,) integers, optional: the data cloud b is ``xyz1[b, :lengths[b]]`` (variable-size clouds padded to
    N); each row is then exactly what this function returns for that cloud alone, and the padding rows are never read.
    Reference: tf_grouping.py:8-20 -> QueryBallPointGpuOp (tf_grouping.cpp:67-106) ->
    query_ball_point_gpu (tf_grouping_g.cu:3-36).  Rows with no point in the ball (undefined in the
    reference) come back as zeros with pts_cnt 0.
    """
    radius = float(radius)
    nsample = int(nsample)
    if not radius > 0:
        raise ValueError("QueryBallPoint expects positive radius")
    if nsample <= 0:
        raise ValueError("QueryBallPoint expects positive nsample")
    xyz1 = require_cuda(xyz1, "xyz1", torch.float32)
    xyz2 = require_cuda(xyz2, "xyz2", torch.float32)
    same_device(xyz1, xyz2)
    if xyz1.dim() != 3 or xyz1.shape[2] != 3:
        raise ValueError(f"QueryBallPoint expects (batch_size, ndataset, 3) xyz1 shape, got {tuple(xyz1.shape)}")
    if xyz2.dim() != 3 or xyz2.shape[2] != 3 or xyz2.shape[0] != xyz1.shape[0]:
        raise ValueError(f"QueryBallPoint expects (batch_size, npoint, 3) xyz2 shape, got {tuple(xyz2.shape)}")
    b, n, _ = xyz1.shape
    m = xyz2.shape[1]
    if n <= 0 and b * m:
        raise ValueError("QueryBallPoint expects a non-empty xyz1")
    lens = device_lengths(lengths, b, n, xyz1.device, "QueryBallPoint")
    if torch.compiler.is_compiling():
        return torch.ops.pn2.query_ball_point(radius, nsample, xyz1.detach(), xyz2.detach(), lens)
    return query_ball_point_launch(radius, nsample, xyz1, xyz2, lens)


def query_ball_point_launch(radius: float, nsample: int, xyz1: torch.Tensor, xyz2: torch.Tensor, lens):
    b, n, _ = xyz1.shape
    m = xyz2.shape[1]
    idx = torch.empty((b, m, nsample), dtype=torch.int32, device=xyz1.device)
    pts_cnt = torch.empty((b, m), dtype=torch.int32, device=xyz1.device)
    if b * m:
        lib = _lib.load()
        with on_device(xyz1):
            ws_bytes = int(lib.pn2_query_ball_point_workspace_bytes(b, n))
            if lens is not None:  # same paths as below; the library takes the lengths to every kernel
                ws = torch.empty(ws_bytes, dtype=torch.uint8, device=xyz1.device) if ws_bytes else None
                rc = lib.pn2_query_ball_point_ragged(b, n, m, radius, nsample, ptr(xyz1), ptr(lens), ptr(xyz2), ptr(idx),
                                                     ptr(pts_cnt), ptr(ws), ws_bytes, stream_ptr(xyz1.device))
            elif ws_bytes:  # sparse balls are served through a uniform grid built in this scratch
                ws = torch.empty(ws_bytes, dtype=torch.uint8, device=xyz1.device)
                rc = lib.pn2_query_ball_point_ws(b, n, m, radius, nsample, ptr(xyz1), ptr(xyz2), ptr(idx), ptr(pts_cnt),
                                                 ptr(ws), ws_bytes, stream_ptr(xyz1.device))
            else:
                rc = lib.pn2_query_ball_point(b, n, m, radius, nsample, ptr(xyz1), ptr(xyz2), ptr(idx),
                                              ptr(pts_cnt), stream_ptr(xyz1.device))
        _lib.check(rc, "pn2_query_ball_point")
    return idx, pts_cnt


def select_top_k(k: int, dist: torch.Tensor):
    """k rounds of selection sort along the last axis of a distance matrix.

    Arguments: ``k`` — how many of the smallest entries to bring to the front; ``dist`` float32 (B, M, N), one row
    of N distances per query.
    Returns ``(idx, dist_out)``, both (B, M, N): columns [0, k) hold the k smallest distances in ascending order and
    their original column numbers, the remaining columns the reference's swapped-around tail.
    Reference: tf_grouping.py:22-31 -> SelectionSortGpuOp (tf_grouping.cpp:110-139) ->
    selection_sort_gpu (tf_grouping_g.cu:83-123).
    """
    k = int(k)
    if k <= 0:
        raise ValueError("SelectionSort expects positive k")
    dist = require_cuda(dist, "dist", torch.float32)
    if dist.dim() != 3:
        raise ValueError(f"SelectionSort expects (b,m,n) dist shape, got {tuple(dist.shape)}")
    if torch.compiler.is_compiling():
        return torch.ops.pn2.select_top_k(k, dist.detach())
    return select_top_k_launch(k, dist)


def select_top_k_launch(k: int, dist: torch.Tensor):
    b, m, n = dist.shape
    outi = torch.empty((b, m, n), dtype=torch.int32, device=dist.device)
    out = torch.empty((b, m, n), dtype=torch.float32, device=dist.device)
    if b * m * n:
        with on_device(dist):
            rc = _lib.load().pn2_selection_sort(b, n, m, k, ptr(dist), ptr(outi), ptr(out), stream_ptr(dist.device))
        _lib.check(rc, "pn2_selection_sort")
    return outi, out


def group_point_launch(points: torch.Tensor, idx: torch.Tensor) -> torch.Tensor:
    b, n, c = points.shape
    _, m, s = idx.shape
    out = torch.empty((b, m, s, c), dtype=points.dtype, device=points.device)
    if out.numel():
        with on_device(points):
            if points.dtype == torch.float32:
                rc = _lib.load().pn2_group_point(b, n, c, m, s, ptr(points), ptr(idx), ptr(out),
                                                 stream_ptr(points.device))
            else:
                rc = _lib.load().pn2_group_point_typed(DTYPE_CODES[points.dtype], b, n, c, m, s, ptr(points), ptr(idx),
                                                       ptr(out), stream_ptr(points.device))
        _lib.check(rc, "pn2_group_point")
    return out


class _GroupPoint(torch.autograd.Function):
    @staticmethod
    def forward(ctx, points, idx):
        ctx.save_for_backward(idx)
        ctx.shape = tuple(points.shape)
        ctx.dtype = points.dtype
        return group_point_launch(points, idx)

    @staticmethod
    def backward(ctx, grad_out):
        (idx,) = ctx.saved_tensors
        return group_point_grad(grad_out.to(ctx.dtype).contiguous(), idx, ctx.shape), None


def group_point_grad(grad_out: torch.Tensor, idx: torch.Tensor, shape) -> torch.Tensor:
    """Backward of group_point: scatter-add of ``grad_out`` (B, M, S, C) into a (B, N, C) gradient of
    ``grad_out``'s dtype; a 16-bit gradient is the float32 sum rounded once.  Float32 atomics, unless
    ``torch.are_deterministic_algorithms_enabled()``: then every point's rows are added in ascending (j, k) order, run to
    run identical and bit-identical to the reference's group_point_grad_cpu."""
    b, n, c = shape
    _, m, s = idx.shape
    dev = grad_out.device
    if torch.are_deterministic_algorithms_enabled():
        grad_points = torch.empty((b, n, c), dtype=grad_out.dtype, device=dev)  # every element is written
        if grad_points.numel():
            lib = _lib.load()
            with on_device(grad_out):
                wsb = int(lib.pn2_group_point_grad_det_workspace_bytes(b, n, max(m, 1), max(s, 1)))
                ws = torch.empty(wsb, dtype=torch.uint8, device=dev)
                rc = lib.pn2_group_point_grad_det_typed(DTYPE_CODES[grad_out.dtype], b, n, c, m, s, ptr(grad_out), ptr(idx),
                                                        ptr(grad_points), ptr(ws), wsb, stream_ptr(dev))
            _lib.check(rc, "pn2_group_point_grad_det")
        return grad_points
    # zero-filled by the caller, as GroupPointGradGpuOp does (tf_grouping.cpp:204)
    accum = torch.zeros((b, n, c), dtype=torch.float32, device=dev)
    if grad_out.dtype == torch.float32:
        if grad_out.numel():
            with on_device(grad_out):
                rc = _lib.load().pn2_group_point_grad(b, n, c, m, s, ptr(grad_out), ptr(idx), ptr(accum), stream_ptr(dev))
            _lib.check(rc, "pn2_group_point_grad")
        return accum
    if not grad_out.numel():
        return torch.zeros((b, n, c), dtype=grad_out.dtype, device=dev)
    grad_points = torch.empty((b, n, c), dtype=grad_out.dtype, device=dev)  # every element written by the rounding pass
    with on_device(grad_out):
        rc = _lib.load().pn2_group_point_grad_typed(DTYPE_CODES[grad_out.dtype], b, n, c, m, s, ptr(grad_out), ptr(idx),
                                                    ptr(grad_points), ptr(accum), stream_ptr(dev))
    _lib.check(rc, "pn2_group_point_grad")
    return grad_points


def group_point(points: torch.Tensor, idx: torch.Tensor) -> torch.Tensor:
    """Row gather: ``out[b, j, s, :] = points[b, idx[b, j, s], :]``.

    Arguments: ``points`` float32, bfloat16 or float16 (B, N, C), the rows to pick from; ``idx`` int32 (B, M, S), row
    numbers into ``points``.  Returns (B, M, S, C) in the dtype of ``points``, a bit-exact copy.  Differentiable in
    ``points``: the gradient is accumulated in float32 and, for 16-bit ``points``, rounded once.
    Reference: tf_grouping.py:33-41 -> group_point_gpu (tf_grouping_g.cu:40-57); gradient
    tf_grouping.py:42-46 -> group_point_grad_gpu (:61-78).
    """
    points = require_cuda(points, "points", FEATURE_DTYPES)
    idx = require_cuda(idx, "idx", torch.int32)
    same_device(points, idx)
    if points.dim() != 3:
        raise ValueError(f"GroupPoint expects (batch_size, num_points, channel) points shape, got {tuple(points.shape)}")
    if idx.dim() != 3 or idx.shape[0] != points.shape[0]:
        raise ValueError(f"GroupPoint expects (batch_size, npoints, nsample) idx shape, got {tuple(idx.shape)}")
    if points.shape[1] <= 0 and idx.numel():
        raise ValueError("GroupPoint expects a non-empty points tensor")
    if torch.compiler.is_compiling():
        return torch.ops.pn2.group_point(points, idx)
    return _GroupPoint.apply(points, idx)


def knn_point(k: int, xyz1: torch.Tensor, xyz2: torch.Tensor, *, lengths=None, query_lengths=None):
    """The k nearest data points of every query point, by squared Euclidean distance.

    Arguments: ``k`` neighbours per query; ``xyz1`` float32 (B, N, c), the cloud that is searched; ``xyz2`` float32
    (B, M, c), the queries.  Returns ``val`` float32 (B, M, k), the squared distances in ascending order, and
    ``idx`` int32 (B, M, k), the matching positions in ``xyz1``.
    Reference: tf_grouping.py:48-73.  The reference builds the (b,m,n) matrix of squared distances
    sum((xyz1 - xyz2)**2, -1) and runs select_top_k on it; for 3-D points and k <= 128 this runs one
    tiled top-k kernel instead (pn2_knn_point: no matrix), whose val / idx equal the first k columns
    of that composite bit for bit, ties included.  Other shapes take the composite itself.

    ``lengths`` (B,) integers, optional: the data cloud b is ``xyz1[b, :lengths[b]]`` (variable-size clouds padded to
    N).  With k_b = min(k, lengths[b]), columns [0, k_b) of each row are what this function returns for that cloud
    alone with k_b neighbours; a cloud shorter than k repeats column 0 in columns [k_b, k) (``val`` and ``idx``), as
    the ball query pads a short row with its first hit.  ``query_lengths`` (B,) integers, optional: the query cloud b
    is ``xyz2[b, :query_lengths[b]]``; rows past it come back as idx 0 / val +inf.  Padding rows are never read.  A
    device tensor is never read on the host (its values are clamped to [1, N] / [1, M] on the device), so the call
    can be captured in a CUDA graph; a host tensor or sequence is checked here.  Lengths need the kernel: 3-D points
    and k <= 128 (ValueError otherwise).
    """
    k = int(k)
    if k <= 0:
        raise ValueError("knn_point expects positive k")
    xyz1 = require_cuda(xyz1, "xyz1", torch.float32)
    xyz2 = require_cuda(xyz2, "xyz2", torch.float32)
    same_device(xyz1, xyz2)
    if xyz1.dim() != 3 or xyz2.dim() != 3 or xyz1.shape[0] != xyz2.shape[0] or xyz1.shape[2] != xyz2.shape[2]:
        raise ValueError("knn_point expects (b,n,c) xyz1 and (b,m,c) xyz2")
    b, n, c = xyz1.shape
    m = xyz2.shape[1]
    if k > n:
        raise ValueError(f"knn_point expects k <= ndataset (the reference slices k columns of an n-column matrix), got k={k}, n={n}")
    ragged = lengths is not None or query_lengths is not None
    if ragged and not (c == 3 and k <= 128):
        raise ValueError(f"knn_point takes lengths only for 3-D points and k <= 128 (the kernel), got c={c}, k={k}")
    lens = device_lengths(lengths, b, n, xyz1.device, "knn_point")
    qlens = device_lengths(query_lengths, b, m, xyz1.device, "knn_point") if m else None
    if c == 3 and k <= 128:
        if torch.compiler.is_compiling():
            return torch.ops.pn2.knn_point(k, xyz1.detach(), xyz2.detach(), lens, qlens)
        return knn_point_launch(k, xyz1, xyz2, lens, qlens)
    diff = xyz1.unsqueeze(1) - xyz2.unsqueeze(2)  # (b,m,n,c): tile(xyz1) - tile(xyz2), tf_grouping.py:64-66
    dist = (diff * diff).sum(-1)
    outi, out = select_top_k(k, dist)
    return out[:, :, :k].contiguous(), outi[:, :, :k].contiguous()


def knn_point_launch(k: int, xyz1: torch.Tensor, xyz2: torch.Tensor, lens, qlens):
    """knn_point's kernel (3-D points, k <= 128): (val, idx)"""
    b, n, _ = xyz1.shape
    m = xyz2.shape[1]
    ragged = lens is not None or qlens is not None
    val = torch.empty((b, m, k), dtype=torch.float32, device=xyz1.device)
    idx = torch.empty((b, m, k), dtype=torch.int32, device=xyz1.device)
    if b * m:
        with on_device(xyz1):
            if ragged:
                rc = _lib.load().pn2_knn_point_ragged(b, n, m, k, ptr(xyz1.detach()), ptr(lens), ptr(xyz2.detach()), ptr(qlens),
                                                      ptr(val), ptr(idx), stream_ptr(xyz1.device))
            else:
                rc = _lib.load().pn2_knn_point(b, n, m, k, ptr(xyz1.detach()), ptr(xyz2.detach()), ptr(val), ptr(idx),
                                               stream_ptr(xyz1.device))
        _lib.check(rc, "pn2_knn_point")
    return val, idx
