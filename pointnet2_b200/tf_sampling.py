"""Sampling ops — drop-in for the reference's tf_ops/sampling/tf_sampling.py.

Same function names, positional order and return values as tf_sampling.py:29-57, taking and
returning contiguous CUDA torch tensors (float32 / int32).  Differentiable exactly where the
reference registers a gradient: gather_point w.r.t. ``inp`` (tf_sampling.py:43-47);
farthest_point_sample has none (ops.NoGradient, :57).

``prob_sample`` (tf_sampling.py:13-21) is outside the set-abstraction path (SURVEY.md §8: only the
module's __main__ demo calls it); it is provided for completeness and kept out of every measurement.
"""
from __future__ import annotations

import torch

from . import _lib
from ._tensor import on_device, ptr, require_cuda, same_device, stream_ptr


def _check_xyz(t: torch.Tensor, name: str, op: str) -> None:
    if t.dim() != 3 or t.shape[2] != 3:
        raise ValueError(f"{op} expects (batch_size,num_points,3) {name} shape, got {tuple(t.shape)}")


def prob_sample(inp: torch.Tensor, inpr: torch.Tensor) -> torch.Tensor:
    """Inverse-CDF sampling: one category per uniform draw.

    ``inp`` float32 (B, K): non-negative, unnormalised weights of K categories; ``inpr`` float32 (B, M): draws in
    [0, 1].  Returns int32 (B, M), the category each draw falls into.
    Reference: tf_sampling.py:13-21 -> ProbSampleGpuOp (tf_sampling.cpp:66-92) ->
    probsampleLauncher (tf_sampling_g.cu:198-201): cumulative sum, then the first index whose
    cumulative sum reaches inpr * total.  No gradient (ops.NoGradient, tf_sampling.py:22).
    """
    inp = require_cuda(inp, "inp", torch.float32)
    inpr = require_cuda(inpr, "inpr", torch.float32)
    same_device(inp, inpr)
    if inp.dim() != 2:
        raise ValueError(f"ProbSample expects (batch_size,num_choices) inp shape, got {tuple(inp.shape)}")
    if inpr.dim() != 2 or inpr.shape[0] != inp.shape[0]:
        raise ValueError(f"ProbSample expects (batch_size,num_points) inpr shape, got {tuple(inpr.shape)}")
    b, n = inp.shape
    m = inpr.shape[1]
    if n <= 0 and b * m:
        raise ValueError("ProbSample expects a non-empty inp")
    out = torch.empty((b, m), dtype=torch.int32, device=inp.device)
    if b * m:
        temp = torch.empty((b, n), dtype=torch.float32, device=inp.device)  # the op's allocate_temp
        with on_device(inp):
            rc = _lib.load().pn2_prob_sample(b, n, m, ptr(inp), ptr(inpr), ptr(temp), ptr(out), stream_ptr(inp.device))
        _lib.check(rc, "pn2_prob_sample")
    return out


def farthest_point_sample(npoint: int, inp: torch.Tensor) -> torch.Tensor:
    """Farthest point sampling: ``npoint`` picks per cloud, each the point farthest from everything picked so far.

    ``inp`` float32 (B, N, 3).  Returns int32 (B, npoint), positions in ``inp``; the first pick is point 0.
    Reference: tf_sampling.py:48-56 -> FarthestPointSampleGpuOp (tf_sampling.cpp:95-123) ->
    farthestpointsamplingKernel (tf_sampling_g.cu:105-170).  Deterministic, starts at index 0.
    """
    npoint = int(npoint)
    if npoint <= 0:
        raise ValueError("FarthestPointSample expects positive npoint")
    inp = require_cuda(inp, "inp", torch.float32)
    _check_xyz(inp, "inp", "FarthestPointSample")
    b, n, _ = inp.shape
    if n <= 0:
        raise ValueError("FarthestPointSample expects at least one point per batch entry")
    out = torch.empty((b, npoint), dtype=torch.int32, device=inp.device)
    if b == 0:
        return out
    lib = _lib.load()
    with on_device(inp):
        # clouds beyond the cluster kernels' capacity (n > 425984) need the reference's own
        # (32, n) float scratch (tf_sampling.cpp:115); the library says how much
        tb = int(lib.pn2_fps_scratch_bytes(b, n))
        temp = torch.empty(tb, dtype=torch.uint8, device=inp.device) if tb else None
        rc = lib.pn2_fps(b, n, npoint, ptr(inp), ptr(temp), ptr(out), stream_ptr(inp.device))
    _lib.check(rc, "pn2_fps")
    return out


def farthest_point_sample_and_gather(npoint: int, inp: torch.Tensor):
    """FPS and gather_point in one launch: returns (idx (b,npoint) int32, new_xyz (b,npoint,3)).
    Equivalent to ``idx = farthest_point_sample(npoint, inp); gather_point(inp, idx)``
    (utils/pointnet_util.py:40); new_xyz carries no gradient here."""
    npoint = int(npoint)
    if npoint <= 0:
        raise ValueError("FarthestPointSample expects positive npoint")
    inp = require_cuda(inp, "inp", torch.float32)
    _check_xyz(inp, "inp", "FarthestPointSample")
    b, n, _ = inp.shape
    if n <= 0:
        raise ValueError("FarthestPointSample expects at least one point per batch entry")
    idx = torch.empty((b, npoint), dtype=torch.int32, device=inp.device)
    new_xyz = torch.empty((b, npoint, 3), dtype=torch.float32, device=inp.device)
    if b == 0:
        return idx, new_xyz
    lib = _lib.load()
    with on_device(inp):
        tb = int(lib.pn2_fps_scratch_bytes(b, n))
        temp = torch.empty(tb, dtype=torch.uint8, device=inp.device) if tb else None
        rc = lib.pn2_fps_gather(b, n, npoint, ptr(inp), ptr(temp), ptr(idx), ptr(new_xyz), stream_ptr(inp.device))
    _lib.check(rc, "pn2_fps_gather")
    return idx, new_xyz


class _GatherPoint(torch.autograd.Function):
    @staticmethod
    def forward(ctx, inp, idx):
        b, n, _ = inp.shape
        m = idx.shape[1]
        out = torch.empty((b, m, 3), dtype=torch.float32, device=inp.device)
        if b * m:
            with on_device(inp):
                rc = _lib.load().pn2_gather_point(b, n, m, ptr(inp), ptr(idx), ptr(out), stream_ptr(inp.device))
            _lib.check(rc, "pn2_gather_point")
        ctx.save_for_backward(idx)
        ctx.n = n
        return out

    @staticmethod
    def backward(ctx, out_g):
        (idx,) = ctx.saved_tensors
        b, m = idx.shape
        out_g = out_g.contiguous()
        lib = _lib.load()
        if torch.are_deterministic_algorithms_enabled():
            # no atomics: each point's rows added in ascending j, every element of inp_g written
            inp_g = torch.empty((b, ctx.n, 3), dtype=torch.float32, device=out_g.device)
            if inp_g.numel():
                with on_device(out_g):
                    wsb = int(lib.pn2_group_point_grad_det_workspace_bytes(b, ctx.n, max(m, 1), 1))
                    ws = torch.empty(wsb, dtype=torch.uint8, device=out_g.device)
                    rc = lib.pn2_gather_point_grad_det(b, ctx.n, m, ptr(out_g), ptr(idx), ptr(inp_g), ptr(ws), wsb,
                                                       stream_ptr(out_g.device))
                _lib.check(rc, "pn2_gather_point_grad_det")
            return inp_g, None
        # the caller zero-fills, as GatherPointGradGpuOp does (tf_sampling.cpp:174)
        inp_g = torch.zeros((b, ctx.n, 3), dtype=torch.float32, device=out_g.device)
        if b * m:
            with on_device(out_g):
                rc = lib.pn2_gather_point_grad(b, ctx.n, m, ptr(out_g), ptr(idx), ptr(inp_g), stream_ptr(out_g.device))
            _lib.check(rc, "pn2_gather_point_grad")
        return inp_g, None


def gather_point(inp: torch.Tensor, idx: torch.Tensor) -> torch.Tensor:
    """Row gather of coordinates: ``out[b, j, :] = inp[b, idx[b, j], :]``.

    ``inp`` float32 (B, N, 3); ``idx`` int32 (B, M).  Returns float32 (B, M, 3).  Differentiable in ``inp``: float
    atomics, or, when ``torch.are_deterministic_algorithms_enabled()``, ordered sums (ascending j, run to run identical).
    Reference: tf_sampling.py:29-37 -> gatherpointKernel (tf_sampling_g.cu:172-181);
    gradient tf_sampling.py:43-47 -> scatteraddpointKernel (:183-192).
    """
    inp = require_cuda(inp, "inp", torch.float32)
    idx = require_cuda(idx, "idx", torch.int32)
    same_device(inp, idx)
    _check_xyz(inp, "inp", "GatherPoint")
    if idx.dim() != 2 or idx.shape[0] != inp.shape[0]:
        raise ValueError(f"GatherPoint expects (batch_size,num_result) idx shape, got {tuple(idx.shape)}")
    return _GatherPoint.apply(inp, idx)
