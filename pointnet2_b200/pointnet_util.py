"""PointNet++ layer glue — the torch twin of the reference's utils/pointnet_util.py for the
set-abstraction / feature-propagation geometry path.

``sample_and_group`` / ``sample_and_group_all`` keep the reference's signatures and return tuples
(utils/pointnet_util.py:22-56, :59-84).  ``pointnet_sa_module``, ``pointnet_sa_module_msg`` and
``pointnet_fp_module`` keep the reference's full positional signatures (:87, :156, :199 — ``mlp`` lists of
widths, ``is_training``, ``bn_decay``, ``scope``, ``bn`` ...), so the reference's model files call them
unchanged; the dense half (1x1 conv + BN + ReLU stacks, :115-153, :187-195, :218-228) is torch layers: width lists
resolve to ``layers.SharedMLP`` modules kept in a variable-scope registry (``layers.scoped_mlp``), or pass a callable, or
None to get the grouped tensor pooled as-is.

``fused=True`` (default) routes through the fused kernels (FPS+gather in one launch,
group+centre+concat in one pass); ``fused=False`` issues the reference's exact op sequence.  Both
produce identical values.  At inference (a SharedMLP in eval mode, grad mode off, max-pooling: ``layers.sa_mlp_applies``)
``fused=True`` also runs the learned tail of a set-abstraction level in the kernel behind ``layers.sa_mlp_max``: gather,
every layer and the max-pool in one launch, no grouped tensor in between.  Its float32 results differ from the torch
layers' by float32 rounding (the sums are ordered differently), and unlike theirs do not depend on the batch size.
"""
from __future__ import annotations

from typing import Callable, Optional, Sequence

import torch

from . import _lib, layers
from ._tensor import DTYPE_CODES, FEATURE_DTYPES, device_lengths, on_device, ptr, require_cuda, same_device, stream_ptr
from .tf_grouping import group_point, group_point_grad, knn_point, query_ball_point
from .tf_interpolate import fp_interpolate_concat, three_interpolate, three_nn, three_nn_interpolate
from .sa_layer import KNN_MAX_K, sample_group, sample_group_msg, sample_knn
from .tf_sampling import farthest_point_sample, farthest_point_sample_and_gather, gather_point


def group_and_concat_launch(xyz, new_xyz, points, idx, xyz_first: bool):
    """(out, grouped_xyz) of group_and_concat: out has the dtype of ``points`` (float32 without points); grouped_xyz is
    float32."""
    b, n, _ = xyz.shape
    _, m, s = idx.shape
    c = 0 if points is None else points.shape[2]
    dtype = torch.float32 if points is None else points.dtype
    out = torch.empty((b, m, s, 3 + c), dtype=dtype, device=xyz.device)
    gxyz = torch.empty((b, m, s, 3), dtype=torch.float32, device=xyz.device)
    if out.numel():
        with on_device(xyz):
            if dtype == torch.float32:
                rc = _lib.load().pn2_group_concat(b, n, c, m, s, ptr(xyz), ptr(new_xyz), ptr(points), ptr(idx),
                                                  1 if xyz_first else 0, ptr(out), ptr(gxyz), stream_ptr(xyz.device))
            else:
                rc = _lib.load().pn2_group_concat_typed(DTYPE_CODES[dtype], b, n, c, m, s, ptr(xyz), ptr(new_xyz), ptr(points),
                                                        ptr(idx), 1 if xyz_first else 0, ptr(out), ptr(gxyz),
                                                        stream_ptr(xyz.device))
        _lib.check(rc, "pn2_group_concat")
    return out, gxyz


def group_and_concat_backward(g_out, g_gxyz, idx, n: int, xyz_first: bool, has_points: bool, need_xyz: bool,
                              need_new_xyz: bool):
    """Gradients (xyz, new_xyz, points) of group_and_concat from those of (out, grouped_xyz), each None when not wanted;
    ``g_out`` in the dtype of out, ``g_gxyz`` float32 or None."""
    c = g_out.shape[-1] - 3
    lo = 0 if xyz_first else c
    g_xyz = g_new_xyz = g_points = None
    if need_xyz or need_new_xyz:  # in the networks the coordinates need none
        g_xyz_part = g_out[..., lo:lo + 3].float()  # the coordinates' gradient is float32 (an exact upcast)
        if g_gxyz is not None:
            g_xyz_part = g_xyz_part + g_gxyz
        g_xyz_part = g_xyz_part.contiguous()
        if need_xyz:
            g_xyz = group_point_grad(g_xyz_part, idx, (idx.shape[0], n, 3))
        if need_new_xyz:
            g_new_xyz = -g_xyz_part.sum(dim=2)
    if has_points:
        g_feat = (g_out[..., 3:] if xyz_first else g_out[..., :c]).contiguous()
        g_points = group_point_grad(g_feat, idx, (idx.shape[0], n, c))
    return g_xyz, g_new_xyz, g_points


class _GroupConcat(torch.autograd.Function):
    @staticmethod
    def forward(ctx, xyz, new_xyz, points, idx, xyz_first):
        b, n, _ = xyz.shape
        _, m, s = idx.shape
        c = 0 if points is None else points.shape[2]
        ctx.save_for_backward(idx)
        ctx.meta = (b, n, c, m, s, bool(xyz_first), points is not None)
        ctx.dtype = torch.float32 if points is None else points.dtype
        return group_and_concat_launch(xyz, new_xyz, points, idx, xyz_first)

    @staticmethod
    def backward(ctx, g_out, g_gxyz):
        (idx,) = ctx.saved_tensors
        _, n, _, _, _, xyz_first, has_points = ctx.meta
        return (*group_and_concat_backward(g_out.to(ctx.dtype), g_gxyz, idx, n, xyz_first, has_points,
                                           ctx.needs_input_grad[0], ctx.needs_input_grad[1]), None, None)


def group_and_concat(xyz, new_xyz, points, idx, xyz_first: bool = True):
    """Fused tail of sample_and_group: returns (new_points (b,m,s,3+c), grouped_xyz (b,m,s,3)).

    ``points`` may be float32, bfloat16 or float16: new_points then has its dtype, with the feature channels copied and
    the xyz channels (float32 differences) rounded once; grouped_xyz is float32 in every case."""
    xyz = require_cuda(xyz, "xyz", torch.float32)
    new_xyz = require_cuda(new_xyz, "new_xyz", torch.float32)
    idx = require_cuda(idx, "idx", torch.int32)
    if points is not None:
        points = require_cuda(points, "points", FEATURE_DTYPES)
        same_device(xyz, new_xyz, idx, points)
        if points.dim() != 3 or points.shape[:2] != xyz.shape[:2]:
            raise ValueError("points must be (batch_size, ndataset, channel) matching xyz")
    else:
        same_device(xyz, new_xyz, idx)
    if idx.dim() != 3 or idx.shape[0] != xyz.shape[0] or new_xyz.shape[:2] != idx.shape[:2]:
        raise ValueError("idx must be (batch_size, npoint, nsample) matching new_xyz")
    if torch.compiler.is_compiling():
        return torch.ops.pn2.group_and_concat(xyz, new_xyz, points, idx, bool(xyz_first))
    return _GroupConcat.apply(xyz, new_xyz, points, idx, xyz_first)


def _no_lengths_with(lengths, what: str) -> None:
    if lengths is not None:
        raise ValueError(f"lengths (variable-size clouds) are not supported with {what}")


def sample_and_group(npoint, radius, nsample, xyz, points, knn=False, use_xyz=True, fused=True, *, lengths=None):
    """Sampling + grouping half of a set-abstraction layer (same positional arguments and return
    tuple as the reference's sample_and_group, utils/pointnet_util.py:22-56).

    Args:
        npoint, radius, nsample: centroids to sample, ball radius, neighbours kept per centroid.
        xyz (b, n, 3) float32; points (b, n, c) float32, bfloat16 or float16, or None (then the grouped xyz are
        the features).  new_points has the dtype of points (float32 without points).
        knn: k-nearest-neighbour grouping instead of the ball query; use_xyz: keep the centred xyz
        in front of the grouped features.
    Returns:
        new_xyz (b, npoint, 3), new_points (b, npoint, nsample, 3 + c) [c alone when use_xyz is False],
        idx (b, npoint, nsample) int32 into the n input points, grouped_xyz (b, npoint, nsample, 3)
        centred on new_xyz.
        lengths: optional (b,) integers: cloud i is ``xyz[i, :lengths[i]]`` (and ``points[i, :lengths[i]]``), padded to
        n.  Sampling and the ball query then see each cloud alone; every index is below its length, so the grouping
        never reads the padding.  Not with knn (ValueError): kNN grouping of variable-size clouds is
        ``pointnet_sa_module(..., knn=True, lengths=)``, or ``sa_layer.sample_knn(..., lengths=)`` for the grouped xyz.

    ``fused=True`` uses the overlapped sampling+grouping layer (sa_layer.sample_group, or sa_layer.sample_knn for
    knn with nsample <= 128) and the single-pass concat kernel; ``fused=False`` issues the reference's op sequence one by one.  Both
    return identical values.
    """
    if knn:
        _no_lengths_with(lengths, "knn grouping in sample_and_group (pointnet_sa_module(knn=True) and sa_layer.sample_knn "
                                  "take them)")
    return _sample_and_group(npoint, radius, nsample, xyz, points, knn, use_xyz, fused, lengths)


def _sample_and_group(npoint, radius, nsample, xyz, points, knn, use_xyz, fused, lengths):
    """sample_and_group, with lengths for kNN grouping too: knn_point(lengths=) semantics, so a cloud shorter than
    nsample repeats its nearest neighbour (column 0) in the rest of each row, as the ball query pads a short row."""
    no_grad_xyz = not xyz.requires_grad
    if fused and no_grad_xyz and knn and 0 < int(nsample) <= min(KNN_MAX_K, xyz.shape[1]):
        # one call: FPS + gather + kNN (+ centred grouped xyz when they are the whole output), the kNN grouping
        # overlapping the sampling chain
        need_g = points is None or not use_xyz
        _, new_xyz, idx, _, grouped_xyz = sample_knn(npoint, nsample, xyz, center=True, want_grouped=need_g, lengths=lengths)
        if points is None:
            return new_xyz, grouped_xyz, idx, grouped_xyz
        if not use_xyz:
            return new_xyz, group_point(points, idx), idx, grouped_xyz
        new_points, grouped_xyz = group_and_concat(xyz, new_xyz, points, idx, xyz_first=True)
        return new_xyz, new_points, idx, grouped_xyz
    if fused and no_grad_xyz and not knn:
        # one call: FPS + gather + ball query (+ centred grouped xyz when they are the whole output)
        need_g = points is None or not use_xyz
        _, new_xyz, idx, _, grouped_xyz = sample_group(npoint, radius, nsample, xyz, center=True, want_grouped=need_g,
                                                       lengths=lengths)
        if points is None:
            return new_xyz, grouped_xyz, idx, grouped_xyz
        if not use_xyz:
            return new_xyz, group_point(points, idx), idx, grouped_xyz
        new_points, grouped_xyz = group_and_concat(xyz, new_xyz, points, idx, xyz_first=True)
        return new_xyz, new_points, idx, grouped_xyz
    if fused and no_grad_xyz:
        _, new_xyz = farthest_point_sample_and_gather(npoint, xyz, lengths=lengths)
    else:
        new_xyz = gather_point(xyz, farthest_point_sample(npoint, xyz, lengths=lengths))
    if knn:
        _, idx = knn_point(nsample, xyz, new_xyz, lengths=lengths)
    else:
        idx, _ = query_ball_point(radius, nsample, xyz, new_xyz, lengths=lengths)
    if fused:
        feats = points if (points is not None and use_xyz) else None
        if points is not None and not use_xyz:
            grouped_xyz = group_point(xyz, idx) - new_xyz.unsqueeze(2)
            return new_xyz, group_point(points, idx), idx, grouped_xyz
        new_points, grouped_xyz = group_and_concat(xyz, new_xyz, feats, idx, xyz_first=True)
        return new_xyz, new_points, idx, grouped_xyz
    # the reference's sequence, op by op (:44-54)
    grouped_xyz = group_point(xyz, idx) - new_xyz.unsqueeze(2)
    if points is None:
        new_points = grouped_xyz
    else:
        grouped_points = group_point(points, idx)
        # (cast back: torch.cat promotes 16-bit features to the coordinates' float32)
        new_points = torch.cat([grouped_xyz, grouped_points], dim=-1).to(points.dtype) if use_xyz else grouped_points
    return new_xyz, new_points, idx, grouped_xyz


def sample_and_group_all(xyz, points, use_xyz=True):
    """The group_all variant (reference utils/pointnet_util.py:59-84): one group holding every point,
    centred on the origin — no sampling, no search, no kernel.

    Returns new_xyz (b, 1, 3) zeros, new_points (b, 1, n, 3 + c) (xyz first; c alone when use_xyz is
    False; the xyz themselves when points is None), idx (b, 1, n) = arange, grouped_xyz (b, 1, n, 3).
    """
    b, n = xyz.shape[0], xyz.shape[1]
    new_xyz = xyz.new_zeros((b, 1, 3))
    idx = torch.arange(n, dtype=torch.int32, device=xyz.device).view(1, 1, n).expand(b, 1, n).contiguous()
    grouped_xyz = xyz.view(b, 1, n, 3)
    if points is None:
        return new_xyz, grouped_xyz, idx, grouped_xyz
    new_points = (torch.cat([xyz, points], dim=2) if use_xyz else points).unsqueeze(1)
    return new_xyz, new_points, idx, grouped_xyz


def _apply_mlp(mlp, t: torch.Tensor, scope=None, name="mlp", bn=True, is_training=None, bn_decay=None, mask=None) -> torch.Tensor:
    """``mlp`` is None (identity), a callable on a (..., channel) tensor, or — the reference's form — a list of
    output widths, resolved to the SharedMLP registered under ``scope/name`` (layers.scoped_mlp).  ``mask`` (rows of a
    padded batch, see layers.SharedMLP.forward) is passed on to a SharedMLP; the caller has refused other callables."""
    if mlp is None:
        return t
    if callable(mlp):
        return mlp(t) if mask is None else mlp(t, mask)
    widths = [int(w) for w in mlp]
    if not widths:
        return t
    mod = layers.scoped_mlp(scope, name, t.shape[-1], widths, bn, t.device, is_training, bn_decay)
    return mod(t) if mask is None else mod(t, mask)


def _sa_mlp_route(mlp, xyz, points, use_xyz, scope, name, bn, is_training, bn_decay, pooling='max'):
    """The SharedMLP behind ``mlp`` (a module, or a width list resolved through the scope registry) when the level's
    tail runs through layers.sa_mlp_max, else None."""
    if mlp is None or xyz.requires_grad or torch.is_grad_enabled() or pooling != 'max':
        return None
    if not callable(mlp):
        widths = [int(w) for w in mlp]
        if not widths:
            return None
        cin = 3 if points is None else points.shape[-1] + (3 if use_xyz else 0)
        mlp = layers.scoped_mlp(scope, name, cin, widths, bn, xyz.device, is_training, bn_decay)
    return mlp if layers.sa_mlp_applies(mlp, xyz, points, pooling) else None


def _fp_mlp_route(mlp, xyz1, points1, points2, scope, bn, is_training, bn_decay):
    """The SharedMLP behind ``mlp`` (a module, or a width list resolved through the scope registry) when a
    feature-propagation level runs through layers.fp_mlp: inside layers.batch_invariant(), where layers.invariant_applies.
    Else None."""
    if not layers.is_batch_invariant() or torch.is_grad_enabled() or not xyz1.is_cuda:
        return None
    if not callable(mlp):
        widths = [int(w) for w in mlp]
        if not widths:
            return None
        cin = points2.shape[-1] + (0 if points1 is None else points1.shape[-1])
        mlp = layers.scoped_mlp(scope, "conv", cin, widths, bn, xyz1.device, is_training, bn_decay)
    if not isinstance(mlp, layers.SharedMLP):
        return None  # another callable: its own SharedMLP calls route themselves
    return mlp if layers.invariant_applies(mlp, xyz1) else None


def pointnet_sa_module(xyz, points, npoint, radius, nsample, mlp=None, mlp2=None, group_all=False, is_training=None,
                       bn_decay=None, scope=None, bn=True, pooling='max', knn=False, use_xyz=True, use_nchw=False, fused=True,
                       lengths=None):
    ''' PointNet Set Abstraction (SA) Module — same positional arguments as the reference
        (utils/pointnet_util.py:87-154), so its call sites run unchanged, e.g. models/pointnet2_sem_seg.py:28:
            pointnet_sa_module(l0_xyz, l0_points, npoint=1024, radius=0.1, nsample=32, mlp=[32,32,64], mlp2=None,
                               group_all=False, is_training=is_training, bn_decay=bn_decay, scope='layer1')
        mlp / mlp2: lists of output widths (layers live in the variable-scope registry, layers.scoped_mlp; is_training
        and bn_decay set their mode and batch-norm momentum), or callables on a (batch, npoint, nsample, channel) tensor,
        or None.  use_nchw is accepted and ignored (a layout hint for TensorFlow's conv2d).
        lengths: optional (b,) per-cloud point counts of a padded batch (see sample_and_group); the outputs are dense.
        With knn, a cloud shorter than nsample repeats its nearest neighbour in the rest of each group
        (tf_grouping.knn_point), which leaves the max-pool unchanged (the other poolings count that neighbour again).
        Not with group_all (ValueError).
        Return: new_xyz (b,npoint,3), new_points (b,npoint,channels), idx (b,npoint,nsample)
    '''
    tail = _sa_mlp_route(mlp, xyz, points, use_xyz, scope, "conv", bn, is_training, bn_decay, pooling) if fused else None
    if tail is not None:
        # inference: the kernel gathers the groups itself, so only the centroids and the indices are made here
        if group_all:
            _no_lengths_with(lengths, "group_all (the max-pool over every point would need a mask)")
            b, n = xyz.shape[0], xyz.shape[1]
            new_xyz = xyz.new_zeros((b, 1, 3))
            idx = torch.arange(n, dtype=torch.int32, device=xyz.device).view(1, 1, n).expand(b, 1, n).contiguous()
            new_points = layers.sa_mlp_max(xyz, None, points, None, tail, True, use_xyz)
        else:
            if knn:
                if 0 < int(nsample) <= min(KNN_MAX_K, xyz.shape[1]):
                    _, new_xyz, idx, _, _ = sample_knn(npoint, nsample, xyz, center=True, want_grouped=False, lengths=lengths)
                else:
                    _, new_xyz = farthest_point_sample_and_gather(npoint, xyz, lengths=lengths)
                    _, idx = knn_point(nsample, xyz, new_xyz, lengths=lengths)
            else:
                _, new_xyz, idx, _, _ = sample_group(npoint, radius, nsample, xyz, center=True, want_grouped=False,
                                                     lengths=lengths)
            new_points = layers.sa_mlp_max(xyz, new_xyz, points, idx, tail, True, use_xyz)
        new_points = _apply_mlp(mlp2, new_points.unsqueeze(2), scope, "conv_post", bn, is_training, bn_decay)
        return new_xyz, new_points.squeeze(2), idx
    if group_all:
        _no_lengths_with(lengths, "group_all (the max-pool over every point would need a mask)")
        new_xyz, new_points, idx, grouped_xyz = sample_and_group_all(xyz, points, use_xyz)
    else:
        new_xyz, new_points, idx, grouped_xyz = _sample_and_group(npoint, radius, nsample, xyz, points, knn, use_xyz, fused,
                                                                  lengths)
    new_points = _apply_mlp(mlp, new_points, scope, "conv", bn, is_training, bn_decay)
    if pooling == 'max':
        new_points = new_points.max(dim=2, keepdim=True).values
    elif pooling == 'avg':
        new_points = new_points.mean(dim=2, keepdim=True)
    elif pooling == 'weighted_avg':
        dists = torch.linalg.vector_norm(grouped_xyz, ord=2, dim=-1, keepdim=True)
        exp_dists = torch.exp(-dists * 5)
        weights = exp_dists / exp_dists.sum(dim=2, keepdim=True)
        new_points = (new_points * weights).sum(dim=2, keepdim=True)
    elif pooling == 'max_and_avg':
        new_points = torch.cat([new_points.mean(dim=2, keepdim=True), new_points.max(dim=2, keepdim=True).values], dim=-1)
    else:
        raise ValueError(f"unknown pooling {pooling!r}")
    new_points = _apply_mlp(mlp2, new_points, scope, "conv_post", bn, is_training, bn_decay)
    return new_xyz, new_points.squeeze(2), idx


def pointnet_sa_module_msg(xyz, points, npoint, radius_list: Sequence[float], nsample_list: Sequence[int], mlp_list=None,
                           is_training=None, bn_decay=None, scope=None, bn=True, use_xyz=True, use_nchw=False, fused=True,
                           lengths=None):
    ''' PointNet Set Abstraction (SA) module with Multi-Scale Grouping — same positional arguments as the
        reference (utils/pointnet_util.py:156-196).  One FPS+gather, then per scale: ball query, group,
        centre, concat in the MSG order [features, xyz] (:184), MLP, max-pool; scales concatenated.
        mlp_list: per scale a list of output widths (scope registry), a callable, or None.
        lengths: optional (b,) per-cloud point counts of a padded batch (see sample_and_group); the outputs are dense.
        Return: new_xyz (b,npoint,3), new_points (b,npoint,sum of channels)
    '''
    pre = None
    if fused and not xyz.requires_grad and (points is None or use_xyz):
        tails = None if mlp_list is None else [
            _sa_mlp_route(mlp_list[i], xyz, points, use_xyz, scope, f"conv{i}", bn, is_training, bn_decay)
            for i in range(len(radius_list))]
        to_kernel = tails is not None and len(tails) > 0 and all(t is not None for t in tails)
        # one call: the sampling pass and every scale's ball query (+ centred grouped xyz when they are the features)
        _, new_xyz, idx_list, _, gxyz_list = sample_group_msg(npoint, radius_list, nsample_list, xyz, center=True,
                                                              want_grouped=points is None and not to_kernel,
                                                              lengths=lengths)
        if to_kernel:
            # inference: each scale's kernel gathers its groups and writes its channels of the concatenated result
            new_points = torch.empty((xyz.shape[0], new_xyz.shape[1], sum(t.out_channels for t in tails)),
                                     dtype=layers.sa_mlp_dtype(points), device=xyz.device)
            lo = 0
            for idx, t in zip(idx_list, tails):
                layers.sa_mlp_max(xyz, new_xyz, points, idx, t, False, use_xyz, out=new_points[..., lo:lo + t.out_channels])
                lo += t.out_channels
            return new_xyz, new_points
        pre = (idx_list, gxyz_list)
    elif fused and not xyz.requires_grad:
        _, new_xyz = farthest_point_sample_and_gather(npoint, xyz, lengths=lengths)
    else:
        new_xyz = gather_point(xyz, farthest_point_sample(npoint, xyz, lengths=lengths))
    new_points_list = []
    for i in range(len(radius_list)):
        radius, nsample = radius_list[i], nsample_list[i]
        if pre is not None:
            idx = pre[0][i]
            if points is None:
                grouped_points = pre[1][i]
            else:
                grouped_points, _ = group_and_concat(xyz, new_xyz, points, idx, xyz_first=False)
        else:
            idx, pts_cnt = query_ball_point(radius, nsample, xyz, new_xyz, lengths=lengths)
            if fused and (points is None or use_xyz):
                grouped_points, _ = group_and_concat(xyz, new_xyz, points, idx, xyz_first=False)
            else:
                grouped_xyz = group_point(xyz, idx) - new_xyz.unsqueeze(2)
                if points is not None:
                    grouped_points = group_point(points, idx)
                    if use_xyz:
                        grouped_points = torch.cat([grouped_points, grouped_xyz], dim=-1).to(points.dtype)
                else:
                    grouped_points = grouped_xyz
        grouped_points = _apply_mlp(None if mlp_list is None else mlp_list[i], grouped_points, scope, f"conv{i}", bn, is_training, bn_decay)
        new_points_list.append(grouped_points.max(dim=2).values)
    return new_xyz, torch.cat(new_points_list, dim=-1)


def pointnet_fp_module(xyz1, xyz2, points1, points2, mlp=None, is_training=None, bn_decay=None, scope=None, bn=True, fused=True,
                       lengths=None):
    ''' PointNet Feature Propogation (FP) Module — same positional arguments as the reference
        (utils/pointnet_util.py:199-229).
        xyz1 (b,n1,3) dense, xyz2 (b,n2,3) sparser, points1 (b,n1,c1) or None, points2 (b,n2,c2);
        mlp: list of output widths (scope registry), a callable on a (b,n1,1,channel) tensor, or None.
        lengths: optional (b,) integers: cloud i of the dense level is xyz1[i, :lengths[i]] (and points1[i, :lengths[i]]),
        padded to n1; xyz2 / points2 stay dense.  Real rows are what the call without lengths computes for them (the
        batch norm statistics of the mlp come from the real rows only); padding rows are never read and come out 0.
        With lengths, mlp must be a list of widths or a layers.SharedMLP (it takes the row mask); another callable
        raises ValueError.
        Inside layers.batch_invariant() (eval-mode batch norms, grad mode off, CUDA) a SharedMLP tail runs with the
        interpolation and the concat in one kernel (layers.fp_mlp), with or without lengths.
        Return: new_points (b,n1,mlp[-1]) (or (b,n1,c2+c1) when mlp is None)
    '''
    mask = None
    if lengths is not None:
        if mlp is not None and callable(mlp) and not isinstance(mlp, layers.SharedMLP):
            raise ValueError("pointnet_fp_module with lengths needs mlp as a list of widths or a layers.SharedMLP "
                             "(the batch norm must see the row mask)")
        b, n = xyz1.shape[0], xyz1.shape[1]
        lengths = device_lengths(lengths, b, n, xyz1.device, "pointnet_fp_module")
        mask = layers.row_mask(lengths, n)
    tail = _fp_mlp_route(mlp, xyz1, points1, points2, scope, bn, is_training, bn_decay) if mlp is not None else None
    if tail is not None:
        # batch-invariant inference: interpolation, concat and every layer in the row kernel behind layers.fp_mlp
        return layers._invariant_call(layers.fp_mlp, xyz1, xyz2, points1, points2, tail, lengths=lengths)
    no_grad = not points2.requires_grad and (points1 is None or not points1.requires_grad)
    same_dtype = points1 is None or points1.dtype == points2.dtype
    if fused and no_grad and same_dtype and points2.shape[2] > 0:
        # one kernel: 3-NN, weights, interpolation and the concat of :219
        new_points1 = fp_interpolate_concat(xyz1, xyz2, points1, points2, lengths=lengths)
    else:
        if fused and not points2.requires_grad:
            interpolated_points = three_nn_interpolate(xyz1, xyz2, points2, lengths=lengths)
        else:
            dist, idx = three_nn(xyz1, xyz2, lengths=lengths)
            dist = torch.clamp(dist, min=1e-10)
            norm = (1.0 / dist).sum(dim=2, keepdim=True)
            # with lengths, the padding rows' weights are NaN (1/inf = 0, then 0/0): three_interpolate never reads them
            weight = (1.0 / dist) / norm
            interpolated_points = three_interpolate(points2, idx, weight, lengths=lengths)
        if points1 is not None:
            if mask is not None:
                points1 = torch.where(mask.unsqueeze(2), points1, 0)  # padding rows are 0, as the fused kernel writes them
            new_points1 = torch.cat([interpolated_points, points1], dim=2)  # B,ndataset1,nchannel1+nchannel2
        else:
            new_points1 = interpolated_points
    if mlp is not None:
        new_points1 = _apply_mlp(mlp, new_points1.unsqueeze(2), scope, "conv", bn, is_training, bn_decay,
                                 mask=None if mask is None else mask.unsqueeze(2)).squeeze(2)
    return new_points1
