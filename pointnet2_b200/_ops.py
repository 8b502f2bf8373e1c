"""The library's launch sequences as torch operators (namespace ``pn2``), so that torch.compile and torch.export see
every geometry op, fused batch norm and fused MLP as one node of the graph instead of a graph break.

Each operator's real implementation is the launch helper the eager wrapper calls (tf_sampling.fps_launch, ...), so
there is one copy of every launch sequence.  The public functions keep their argument checks and call
``torch.ops.pn2.*`` only while ``torch.compiler.is_compiling()``; in eager mode they launch directly, through their
own autograd Functions, without the dispatcher's per-call host cost.

Registering the operators loads nothing: the fake implementations below are shape arithmetic on symbolic sizes, and
the library is opened by the first real launch.

Encodings a schema needs:
* an absent optional output (grouped_xyz when not wanted, sample_knn's dist, an absent gradient) is an empty tensor,
  mapped back to None by the caller;
* the masked batch-norm operators are functional: they return the updated running statistics, which the wrapper
  copies into the module's buffers (a registered operator cannot both mutate its inputs and carry an autograd formula);
* a SharedMLP is passed as its tensors, six per layer (see layers._stack_params), with the epsilons and ReLU flags.
"""
from __future__ import annotations

from typing import List, Optional, Tuple

import torch
from torch import Tensor

from . import layers, pointnet_util, sa_layer, tf_grouping, tf_interpolate, tf_sampling

I32, F32 = torch.int32, torch.float32


def _op(name: str):
    return torch.library.custom_op(f"pn2::{name}", mutates_args=())


def _none(t: Optional[Tensor], dtype=F32, like: Optional[Tensor] = None) -> Tensor:
    """t, or the empty tensor that stands for an absent one"""
    if t is not None:
        return t
    return like.new_empty((0,), dtype=dtype)


# ---- sampling -------------------------------------------------------------------------------------------------------
@_op("farthest_point_sample")
def farthest_point_sample(npoint: int, inp: Tensor, lengths: Optional[Tensor]) -> Tensor:
    return tf_sampling.fps_launch(npoint, inp, lengths)


@farthest_point_sample.register_fake
def _(npoint, inp, lengths):
    return inp.new_empty((inp.shape[0], npoint), dtype=I32)


@_op("farthest_point_sample_and_gather")
def farthest_point_sample_and_gather(npoint: int, inp: Tensor, lengths: Optional[Tensor]) -> Tuple[Tensor, Tensor]:
    return tf_sampling.fps_gather_launch(npoint, inp, lengths)


@farthest_point_sample_and_gather.register_fake
def _(npoint, inp, lengths):
    return inp.new_empty((inp.shape[0], npoint), dtype=I32), inp.new_empty((inp.shape[0], npoint, 3))


@_op("prob_sample")
def prob_sample(inp: Tensor, inpr: Tensor) -> Tensor:
    return tf_sampling.prob_sample_launch(inp, inpr)


@prob_sample.register_fake
def _(inp, inpr):
    return inp.new_empty((inp.shape[0], inpr.shape[1]), dtype=I32)


@_op("gather_point")
def gather_point(inp: Tensor, idx: Tensor) -> Tensor:
    return tf_sampling.gather_point_launch(inp, idx)


@gather_point.register_fake
def _(inp, idx):
    return inp.new_empty((inp.shape[0], idx.shape[1], 3))


@_op("gather_point_grad")
def gather_point_grad(out_g: Tensor, idx: Tensor, n: int) -> Tensor:
    """float atomics, or ordered sums when torch.are_deterministic_algorithms_enabled() as the op runs"""
    return tf_sampling.gather_point_grad_launch(out_g, idx, n)


@gather_point_grad.register_fake
def _(out_g, idx, n):
    return out_g.new_empty((idx.shape[0], n, 3), dtype=F32)


def _gather_point_setup(ctx, inputs, output):
    inp, idx = inputs
    ctx.save_for_backward(idx)
    ctx.n = inp.shape[1]


def _gather_point_backward(ctx, out_g):
    (idx,) = ctx.saved_tensors
    return torch.ops.pn2.gather_point_grad(out_g.contiguous(), idx, ctx.n), None


gather_point.register_autograd(_gather_point_backward, setup_context=_gather_point_setup)


# ---- grouping -------------------------------------------------------------------------------------------------------
@_op("query_ball_point")
def query_ball_point(radius: float, nsample: int, xyz1: Tensor, xyz2: Tensor,
                     lengths: Optional[Tensor]) -> Tuple[Tensor, Tensor]:
    return tf_grouping.query_ball_point_launch(radius, nsample, xyz1, xyz2, lengths)


@query_ball_point.register_fake
def _(radius, nsample, xyz1, xyz2, lengths):
    b, m = xyz2.shape[0], xyz2.shape[1]
    return xyz1.new_empty((b, m, nsample), dtype=I32), xyz1.new_empty((b, m), dtype=I32)


@_op("select_top_k")
def select_top_k(k: int, dist: Tensor) -> Tuple[Tensor, Tensor]:
    return tf_grouping.select_top_k_launch(k, dist)


@select_top_k.register_fake
def _(k, dist):
    return dist.new_empty(dist.shape, dtype=I32), dist.new_empty(dist.shape)


@_op("group_point")
def group_point(points: Tensor, idx: Tensor) -> Tensor:
    return tf_grouping.group_point_launch(points, idx)


@group_point.register_fake
def _(points, idx):
    return points.new_empty((idx.shape[0], idx.shape[1], idx.shape[2], points.shape[2]))


@_op("group_point_grad")
def group_point_grad(grad_out: Tensor, idx: Tensor, n: int) -> Tensor:
    """float atomics, or ordered sums when torch.are_deterministic_algorithms_enabled() as the op runs"""
    return tf_grouping.group_point_grad(grad_out, idx, (idx.shape[0], n, grad_out.shape[-1]))


@group_point_grad.register_fake
def _(grad_out, idx, n):
    return grad_out.new_empty((idx.shape[0], n, grad_out.shape[-1]))


def _group_point_setup(ctx, inputs, output):
    points, idx = inputs
    ctx.save_for_backward(idx)
    ctx.n, ctx.dtype = points.shape[1], points.dtype


def _group_point_backward(ctx, grad):
    (idx,) = ctx.saved_tensors
    return torch.ops.pn2.group_point_grad(grad.to(ctx.dtype).contiguous(), idx, ctx.n), None


group_point.register_autograd(_group_point_backward, setup_context=_group_point_setup)


@_op("knn_point")
def knn_point(k: int, xyz1: Tensor, xyz2: Tensor, lengths: Optional[Tensor],
              query_lengths: Optional[Tensor]) -> Tuple[Tensor, Tensor]:
    return tf_grouping.knn_point_launch(k, xyz1, xyz2, lengths, query_lengths)


@knn_point.register_fake
def _(k, xyz1, xyz2, lengths, query_lengths):
    b, m = xyz2.shape[0], xyz2.shape[1]
    return xyz1.new_empty((b, m, k)), xyz1.new_empty((b, m, k), dtype=I32)


# ---- interpolation --------------------------------------------------------------------------------------------------
@_op("three_nn")
def three_nn(xyz1: Tensor, xyz2: Tensor, lengths: Optional[Tensor]) -> Tuple[Tensor, Tensor]:
    return tf_interpolate.three_nn_launch(xyz1, xyz2, lengths)


@three_nn.register_fake
def _(xyz1, xyz2, lengths):
    b, n = xyz1.shape[0], xyz1.shape[1]
    return xyz1.new_empty((b, n, 3)), xyz1.new_empty((b, n, 3), dtype=I32)


@_op("three_interpolate")
def three_interpolate(points: Tensor, idx: Tensor, weight: Tensor, lengths: Optional[Tensor]) -> Tensor:
    return tf_interpolate.three_interpolate_launch(points, idx, weight, lengths)


@three_interpolate.register_fake
def _(points, idx, weight, lengths):
    return points.new_empty((points.shape[0], idx.shape[1], points.shape[2]))


@_op("three_interpolate_grad")
def three_interpolate_grad(grad_out: Tensor, idx: Tensor, weight: Tensor, lengths: Optional[Tensor], m: int) -> Tensor:
    """the path (tf_interpolate.DETERMINISTIC_GRAD, torch.are_deterministic_algorithms_enabled()) is chosen as the op
    runs"""
    return tf_interpolate.three_interpolate_grad_launch(grad_out, idx, weight, lengths, m)


@three_interpolate_grad.register_fake
def _(grad_out, idx, weight, lengths, m):
    return grad_out.new_empty((grad_out.shape[0], m, grad_out.shape[2]))


def _three_interpolate_setup(ctx, inputs, output):
    points, idx, weight, lengths = inputs
    ctx.save_for_backward(idx, weight, lengths)
    ctx.m, ctx.dtype = points.shape[1], points.dtype


def _three_interpolate_backward(ctx, grad):
    idx, weight, lengths = ctx.saved_tensors
    g = torch.ops.pn2.three_interpolate_grad(grad.to(ctx.dtype).contiguous(), idx, weight, lengths, ctx.m)
    return g, None, None, None


three_interpolate.register_autograd(_three_interpolate_backward, setup_context=_three_interpolate_setup)


@_op("three_nn_interpolate")
def three_nn_interpolate(xyz1: Tensor, xyz2: Tensor, points2: Tensor, lengths: Optional[Tensor],
                         return_aux: bool) -> Tuple[Tensor, Tensor, Tensor, Tensor]:
    out, dist, idx, weight = tf_interpolate.three_nn_interpolate_launch(xyz1, xyz2, points2, lengths, return_aux)
    return out, _none(dist, F32, xyz1), _none(idx, I32, xyz1), _none(weight, F32, xyz1)


@three_nn_interpolate.register_fake
def _(xyz1, xyz2, points2, lengths, return_aux):
    b, n = xyz1.shape[0], xyz1.shape[1]
    aux = (b, n, 3) if return_aux else (0,)
    return (points2.new_empty((b, n, points2.shape[2])), xyz1.new_empty(aux), xyz1.new_empty(aux, dtype=I32),
            xyz1.new_empty(aux))


@_op("fp_interpolate_concat")
def fp_interpolate_concat(xyz1: Tensor, xyz2: Tensor, points1: Optional[Tensor], points2: Tensor,
                          lengths: Optional[Tensor]) -> Tensor:
    return tf_interpolate.fp_interpolate_concat_launch(xyz1, xyz2, points1, points2, lengths)


@fp_interpolate_concat.register_fake
def _(xyz1, xyz2, points1, points2, lengths):
    c1 = 0 if points1 is None else points1.shape[2]
    return points2.new_empty((xyz1.shape[0], xyz1.shape[1], points2.shape[2] + c1))


# ---- set-abstraction layers -----------------------------------------------------------------------------------------
@_op("sample_group")
def sample_group(npoint: int, radius: float, nsample: int, xyz: Tensor, center: bool, want_grouped: bool,
                 lengths: Optional[Tensor]) -> Tuple[Tensor, Tensor, Tensor, Tensor, Tensor]:
    *res, grouped = sa_layer.sample_group_launch(npoint, radius, nsample, xyz, center, want_grouped, lengths)
    return (*res, _none(grouped, F32, xyz))


@sample_group.register_fake
def _(npoint, radius, nsample, xyz, center, want_grouped, lengths):
    b = xyz.shape[0]
    return (xyz.new_empty((b, npoint), dtype=I32), xyz.new_empty((b, npoint, 3)),
            xyz.new_empty((b, npoint, nsample), dtype=I32), xyz.new_empty((b, npoint), dtype=I32),
            xyz.new_empty((b, npoint, nsample, 3) if want_grouped else (0,)))


@_op("sample_group_msg")
def sample_group_msg(npoint: int, radius_list: List[float], nsample_list: List[int], xyz: Tensor, center: bool,
                     want_grouped: bool, lengths: Optional[Tensor]
                     ) -> Tuple[Tensor, Tensor, List[Tensor], List[Tensor], List[Tensor]]:
    fps_idx, new_xyz, idx, cnt, grouped = sa_layer.sample_group_msg_launch(npoint, radius_list, nsample_list, xyz, center,
                                                                           want_grouped, lengths)
    return fps_idx, new_xyz, idx, cnt, grouped if grouped is not None else []


@sample_group_msg.register_fake
def _(npoint, radius_list, nsample_list, xyz, center, want_grouped, lengths):
    b = xyz.shape[0]
    return (xyz.new_empty((b, npoint), dtype=I32), xyz.new_empty((b, npoint, 3)),
            [xyz.new_empty((b, npoint, s), dtype=I32) for s in nsample_list],
            [xyz.new_empty((b, npoint), dtype=I32) for _ in nsample_list],
            [xyz.new_empty((b, npoint, s, 3)) for s in nsample_list] if want_grouped else [])


@_op("sample_knn")
def sample_knn(npoint: int, k: int, xyz: Tensor, center: bool, want_grouped: bool, want_dist: bool,
               lengths: Optional[Tensor]) -> Tuple[Tensor, Tensor, Tensor, Tensor, Tensor]:
    fps_idx, new_xyz, idx, dist, grouped = sa_layer.sample_knn_launch(npoint, k, xyz, center, want_grouped, want_dist,
                                                                      lengths)
    return fps_idx, new_xyz, idx, _none(dist, F32, xyz), _none(grouped, F32, xyz)


@sample_knn.register_fake
def _(npoint, k, xyz, center, want_grouped, want_dist, lengths):
    b = xyz.shape[0]
    return (xyz.new_empty((b, npoint), dtype=I32), xyz.new_empty((b, npoint, 3)), xyz.new_empty((b, npoint, k), dtype=I32),
            xyz.new_empty((b, npoint, k) if want_dist else (0,)),
            xyz.new_empty((b, npoint, k, 3) if want_grouped else (0,)))


@_op("ball_group")
def ball_group(radius: float, nsample: int, xyz1: Tensor, xyz2: Tensor, center: bool,
               want_grouped: bool) -> Tuple[Tensor, Tensor, Tensor]:
    idx, cnt, g = sa_layer.ball_group_launch(radius, nsample, xyz1, xyz2, center, want_grouped)
    return idx, cnt, _none(g, F32, xyz1)


@ball_group.register_fake
def _(radius, nsample, xyz1, xyz2, center, want_grouped):
    b, m = xyz2.shape[0], xyz2.shape[1]
    return (xyz1.new_empty((b, m, nsample), dtype=I32), xyz1.new_empty((b, m), dtype=I32),
            xyz1.new_empty((b, m, nsample, 3) if want_grouped else (0,)))


@_op("group_and_concat")
def group_and_concat(xyz: Tensor, new_xyz: Tensor, points: Optional[Tensor], idx: Tensor,
                     xyz_first: bool) -> Tuple[Tensor, Tensor]:
    return pointnet_util.group_and_concat_launch(xyz, new_xyz, points, idx, xyz_first)


@group_and_concat.register_fake
def _(xyz, new_xyz, points, idx, xyz_first):
    b, m, s = idx.shape
    c = 0 if points is None else points.shape[2]
    dtype = F32 if points is None else points.dtype
    return xyz.new_empty((b, m, s, 3 + c), dtype=dtype), xyz.new_empty((b, m, s, 3))


@_op("group_and_concat_backward")
def group_and_concat_backward(g_out: Tensor, g_gxyz: Optional[Tensor], idx: Tensor, n: int, xyz_first: bool,
                              has_points: bool, need_xyz: bool, need_new_xyz: bool) -> Tuple[Tensor, Tensor, Tensor]:
    g_xyz, g_new_xyz, g_points = pointnet_util.group_and_concat_backward(g_out, g_gxyz, idx, n, xyz_first, has_points,
                                                                         need_xyz, need_new_xyz)
    return _none(g_xyz, F32, g_out), _none(g_new_xyz, F32, g_out), _none(g_points, g_out.dtype, g_out)


@group_and_concat_backward.register_fake
def _(g_out, g_gxyz, idx, n, xyz_first, has_points, need_xyz, need_new_xyz):
    b, m, s, c3 = g_out.shape
    return (g_out.new_empty((b, n, 3) if need_xyz else (0,), dtype=F32),
            g_out.new_empty((b, m, 3) if need_new_xyz else (0,), dtype=F32),
            g_out.new_empty((b, n, c3 - 3) if has_points else (0,)))


def _group_and_concat_setup(ctx, inputs, output):
    xyz, new_xyz, points, idx, xyz_first = inputs
    ctx.save_for_backward(idx)
    ctx.n, ctx.xyz_first, ctx.has_points = xyz.shape[1], xyz_first, points is not None
    ctx.dtype = F32 if points is None else points.dtype


def _group_and_concat_backward(ctx, g_out, g_gxyz):
    (idx,) = ctx.saved_tensors
    need_xyz, need_new_xyz = ctx.needs_input_grad[0], ctx.needs_input_grad[1]
    g_xyz, g_new_xyz, g_points = torch.ops.pn2.group_and_concat_backward(
        g_out.to(ctx.dtype).contiguous(), g_gxyz, idx, ctx.n, ctx.xyz_first, ctx.has_points, need_xyz, need_new_xyz)
    return (g_xyz if need_xyz else None, g_new_xyz if need_new_xyz else None, g_points if ctx.has_points else None,
            None, None)


group_and_concat.register_autograd(_group_and_concat_backward, setup_context=_group_and_concat_setup)


# ---- masked batch norm ----------------------------------------------------------------------------------------------
def _stats_copies(nbt, running_mean, running_var):
    """private copies of the running statistics for the kernel to update"""
    return tuple(None if t is None else t.clone() for t in (nbt, running_mean, running_var))


def _stats_out(x, nbt, rm, rv):
    """the updated (running_mean, running_var, num_batches_tracked), empty when the module keeps none"""
    return _none(rm, F32, x), _none(rv, F32, x), _none(nbt, torch.int64, x)


def _stats_fake(x, running_mean, running_var, nbt):
    return (x.new_empty(running_mean.shape if running_mean is not None else (0,), dtype=F32),
            x.new_empty(running_var.shape if running_var is not None else (0,), dtype=F32),
            x.new_empty(nbt.shape if nbt is not None else (0,), dtype=torch.int64))


@_op("masked_batch_norm_relu")
def masked_batch_norm_relu(x: Tensor, weight: Optional[Tensor], bias: Optional[Tensor], keep: Tensor,
                           running_mean: Optional[Tensor], running_var: Optional[Tensor],
                           num_batches_tracked: Optional[Tensor], eps: float, momentum: float
                           ) -> Tuple[Tensor, Tensor, Tensor, Tensor, Tensor, Tensor]:
    """(y, save_mean, save_invstd, running_mean', running_var', num_batches_tracked')"""
    nbt, rm, rv = _stats_copies(num_batches_tracked, running_mean, running_var)
    y, save_mean, save_invstd = layers.masked_bn_relu_forward_launch(x, weight, bias, keep, eps, momentum, nbt, rm, rv)
    return (y, save_mean, save_invstd, *_stats_out(x, nbt, rm, rv))


@masked_batch_norm_relu.register_fake
def _(x, weight, bias, keep, running_mean, running_var, num_batches_tracked, eps, momentum):
    c = x.shape[1]
    return (torch.empty_like(x), x.new_empty((c,), dtype=F32), x.new_empty((c,), dtype=F32),
            *_stats_fake(x, running_mean, running_var, num_batches_tracked))


@_op("masked_batch_norm_relu_backward")
def masked_batch_norm_relu_backward(dy: Tensor, x: Tensor, y: Tensor, keep: Tensor, weight: Optional[Tensor],
                                    save_mean: Tensor, save_invstd: Tensor) -> Tuple[Tensor, Tensor, Tensor]:
    dx, dgamma, dbeta = layers.masked_bn_relu_backward_launch(dy, x, y, keep, weight, save_mean, save_invstd)
    return dx, _none(dgamma, F32, x), _none(dbeta, F32, x)


@masked_batch_norm_relu_backward.register_fake
def _(dy, x, y, keep, weight, save_mean, save_invstd):
    c = (x.shape[1],) if weight is not None else (0,)
    return torch.empty_like(x), x.new_empty(c, dtype=F32), x.new_empty(c, dtype=F32)


def _masked_bn_setup(ctx, inputs, output):
    x, weight, bias, keep = inputs[:4]
    y, save_mean, save_invstd = output[:3]
    ctx.save_for_backward(x, y, keep, weight, save_mean, save_invstd)


def _masked_bn_backward(ctx, dy, *_):
    x, y, keep, weight, save_mean, save_invstd = ctx.saved_tensors
    dx, dgamma, dbeta = torch.ops.pn2.masked_batch_norm_relu_backward(dy.to(x.dtype).contiguous(), x, y, keep, weight,
                                                                      save_mean, save_invstd)
    affine = weight is not None
    return dx, dgamma if affine else None, dbeta if affine else None, None, None, None, None, None, None


masked_batch_norm_relu.register_autograd(_masked_bn_backward, setup_context=_masked_bn_setup)


@_op("masked_bn_relu_max")
def masked_bn_relu_max(x: Tensor, weight: Optional[Tensor], bias: Optional[Tensor], keep: Tensor,
                       running_mean: Optional[Tensor], running_var: Optional[Tensor], num_batches_tracked: Optional[Tensor],
                       eps: float, momentum: float) -> Tuple[Tensor, Tensor, Tensor, Tensor, Tensor, Tensor, Tensor]:
    """x (B, N, C): (out, argmax, save_mean, save_invstd, running_mean', running_var', num_batches_tracked')"""
    b, n, c = x.shape
    nbt, rm, rv = _stats_copies(num_batches_tracked, running_mean, running_var)
    out, argmax, save_mean, save_invstd = layers.masked_bn_relu_max_forward_launch(x.reshape(b * n, c), weight, bias, keep,
                                                                                  eps, momentum, nbt, rm, rv, b, n)
    return (out, argmax, save_mean, save_invstd, *_stats_out(x, nbt, rm, rv))


@masked_bn_relu_max.register_fake
def _(x, weight, bias, keep, running_mean, running_var, num_batches_tracked, eps, momentum):
    b, _, c = x.shape
    return (x.new_empty((b, c)), x.new_empty((b, c), dtype=I32), x.new_empty((c,), dtype=F32),
            x.new_empty((c,), dtype=F32), *_stats_fake(x, running_mean, running_var, num_batches_tracked))


@_op("masked_bn_relu_max_backward")
def masked_bn_relu_max_backward(dout: Tensor, x: Tensor, out: Tensor, argmax: Tensor, keep: Tensor,
                                weight: Optional[Tensor], save_mean: Tensor,
                                save_invstd: Tensor) -> Tuple[Tensor, Tensor, Tensor]:
    b, n, c = x.shape
    dx, dgamma, dbeta = layers.masked_bn_relu_max_backward_launch(dout, x.reshape(b * n, c), out, argmax, keep, weight,
                                                                  save_mean, save_invstd)
    return dx.view(b, n, c), _none(dgamma, F32, x), _none(dbeta, F32, x)


@masked_bn_relu_max_backward.register_fake
def _(dout, x, out, argmax, keep, weight, save_mean, save_invstd):
    c = (x.shape[2],) if weight is not None else (0,)
    return torch.empty_like(x), x.new_empty(c, dtype=F32), x.new_empty(c, dtype=F32)


def _masked_max_setup(ctx, inputs, output):
    x, weight, bias, keep = inputs[:4]
    out, argmax, save_mean, save_invstd = output[:4]
    ctx.save_for_backward(x, out, argmax, keep, weight, save_mean, save_invstd)
    ctx.mark_non_differentiable(argmax)


def _masked_max_backward(ctx, dout, *_):
    x, out, argmax, keep, weight, save_mean, save_invstd = ctx.saved_tensors
    dx, dgamma, dbeta = torch.ops.pn2.masked_bn_relu_max_backward(dout.to(x.dtype).contiguous(), x, out, argmax, keep,
                                                                  weight, save_mean, save_invstd)
    affine = weight is not None
    return dx, dgamma if affine else None, dbeta if affine else None, None, None, None, None, None, None


masked_bn_relu_max.register_autograd(_masked_max_backward, setup_context=_masked_max_setup)


# ---- fused inference MLPs -------------------------------------------------------------------------------------------
@_op("sa_mlp_max")
def sa_mlp_max(xyz: Optional[Tensor], new_xyz: Optional[Tensor], points: Optional[Tensor], idx: Optional[Tensor],
               lengths: Optional[Tensor], params: List[Optional[Tensor]], eps: List[float], relu: List[bool],
               xyz_first: bool, use_xyz: bool, dtype: torch.dtype) -> Tensor:
    """``params``: six tensors per layer (layers._stack_params); idx None is the whole-cloud form"""
    return layers.sa_mlp_max_launch(xyz, new_xyz, points, idx, lengths, params, eps, relu, xyz_first, use_xyz, dtype)


@sa_mlp_max.register_fake
def _(xyz, new_xyz, points, idx, lengths, params, eps, relu, xyz_first, use_xyz, dtype):
    ref = xyz if xyz is not None else points
    s = 1 if idx is None else idx.shape[1]
    return ref.new_empty((ref.shape[0], s, params[-6].shape[0]), dtype=dtype)


@_op("fp_mlp")
def fp_mlp(xyz1: Tensor, xyz2: Tensor, points1: Optional[Tensor], points2: Tensor, lengths: Optional[Tensor],
           params: List[Optional[Tensor]], eps: List[float], relu: List[bool], dtype: torch.dtype) -> Tensor:
    return layers.fp_mlp_launch(xyz1, xyz2, points1, points2, lengths, params, eps, relu, dtype)


@fp_mlp.register_fake
def _(xyz1, xyz2, points1, points2, lengths, params, eps, relu, dtype):
    return xyz1.new_empty((xyz1.shape[0], xyz1.shape[1], params[-6].shape[0]), dtype=dtype)


@_op("mlp_rows")
def mlp_rows(t: Tensor, mask: Optional[Tensor], params: List[Optional[Tensor]], eps: List[float], relu: List[bool],
             dtype: torch.dtype) -> Tensor:
    return layers.mlp_rows_launch(t, mask, params, eps, relu, dtype)


@mlp_rows.register_fake
def _(t, mask, params, eps, relu, dtype):
    return t.new_empty((*t.shape[:-1], params[-6].shape[0]), dtype=dtype)


OPS = ("farthest_point_sample", "farthest_point_sample_and_gather", "prob_sample", "gather_point", "gather_point_grad",
       "query_ball_point", "select_top_k", "group_point", "group_point_grad", "knn_point", "three_nn",
       "three_interpolate", "three_interpolate_grad", "three_nn_interpolate", "fp_interpolate_concat", "sample_group",
       "sample_group_msg", "sample_knn", "ball_group", "group_and_concat", "group_and_concat_backward",
       "masked_batch_norm_relu", "masked_batch_norm_relu_backward", "masked_bn_relu_max", "masked_bn_relu_max_backward",
       "sa_mlp_max", "fp_mlp", "mlp_rows")
