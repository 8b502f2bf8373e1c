"""Learned 1x1-conv stacks and the variable-scope registry behind the reference-form module calls.

The reference builds every learned layer as a 1x1 convolution + batch norm + ReLU on a channels-last
tensor (tf_util.conv2d called from utils/pointnet_util.py:115-121,146-152,187-190,221-226) and finds
its variables by TensorFlow variable scope (``scope='layer1'`` ...).  On a channels-last tensor a 1x1
convolution is a matrix product over the last axis, so ``SharedMLP`` is Linear + BatchNorm1d + ReLU over
the flattened leading axes.  In training that is cuBLAS and torch's batch norm (plus the masked batch norm kernel for
padded batches); at inference the stack of a set-abstraction level runs inside ``sa_mlp_max``, one CUDA kernel that
gathers the groups, applies every layer with the batch norm's running statistics and max-pools (csrc/sa_mlp.cu).
Inside ``batch_invariant()`` the feature-propagation tails and every other eval-mode stack run through the row-wise
twin of that kernel (``fp_mlp``, ``mlp_rows``; csrc/fp_mlp.cu), so that no learned layer's result depends on the batch.

``scoped_mlp`` is the registry that lets the reference's own call form run unchanged::

    l1_xyz, l1_points, l1_indices = pointnet_sa_module(l0_xyz, l0_points, npoint=1024, radius=0.1, nsample=32,
        mlp=[32,32,64], mlp2=None, group_all=False, is_training=is_training, bn_decay=bn_decay, scope='layer1')

(models/pointnet2_sem_seg.py:28): the first call under a scope creates the layers (xavier weights, zero
bias, as tf_util does) on the input's device, later calls reuse them; ``scope_parameters()`` hands them to
an optimiser, ``reset_scopes()`` is ``tf.reset_default_graph()``.
"""
from __future__ import annotations

import contextlib
import ctypes
import math
from typing import Dict, Optional, Sequence

import torch
from torch import nn
from torch.autograd.function import once_differentiable

from . import _lib
from ._tensor import DTYPE_CODES, FEATURE_DTYPES, device_lengths, on_device, ptr, require_cuda, same_device, stream_ptr


# tf_util.batch_norm_template calls tf.contrib.layers.batch_norm without an epsilon, so the reference normalises with
# its default 1e-3, not torch's 1e-5.  It matters where the pre-BN variance is small: at sa1 of the sem-seg net (radius
# 0.1) it is a few 1e-4 at init.
BN_EPS = 1e-3


class SharedMLP(nn.Module):
    """conv2d(1x1)+BN+ReLU stack on (..., C) tensors — tf_util.conv2d with xavier weights, zero bias, and the
    reference's batch-norm epsilon (BN_EPS).  Calling it runs the torch layers; the set-abstraction modules hand an
    eval-mode stack to ``sa_mlp_max`` instead when ``sa_mlp_applies`` (no grad mode, CUDA, max-pooling), which reads
    these same parameters and buffers on every call.  Inside ``batch_invariant()`` a call that ``invariant_applies`` to
    runs through ``mlp_rows``."""

    def __init__(self, in_channels: int, widths: Sequence[int], bn: bool = True, last_activation: bool = True):
        super().__init__()
        layers = []
        c = int(in_channels)
        for i, w in enumerate(widths):
            lin = nn.Linear(c, int(w))
            nn.init.xavier_uniform_(lin.weight)
            nn.init.zeros_(lin.bias)
            layers.append(lin)
            act = last_activation or i + 1 < len(widths)
            if bn and act:
                layers.append(nn.BatchNorm1d(int(w), eps=BN_EPS))
            if act:
                layers.append(nn.ReLU(inplace=True))
            c = int(w)
        self.body = nn.Sequential(*layers)
        self.in_channels, self.out_channels = int(in_channels), c

    def forward(self, t: torch.Tensor, mask: Optional[torch.Tensor] = None) -> torch.Tensor:
        """``mask``: optional bool tensor of t.shape[:-1] (or as many elements), True on the real rows of a padded batch
        (see row_mask).  Batch norm then takes its training statistics from the real rows only, and the padding rows of
        every layer's output are 0 (whatever t holds there, NaN included).  Without a mask: the plain stack."""
        if _BATCH_INVARIANT and invariant_applies(self, t):
            return _invariant_call(mlp_rows, t, self, mask)
        lead = t.shape[:-1]
        if mask is None:
            return self.body(t.reshape(-1, t.shape[-1])).reshape(*lead, self.out_channels)
        keep = mask.reshape(-1, 1)
        return _masked_layers(list(self.body), t.reshape(-1, t.shape[-1]), keep).reshape(*lead, self.out_channels)


def _masked_layers(mods, x: torch.Tensor, keep: torch.Tensor, fuse_last: bool = False) -> torch.Tensor:
    """The modules ``mods`` of a SharedMLP body on the rows of x (R, C) where keep (R, 1) is True: batch norms take
    their statistics from those rows, and every output's padding rows are 0.  fuse_last: mods ends with a Linear whose
    output goes straight to a fused op that reads no padding row (its padding rows are left as they come)."""
    # torch.where, not a multiply: NaN * 0 is NaN.  This one stays even before the fused op: NaN input rows would
    # reach the Linear's weight gradient through x^T dy.
    x = torch.where(keep, x, 0)
    i = 0
    while i < len(mods):
        mod = mods[i]
        if isinstance(mod, nn.BatchNorm1d):
            if _fuses_at(mods, i, x):
                # BatchNorm1d + the ReLU after it in the CUDA op, which reads no padding row and writes 0 there
                x = masked_batch_norm_relu(mod, x, keep.reshape(-1))
                i += 2
                continue
            x = torch.where(keep, masked_batch_norm(mod, x, keep), 0)
        elif isinstance(mod, nn.Linear):
            x = mod(x)
            if not (_fuses_at(mods, i + 1, x) or (fuse_last and i + 1 == len(mods))):
                x = torch.where(keep, x, 0)
        else:
            x = mod(x)  # ReLU keeps the zeros
        i += 1
    return x


def row_mask(lengths: torch.Tensor, n: int) -> torch.Tensor:
    """(b, n) bool, True on rows j < lengths[i] of a padded batch.  The lengths are clamped to [1, n], as the kernels
    clamp them, and never leave the device."""
    return torch.arange(n, device=lengths.device).unsqueeze(0) < lengths.clamp(1, n).unsqueeze(1)


def masked_batch_norm(bn: nn.BatchNorm1d, x: torch.Tensor, keep: torch.Tensor) -> torch.Tensor:
    """``bn`` on the rows of x (R, C) where keep (R, 1) is True.  Training mode: normalised with the mean and (biased)
    variance of those rows, and the running statistics are updated from them as BatchNorm1d would from a batch made of
    them alone (unbiased variance, momentum or the cumulative average, num_batches_tracked).  Eval mode: the running
    statistics, as bn itself.  The statistics are float32 for float32 and 16-bit x (as torch's batch norm keeps them
    under autocast) and float64 for float64 x; the result has x's dtype, and its padding rows are left for the caller to zero.  The padding rows of x
    must be 0 (the caller zeroes them), so the mean is a plain sum over every row.  The variance is a second pass over
    the centred real rows, not E[x^2] - mean^2, which cancels catastrophically once |mean| is large against the
    standard deviation.  The row count stays on the device: nothing synchronises with the host."""
    if not bn.training and bn.running_mean is not None:
        return bn(x)
    xf = x.to(torch.promote_types(x.dtype, torch.float32))  # float64 keeps float64
    cnt = keep.sum(dtype=xf.dtype)
    mean = xf.sum(0) / cnt
    centred = xf - mean
    d = torch.where(keep, centred, 0)
    var = (d * d).sum(0) / cnt
    scale = torch.rsqrt(var + bn.eps)
    if bn.affine:
        y = torch.addcmul(bn.bias, centred, scale * bn.weight)
    else:
        y = centred * scale
    if bn.track_running_stats and bn.running_mean is not None:
        with torch.no_grad():
            bn.num_batches_tracked.add_(1)
            f = 1.0 / bn.num_batches_tracked if bn.momentum is None else bn.momentum
            unbiased = var * cnt / torch.clamp(cnt - 1, min=1)
            bn.running_mean.mul_(1 - f).add_(mean * f)
            bn.running_var.mul_(1 - f).add_(unbiased * f)
    return y.to(x.dtype)


def _bn_tensors_misfit(bn: nn.BatchNorm1d, device) -> Optional[Exception]:
    """Why the kernels cannot take ``bn``'s own tensors (TypeError: dtype or layout, RuntimeError: device), or None: they
    read weight / bias and update the running statistics as contiguous float32 on x's device (num_batches_tracked
    int64), so a module converted with .half() or .to(torch.bfloat16), or left on another device, keeps the torch
    path."""
    tensors = [("weight", bn.weight, torch.float32), ("bias", bn.bias, torch.float32)] if bn.affine else []
    if bn.track_running_stats and bn.running_mean is not None:
        tensors += [("running_mean", bn.running_mean, torch.float32), ("running_var", bn.running_var, torch.float32),
                    ("num_batches_tracked", bn.num_batches_tracked, torch.int64)]
    for name, t, dtype in tensors:
        if t is None or t.dtype != dtype or not t.is_contiguous():
            got = "None" if t is None else f"{t.dtype}{'' if t.is_contiguous() else ' (not contiguous)'}"
            return TypeError(f"batch norm {name} must be a contiguous {dtype} tensor, got {got}")
        if t.device != device:
            return RuntimeError(f"batch norm {name} must be on x's device {device}, got device {t.device}")
    return None


def fused_bn_applies(bn: nn.BatchNorm1d, x: torch.Tensor) -> bool:
    """Whether SharedMLP(t, mask) runs ``bn`` + the ReLU after it through masked_batch_norm_relu: on CUDA, for float32 /
    bfloat16 / float16 x, wherever the torch path would compute batch statistics (training mode, or no running
    statistics), on a non-empty batch, with the module's parameters and buffers float32 on x's device.  Everything else
    (CPU, float64, eval with running statistics, a module converted to 16 bits) keeps masked_batch_norm."""
    return (x.is_cuda and x.dtype in FEATURE_DTYPES and x.shape[0] > 0
            and (bn.training or bn.running_mean is None) and _bn_tensors_misfit(bn, x.device) is None)


def _fuses_at(mods, i: int, x: torch.Tensor) -> bool:
    """mods[i] is a BatchNorm1d followed by a ReLU, and the pair runs through masked_batch_norm_relu"""
    return (i + 1 < len(mods) and isinstance(mods[i], nn.BatchNorm1d) and isinstance(mods[i + 1], nn.ReLU)
            and fused_bn_applies(mods[i], x))


def _bn_state(bn: nn.BatchNorm1d):
    """(eps, momentum, num_batches_tracked, running_mean, running_var) of ``bn`` as the masked batch-norm kernels take
    them: momentum -1 for the cumulative average, the three buffers None when bn keeps no running statistics."""
    tracking = bn.track_running_stats and bn.running_mean is not None
    return (float(bn.eps), -1.0 if bn.momentum is None else float(bn.momentum),
            *((bn.num_batches_tracked, bn.running_mean, bn.running_var) if tracking else (None, None, None)))


def masked_bn_relu_forward_launch(x, weight, bias, keep, eps: float, momentum: float, nbt, running_mean, running_var):
    """masked_batch_norm_relu's forward on x (R, C) and the uint8 keep (R,): (y, save_mean, save_invstd).  Adds 1 to
    ``nbt`` and updates the running statistics in place when they are given."""
    rows, c = x.shape
    dev = x.device
    y = torch.empty_like(x)
    save_mean = torch.empty(c, dtype=torch.float32, device=dev)
    save_invstd = torch.empty(c, dtype=torch.float32, device=dev)
    lib = _lib.load()
    with on_device(x):
        if nbt is not None:
            nbt.add_(1)  # on the device; the kernel reads it for the cumulative average
        wsb = int(lib.pn2_masked_bn_workspace_bytes(rows, c))
        ws = torch.empty(wsb, dtype=torch.uint8, device=dev)
        rc = lib.pn2_masked_bn_relu_forward_typed(
            DTYPE_CODES[x.dtype], rows, c, ptr(x), ptr(keep), ptr(weight), ptr(bias), eps, momentum, ptr(nbt),
            ptr(running_mean), ptr(running_var), ptr(y), ptr(save_mean), ptr(save_invstd), ptr(ws), wsb, stream_ptr(dev))
    _lib.check(rc, "pn2_masked_bn_relu_forward_typed")
    return y, save_mean, save_invstd


def masked_bn_relu_backward_launch(dy, x, y, keep, weight, save_mean, save_invstd):
    """masked_batch_norm_relu's backward from the contiguous dy in x's dtype: (dx, dgamma, dbeta), the last two None
    without weight."""
    rows, c = x.shape
    dev = x.device
    dx = torch.empty_like(x)
    dgamma = torch.empty(c, dtype=torch.float32, device=dev) if weight is not None else None
    dbeta = torch.empty(c, dtype=torch.float32, device=dev) if weight is not None else None
    lib = _lib.load()
    with on_device(x):
        wsb = int(lib.pn2_masked_bn_workspace_bytes(rows, c))
        ws = torch.empty(wsb, dtype=torch.uint8, device=dev)
        rc = lib.pn2_masked_bn_relu_backward_typed(
            DTYPE_CODES[x.dtype], rows, c, ptr(dy), ptr(x), ptr(y), ptr(keep), ptr(weight), ptr(save_mean),
            ptr(save_invstd), ptr(dx), ptr(dgamma), ptr(dbeta), ptr(ws), wsb, stream_ptr(dev))
    _lib.check(rc, "pn2_masked_bn_relu_backward_typed")
    return dx, dgamma, dbeta


class _MaskedBatchNormReLU(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, weight, bias, keep, bn):
        y, save_mean, save_invstd = masked_bn_relu_forward_launch(x, weight, bias, keep, *_bn_state(bn))
        ctx.save_for_backward(x, y, keep, weight, save_mean, save_invstd)
        return y

    @staticmethod
    @once_differentiable
    def backward(ctx, dy):
        x, y, keep, weight, save_mean, save_invstd = ctx.saved_tensors
        return (*masked_bn_relu_backward_launch(dy.to(x.dtype).contiguous(), x, y, keep, weight, save_mean, save_invstd),
                None, None)


def masked_batch_norm_relu(bn: nn.BatchNorm1d, x: torch.Tensor, keep: torch.Tensor) -> torch.Tensor:
    """relu(masked_batch_norm(bn, x, keep)) with its padding rows 0, as one CUDA op (csrc/masked_bn.cu) forward and
    backward.  ``x`` (R, C) float32 / bfloat16 / float16 on CUDA; ``keep`` (R,) bool, True on the real rows.  The
    statistics come from the real rows only (a two-pass per row group, merged with Chan's formula in a fixed order, in
    float32), the running statistics are updated as masked_batch_norm updates them, and the padding rows of x and of the
    incoming gradient are never read (they may be NaN).  Results are bit-identical from run to run; against the torch
    composition they differ by float32 rounding (the sums are ordered differently).  Nothing is read back to the host.
    For batch statistics only: in eval mode with running statistics it raises (that is ``bn(x)``).  ``bn``'s weight,
    bias and running buffers must be float32 on x's device."""
    if not (x.is_cuda and x.dtype in FEATURE_DTYPES):
        raise RuntimeError(f"masked_batch_norm_relu needs a float32/bfloat16/float16 CUDA tensor, got {x.dtype} on {x.device}")
    if x.dim() != 2 or x.shape[1] != bn.num_features:
        raise ValueError(f"masked_batch_norm_relu expects (rows, {bn.num_features}) x, got {tuple(x.shape)}")
    if not isinstance(keep, torch.Tensor) or keep.dtype != torch.bool or keep.numel() != x.shape[0]:
        raise ValueError(f"masked_batch_norm_relu expects a bool keep of {x.shape[0]} rows, got "
                         f"{getattr(keep, 'dtype', type(keep).__name__)} {tuple(getattr(keep, 'shape', ()))}")
    if keep.device != x.device:
        raise RuntimeError(f"keep must be on x's device ({x.device}), got {keep.device}")
    if not bn.training and bn.running_mean is not None:
        raise ValueError("masked_batch_norm_relu computes batch statistics; in eval mode with running statistics use bn(x)")
    misfit = _bn_tensors_misfit(bn, x.device)
    if misfit is not None:
        raise misfit
    x = x.contiguous()
    weight = bn.weight if bn.affine else None
    bias = bn.bias if bn.affine else None
    if torch.compiler.is_compiling():  # the mask as bytes by a cast: inductor cannot view bool as uint8
        eps, momentum, nbt, rm, rv = _bn_state(bn)
        y, _, _, *stats = torch.ops.pn2.masked_batch_norm_relu(x, weight, bias, keep.reshape(-1).to(torch.uint8), rm, rv,
                                                               nbt, eps, momentum)
        _write_back(stats, nbt, rm, rv)
        return y
    keep = keep.reshape(-1).contiguous().view(torch.uint8)  # the bool mask as bytes, no copy
    return _MaskedBatchNormReLU.apply(x, weight, bias, keep, bn)


def _write_back(stats, nbt, rm, rv) -> None:
    """Copy the running statistics a registered masked batch-norm op returns into the module's buffers: the op is
    functional so that it can carry an autograd formula, and this copy is the in-place update the eager kernel makes."""
    if nbt is not None:
        with torch.no_grad():
            for buf, new in zip((rm, rv, nbt), stats):
                buf.copy_(new)


def masked_bn_relu_max_forward_launch(x, weight, bias, keep, eps: float, momentum: float, nbt, running_mean, running_var,
                                      b: int, n: int):
    """masked_bn_relu_max's forward on x (b * n, C) and the uint8 keep (b * n,): (out, argmax, save_mean, save_invstd),
    the running statistics updated as masked_bn_relu_forward_launch updates them."""
    c = x.shape[1]
    dev = x.device
    out = torch.empty((b, c), dtype=x.dtype, device=dev)
    argmax = torch.empty((b, c), dtype=torch.int32, device=dev)
    save_mean = torch.empty(c, dtype=torch.float32, device=dev)
    save_invstd = torch.empty(c, dtype=torch.float32, device=dev)
    lib = _lib.load()
    with on_device(x):
        if nbt is not None:
            nbt.add_(1)  # on the device; the kernel reads it for the cumulative average
        wsb = int(lib.pn2_masked_bn_relu_max_workspace_bytes(b, n, c))
        ws = torch.empty(wsb, dtype=torch.uint8, device=dev)
        rc = lib.pn2_masked_bn_relu_max_forward_typed(
            DTYPE_CODES[x.dtype], b, n, c, ptr(x), ptr(keep), ptr(weight), ptr(bias), eps, momentum, ptr(nbt),
            ptr(running_mean), ptr(running_var), ptr(out), ptr(argmax), ptr(save_mean), ptr(save_invstd),
            ptr(ws), wsb, stream_ptr(dev))
    _lib.check(rc, "pn2_masked_bn_relu_max_forward_typed")
    return out, argmax, save_mean, save_invstd


def masked_bn_relu_max_backward_launch(dout, x, out, argmax, keep, weight, save_mean, save_invstd):
    """masked_bn_relu_max's backward from the contiguous dout (b, C) in x's dtype: (dx (b * n, C), dgamma, dbeta), the
    last two None without weight."""
    b, c = out.shape
    n = x.shape[0] // max(b, 1)
    dev = x.device
    dx = torch.empty_like(x)
    dgamma = torch.empty(c, dtype=torch.float32, device=dev) if weight is not None else None
    dbeta = torch.empty(c, dtype=torch.float32, device=dev) if weight is not None else None
    lib = _lib.load()
    with on_device(x):
        wsb = int(lib.pn2_masked_bn_relu_max_workspace_bytes(b, n, c))
        ws = torch.empty(wsb, dtype=torch.uint8, device=dev)
        rc = lib.pn2_masked_bn_relu_max_backward_typed(
            DTYPE_CODES[x.dtype], b, n, c, ptr(dout), ptr(x), ptr(out), ptr(argmax), ptr(keep), ptr(weight),
            ptr(save_mean), ptr(save_invstd), ptr(dx), ptr(dgamma), ptr(dbeta), ptr(ws), wsb, stream_ptr(dev))
    _lib.check(rc, "pn2_masked_bn_relu_max_backward_typed")
    return dx, dgamma, dbeta


class _MaskedBatchNormReLUMax(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, weight, bias, keep, bn, b, n):
        out, argmax, save_mean, save_invstd = masked_bn_relu_max_forward_launch(x, weight, bias, keep, *_bn_state(bn), b, n)
        ctx.save_for_backward(x, out, argmax, keep, weight, save_mean, save_invstd)
        ctx.mark_non_differentiable(argmax)
        return out, argmax

    @staticmethod
    @once_differentiable
    def backward(ctx, dout, _dargmax):
        x, out, argmax, keep, weight, save_mean, save_invstd = ctx.saved_tensors
        return (*masked_bn_relu_max_backward_launch(dout.to(x.dtype).contiguous(), x, out, argmax, keep, weight, save_mean,
                                                    save_invstd), None, None, None, None)


def masked_bn_relu_max(bn: nn.BatchNorm1d, x: torch.Tensor, lengths=None, *, with_indices: bool = False):
    """max over each cloud's real rows of relu(bn(x)), the batch norm taking its statistics from the real rows, as one
    CUDA op forward and backward (csrc/masked_bn.cu): the last layer of PointNet's point features and its max-pool
    (models/pointnet_cls_basic.py:46-53) on a padded batch.  ``x`` (B, N, C) float32 / bfloat16 / float16 on CUDA, the
    Linear output; ``lengths`` (B,) per-cloud row counts (see device_lengths; None: every row is real).  Returns (B, C)
    in x's dtype, and with ``with_indices`` also the (B, C) int32 row of each maximum: the FIRST row that reaches it,
    where TF's MaxPoolGrad sends the gradient.  The (B, N, C) ReLU output is never stored.

    The statistics, the running-statistics update and every value are bit-identical to masked_batch_norm_relu on the
    same rows followed by a max over the real rows (NaN wins, as in torch).  The padding rows of x are never read (they
    may be NaN).  Backward: the gradient reaches each maximum's row only, through the ReLU and the batch norm, with
    fixed-order sums and no float atomics, so it is bit-identical from run to run.  For batch statistics only, as
    masked_batch_norm_relu; CPU tensors raise RuntimeError."""
    if not (isinstance(x, torch.Tensor) and x.is_cuda and x.dtype in FEATURE_DTYPES):
        raise RuntimeError(f"masked_bn_relu_max needs a float32/bfloat16/float16 CUDA tensor, got "
                           f"{getattr(x, 'dtype', type(x).__name__)} on {getattr(x, 'device', '?')}")
    if x.dim() != 3 or x.shape[2] != bn.num_features:
        raise ValueError(f"masked_bn_relu_max expects (batch_size, num_point, {bn.num_features}) x, got {tuple(x.shape)}")
    if not bn.training and bn.running_mean is not None:
        raise ValueError("masked_bn_relu_max computes batch statistics; in eval mode with running statistics use bn(x)")
    misfit = _bn_tensors_misfit(bn, x.device)
    if misfit is not None:
        raise misfit
    b, n, c = x.shape
    if b * n >= 2 ** 31:
        raise ValueError(f"masked_bn_relu_max takes fewer than 2^31 rows, got {b} x {n}")
    lengths = device_lengths(lengths, b, n, x.device, "masked_bn_relu_max")
    if lengths is None:
        keep = torch.ones(b * n, dtype=torch.uint8, device=x.device)
    else:
        keep = row_mask(lengths, n).reshape(-1)
        # the bool mask as bytes: a view, no copy (a cast under compile: inductor cannot view bool as uint8)
        keep = keep.to(torch.uint8) if torch.compiler.is_compiling() else keep.view(torch.uint8)
    weight = bn.weight if bn.affine else None
    bias = bn.bias if bn.affine else None
    if b == 0:
        out = x.new_empty((0, c))
        return (out, torch.empty((0, c), dtype=torch.int32, device=x.device)) if with_indices else out
    if torch.compiler.is_compiling():
        eps, momentum, nbt, rm, rv = _bn_state(bn)
        out, argmax, _, _, *stats = torch.ops.pn2.masked_bn_relu_max(x.contiguous(), weight, bias, keep, rm, rv, nbt, eps,
                                                                     momentum)
        _write_back(stats, nbt, rm, rv)
    else:
        out, argmax = _MaskedBatchNormReLUMax.apply(x.reshape(b * n, c).contiguous(), weight, bias, keep, bn, b, n)
    return (out, argmax) if with_indices else out


def _first_max(y: torch.Tensor) -> torch.Tensor:
    """y (B, N, C) -> (B, C): the maximum over N (NaN wins, as in torch's max), its gradient going to the first row that
    reaches it only (TF's MaxPoolGrad), whatever the device"""
    m = y.amax(1, keepdim=True)
    hit = (y == m) | (torch.isnan(y) & torch.isnan(m))
    rows = torch.arange(y.shape[1], device=y.device).view(1, -1, 1)
    first = torch.where(hit, rows, y.shape[1]).amin(1, keepdim=True)
    return y.gather(1, first).squeeze(1)


def shared_mlp_max(mlp: "SharedMLP", t: torch.Tensor, lengths=None) -> torch.Tensor:
    """max over each cloud's real rows of mlp(t): t (B, N, C), ``lengths`` (B,) per-cloud row counts (None: every row
    is real; the padding rows are never read and may be NaN).  Returns (B, C_out).  The one place that routes
    "SharedMLP, then a whole-cloud max-pool":

    * training on CUDA: the earlier layers through SharedMLP's masked path, then the last Linear, then masked_bn_relu_max
      when its batch norm and ReLU fuse (fused_bn_applies);
    * eval under no_grad: sa_mlp_max(idx=None, lengths=...) when sa_mlp_applies, and inside batch_invariant() always (a
      stack the kernel cannot take raises RuntimeError there);
    * anything else (CPU, float64, grad mode in eval): the masked layers, the padding rows set to -inf, and a max whose
      gradient goes to the first maximal row."""
    if t.dim() != 3:
        raise ValueError(f"shared_mlp_max expects (batch_size, num_point, channels) t, got {tuple(t.shape)}")
    b, n = t.shape[0], t.shape[1]
    lengths = device_lengths(lengths, b, n, t.device, "shared_mlp_max")
    if t.is_cuda and not torch.is_grad_enabled():
        if _BATCH_INVARIANT and invariant_applies(mlp, t):
            return _invariant_call(sa_mlp_max, None, None, t, None, mlp, True, False, lengths=lengths)[:, 0]
        if sa_mlp_applies(mlp, t, t):
            return sa_mlp_max(None, None, t, None, mlp, True, False, lengths=lengths)[:, 0]
    mask = torch.ones(b, n, dtype=torch.bool, device=t.device) if lengths is None else row_mask(lengths, n)
    keep = mask.reshape(-1, 1)
    mods = list(mlp.body) if isinstance(mlp, SharedMLP) else []
    if (len(mods) >= 3 and isinstance(mods[-3], nn.Linear) and isinstance(mods[-2], nn.BatchNorm1d)
            and isinstance(mods[-1], nn.ReLU)):
        # the layers SharedMLP(t, mask) runs, split before the last batch norm, whose input may go to the fused op
        x = _masked_layers(mods[:-2], t.reshape(-1, t.shape[-1]), keep, fuse_last=True)
        if fused_bn_applies(mods[-2], x):
            return masked_bn_relu_max(mods[-2], x.reshape(b, n, -1), lengths)
        y = _masked_layers(mods[-2:], x, keep).reshape(b, n, -1)
    else:
        y = mlp(t, mask)
    return _first_max(torch.where(mask.unsqueeze(-1), y, float("-inf")))


SA_MLP_MAX_LAYERS = 4
SA_MLP_MAX_WIDTH = 1024  # of a layer's output; the first layer takes up to SA_MLP_MAX_WIDTH + 3 input channels
# Multiply-adds per grouped row (sum of C_in * C_out) up to which the modules take the kernel.  Above it the torch layers
# win: measured on an NVIDIA H100 80GB HBM3 at 700 W (DESIGN.md 6.13), [256, 512, 1024] on 259 inputs (721 K) runs 0.23-0.55 ms through cuBLAS and
# 1.1-1.3 ms fused, while [256, 256, 512] on 259 inputs (263 K) is faster fused.  A function of the widths alone, so
# that a level takes the same route, and gives the same bits, at every batch size.
SA_MLP_MAX_MACS = 300_000


def _mlp_stack(mlp):
    """The layers of a SharedMLP as [(Linear, BatchNorm1d or None, relu: bool)], or None when its body is not a sequence
    of Linear [+ BatchNorm1d] [+ ReLU]."""
    if not isinstance(mlp, SharedMLP):
        return None
    stack = []
    for mod in mlp.body:
        if isinstance(mod, nn.Linear):
            stack.append([mod, None, False])
        elif not stack or stack[-1][2]:
            return None
        elif isinstance(mod, nn.BatchNorm1d) and stack[-1][1] is None:
            stack[-1][1] = mod
        elif isinstance(mod, nn.ReLU):
            stack[-1][2] = True
        else:
            return None
    return [tuple(e) for e in stack] or None


def _linear_misfit(lin: nn.Linear, device) -> Optional[Exception]:
    """As _bn_tensors_misfit, for a Linear's weight and bias."""
    for name, t in (("weight", lin.weight), ("bias", lin.bias)):
        if t is None:
            continue
        if t.dtype != torch.float32 or not t.is_contiguous():
            return TypeError(f"linear {name} must be a contiguous torch.float32 tensor, got {t.dtype}"
                             f"{'' if t.is_contiguous() else ' (not contiguous)'}")
        if t.device != device:
            return RuntimeError(f"linear {name} must be on the inputs' device {device}, got device {t.device}")
    return None


def _eval_stack(mlp, who: str, max_in: int):
    """The layers of ``mlp`` (see _mlp_stack) for a kernel that applies them with the batch norms' running statistics,
    after the checks every such kernel makes: TypeError if it is not a SharedMLP, ValueError for a batch norm in training
    mode or without running statistics and for more layers or wider ones than the kernels take, RuntimeError in grad
    mode (the kernels have no backward)."""
    stack = _mlp_stack(mlp)
    if stack is None:
        raise TypeError(f"{who} expects a SharedMLP of Linear [+ BatchNorm1d] [+ ReLU] layers, got {type(mlp).__name__}")
    for _, bn, _ in stack:
        if bn is not None and bn.training and bn.running_mean is not None:
            raise ValueError(f"{who} uses the batch norms' running statistics; in training mode call the module itself")
        if bn is not None and bn.running_mean is None:
            raise ValueError(f"{who} needs batch norms with running statistics (track_running_stats=True)")
    if len(stack) > SA_MLP_MAX_LAYERS or max(lin.out_features for lin, _, _ in stack) > SA_MLP_MAX_WIDTH \
            or mlp.in_channels > max_in:
        raise ValueError(f"{who} takes at most {SA_MLP_MAX_LAYERS} layers of at most {SA_MLP_MAX_WIDTH} channels "
                         f"({max_in} inputs), got {mlp.in_channels} -> {[lin.out_features for lin, _, _ in stack]}")
    if torch.is_grad_enabled() and any(p.requires_grad for p in mlp.parameters()):
        raise RuntimeError(f"{who} has no backward: call it under torch.no_grad()")
    return stack


def _check_params(stack, dev) -> None:
    for lin, bn, _ in stack:
        misfit = _linear_misfit(lin, dev) or (None if bn is None else _bn_tensors_misfit(bn, dev))
        if misfit is not None:
            raise misfit


def _stack_params(stack):
    """The tensors and flags of a layer stack (see _mlp_stack) as the fused-MLP kernels read them: a flat list of six
    tensors per layer (Linear weight and bias, batch-norm weight, bias, running mean and running variance, None where
    absent), the batch-norm epsilons and the ReLU flags."""
    params, eps, relu = [], [], []
    for lin, bn, r in stack:
        affine = bn is not None and bn.affine
        params += [lin.weight, lin.bias, bn.weight if affine else None, bn.bias if affine else None,
                   None if bn is None else bn.running_mean, None if bn is None else bn.running_var]
        eps.append(0.0 if bn is None else float(bn.eps))
        relu.append(bool(r))
    return params, eps, relu


def _layer_args(stack):
    """nlayers and the per-layer host arrays of the fused-MLP C entries (pn2_sa_mlp_max_typed and its row-wise twins):
    widths, weight, bias, bn_weight, bn_bias, bn_mean, bn_var, bn_eps, relu."""
    return _param_args(*_stack_params(stack))


def _param_args(params, eps, relu):
    """_layer_args from the tensors and flags _stack_params gives"""
    nl = len(eps)
    pa = lambda j: (ctypes.c_void_p * nl)(*[None if t is None else t.data_ptr() for t in params[j::6]])
    return (nl, (ctypes.c_int * nl)(*[w.shape[0] for w in params[0::6]]), pa(0), pa(1), pa(2), pa(3), pa(4), pa(5),
            (ctypes.c_float * nl)(*eps), (ctypes.c_int * nl)(*[1 if r else 0 for r in relu]))


def sa_mlp_dtype(points: Optional[torch.Tensor]):
    """The arithmetic (and output) type of sa_mlp_max: the autocast dtype inside torch.autocast, else that of points
    (float32 without points)."""
    if torch.is_autocast_enabled("cuda"):
        return torch.get_autocast_dtype("cuda")
    return torch.float32 if points is None else points.dtype


def sa_mlp_applies(mlp, xyz: torch.Tensor, points: Optional[torch.Tensor] = None, pooling: str = 'max') -> bool:
    """Whether a set-abstraction level with this learned stack runs through sa_mlp_max: ``mlp`` is a SharedMLP of at
    most SA_MLP_MAX_LAYERS layers no wider than SA_MLP_MAX_WIDTH whose batch norms are all in eval mode with running
    statistics and whose layers add up to at most SA_MLP_MAX_MACS multiply-adds per row (beyond that cuBLAS is faster),
    its parameters and buffers float32 on the inputs' device, grad mode is off, the inputs are on CUDA with
    features in float32 / bfloat16 / float16 (under autocast: an autocast dtype of bfloat16 / float16), and the pooling
    is 'max'.  Everything else (training, grad mode, a module converted to 16 bits, other callables, other poolings)
    keeps the torch layers.  Inside ``batch_invariant()`` the SA_MLP_MAX_MACS limit does not apply: the wide group_all
    levels take the kernel too."""
    stack = _mlp_stack(mlp)
    if stack is None or pooling != 'max' or torch.is_grad_enabled() or not xyz.is_cuda:
        return False
    if points is not None and (not points.is_cuda or points.dtype not in FEATURE_DTYPES):
        return False
    if sa_mlp_dtype(points) not in FEATURE_DTYPES:
        return False
    if len(stack) > SA_MLP_MAX_LAYERS or mlp.in_channels > SA_MLP_MAX_WIDTH + 3:
        return False
    if not _BATCH_INVARIANT and sum(lin.in_features * lin.out_features for lin, _, _ in stack) > SA_MLP_MAX_MACS:
        return False
    for lin, bn, _ in stack:
        if lin.out_features > SA_MLP_MAX_WIDTH or _linear_misfit(lin, xyz.device) is not None:
            return False
        if bn is not None and (bn.training or bn.running_mean is None or _bn_tensors_misfit(bn, xyz.device) is not None):
            return False
    return True


def sa_mlp_max(xyz: Optional[torch.Tensor], new_xyz: Optional[torch.Tensor], points: Optional[torch.Tensor],
               idx: Optional[torch.Tensor], mlp: SharedMLP, xyz_first: bool = True, use_xyz: bool = True,
               out: Optional[torch.Tensor] = None, *, lengths=None) -> torch.Tensor:
    """The inference tail of a set-abstraction level as one CUDA op (csrc/sa_mlp.cu): for every group (b, s)

        rows = concat(xyz[b, idx[b, s]] - new_xyz[b, s], points[b, idx[b, s]])     ([features, xyz] when not xyz_first;
                                                                                    the features alone when not use_xyz)
        out[b, s] = max over the rows of mlp(rows), its batch norms using their running statistics,

    without writing a tensor of B*S*K rows.  ``xyz`` (B, N, 3) float32; ``new_xyz`` (B, S, 3) float32, or None for zeros;
    ``points`` (B, N, C) float32 / bfloat16 / float16 or None; ``idx`` (B, S, K) int32, or None for the single group
    that holds every point in order (S = 1, K = N); ``mlp`` a SharedMLP in eval mode, whose own parameters and buffers
    the kernel reads (nothing is folded or cached, so a loaded checkpoint is seen at once).  ``out``: an optional
    (B, S, C_out) tensor to write, which may be a channel slice of a wider contiguous (B, S, .) tensor.

    The arithmetic type is that of ``points`` (float32 without points), or the autocast dtype inside torch.autocast, and
    the result has it: float32 is FP32 fused multiply-adds, the 16-bit types run on the tensor cores with float32
    accumulation and one rounding per layer.  Each output depends on its own group alone, so it has the same bits on
    every run, at every batch size and next to any other cloud, which a cuBLAS product does not promise.  NaN
    propagates as in the torch layers.  No gradient: call it under torch.no_grad().

    With ``idx=None`` (the group_all form) the call goes to the whole-cloud entry (pn2_sa_mlp_max_all_typed), which
    deals the row tiles of a cloud out to several CTAs when the batch is too small to fill the GPU; the maximum of exact
    keys does not depend on that split, so the bits are those of one CTA per cloud.  There ``lengths`` (B,) may give
    per-cloud row counts (see device_lengths): rows from lengths[i] on are never read and may hold NaN.  ``lengths``
    with an ``idx`` raises ValueError.  ``xyz`` may be None there when the rows take no coordinates (use_xyz=False with
    points).

    Raises ValueError for a batch norm in training mode (that needs batch statistics: use the module itself) or without
    running statistics, for more than 4 layers or widths above 1024, and for shapes that do not fit together; TypeError /
    RuntimeError for tensors of the wrong dtype or device."""
    if lengths is not None and idx is not None:
        raise ValueError("sa_mlp_max takes lengths only with idx=None (the one group of every cloud)")
    stack = _eval_stack(mlp, "sa_mlp_max", SA_MLP_MAX_WIDTH + 3)
    if xyz is None and (idx is not None or points is None or use_xyz):
        raise ValueError("sa_mlp_max needs xyz unless idx is None and the rows are the features alone (use_xyz=False)")
    if xyz is not None:
        xyz = require_cuda(xyz, "xyz", torch.float32)
        if xyz.dim() != 3 or xyz.shape[2] != 3:
            raise ValueError(f"sa_mlp_max expects (batch_size, ndataset, 3) xyz, got {tuple(xyz.shape)}")
        b, n = xyz.shape[0], xyz.shape[1]
        tensors = [xyz]
    else:
        points = require_cuda(points, "points", FEATURE_DTYPES)
        if points.dim() != 3:
            raise ValueError(f"sa_mlp_max expects (batch_size, ndataset, channel) points, got {tuple(points.shape)}")
        b, n = points.shape[0], points.shape[1]
        tensors = []
    if idx is not None:
        idx = require_cuda(idx, "idx", torch.int32)
        if idx.dim() != 3 or idx.shape[0] != b or idx.shape[2] < 1:
            raise ValueError(f"idx must be (batch_size, npoint, nsample >= 1) matching xyz, got {tuple(idx.shape)}")
        s, k = idx.shape[1], idx.shape[2]
        tensors.append(idx)
    else:
        s, k = 1, n
    if new_xyz is not None:
        new_xyz = require_cuda(new_xyz, "new_xyz", torch.float32)
        if tuple(new_xyz.shape) != (b, s, 3):
            raise ValueError(f"new_xyz must be (batch_size, npoint, 3) = {(b, s, 3)}, got {tuple(new_xyz.shape)}")
        tensors.append(new_xyz)
    dtype = sa_mlp_dtype(points)
    if dtype not in FEATURE_DTYPES:
        raise TypeError(f"sa_mlp_max computes in float32, bfloat16 or float16, not the autocast dtype {dtype}")
    c = 0
    if points is not None:
        points = require_cuda(points, "points", FEATURE_DTYPES)
        if points.dim() != 3 or tuple(points.shape[:2]) != (b, n):
            raise ValueError("points must be (batch_size, ndataset, channel) matching xyz")
        tensors.append(points)
        c = points.shape[2]
    cin = c + 3 if (use_xyz or points is None) else c
    if cin != mlp.in_channels:
        raise ValueError(f"the grouped rows have {cin} channels, mlp expects {mlp.in_channels}")
    same_device(*tensors)
    dev = tensors[0].device
    _check_params(stack, dev)
    cout = mlp.out_channels
    if out is not None:
        if not isinstance(out, torch.Tensor) or out.dtype != dtype or tuple(out.shape) != (b, s, cout):
            raise ValueError(f"out must be a {dtype} tensor of shape {(b, s, cout)}, got "
                             f"{getattr(out, 'dtype', type(out).__name__)} {tuple(getattr(out, 'shape', ()))}")
        if out.device != dev:
            raise RuntimeError(f"out must be on the inputs' device ({dev}), got {out.device}")
        if b * s and (out.stride(2) != 1 or out.stride(1) < cout or (b > 1 and out.stride(0) != s * out.stride(1))):
            raise ValueError("out must be a channel slice of a contiguous (batch_size, npoint, channels) tensor")
    if idx is None:
        lengths = device_lengths(lengths, b, n, dev, "sa_mlp_max") if b * s else None
    if torch.compiler.is_compiling():
        res = torch.ops.pn2.sa_mlp_max(xyz, new_xyz, points, idx, lengths, *_stack_params(stack), bool(xyz_first),
                                       bool(use_xyz), dtype)
        return res if out is None else out.copy_(res)
    return sa_mlp_max_launch(xyz, new_xyz, points, idx, lengths, *_stack_params(stack), xyz_first, use_xyz, dtype, out)


def sa_mlp_max_launch(xyz, new_xyz, points, idx, lengths, params, eps, relu, xyz_first: bool, use_xyz: bool, dtype, out=None):
    """sa_mlp_max on checked arguments: the layers as _stack_params gives them, ``lengths`` None or the device tensor,
    ``out`` None (a new (b, s, C_out) tensor) or a checked one."""
    ref = xyz if xyz is not None else points
    b, n = ref.shape[0], ref.shape[1]
    s, k = (1, n) if idx is None else (idx.shape[1], idx.shape[2])
    c = 0 if points is None else points.shape[2]
    dev = ref.device
    if out is None:
        out = torch.empty((b, s, params[-6].shape[0]), dtype=dtype, device=dev)
    if b * s == 0:
        return out
    if points is not None and points.dtype != dtype:
        points = points.to(dtype)  # autocast: as the first Linear would cast its input
    lib = _lib.load()
    if idx is None:
        with on_device(ref):
            wsb = int(lib.pn2_sa_mlp_max_all_workspace_bytes(b, out.shape[2]))
            ws = torch.empty(wsb, dtype=torch.uint8, device=dev)
            rc = lib.pn2_sa_mlp_max_all_typed(
                DTYPE_CODES[dtype], b, n, c, ptr(xyz), ptr(new_xyz), ptr(points), ptr(lengths), 1 if xyz_first else 0,
                1 if use_xyz else 0, *_param_args(params, eps, relu), ptr(out), out.stride(1), ptr(ws), wsb, stream_ptr(dev))
        _lib.check(rc, "pn2_sa_mlp_max_all_typed")
        return out
    with on_device(xyz):
        rc = lib.pn2_sa_mlp_max_typed(
            DTYPE_CODES[dtype], b, n, c, s, k, ptr(xyz), ptr(new_xyz), ptr(points), ptr(idx), 1 if xyz_first else 0,
            1 if use_xyz else 0, *_param_args(params, eps, relu), ptr(out), out.stride(1), stream_ptr(dev))
    _lib.check(rc, "pn2_sa_mlp_max_typed")
    return out


ROW_MLP_MAX_IN = 1536  # first-layer inputs of fp_mlp / mlp_rows (PointNet2PartSegMSG.fp1 takes 512 + 1024)


def _out_rows(out, lead, cout, dtype, dev, who):
    """``out`` checked as a (*lead, cout) tensor of dtype on dev whose rows are cout-wide slices of a contiguous tensor
    (returned with its row stride), or a new one."""
    if out is None:
        return torch.empty((*lead, cout), dtype=dtype, device=dev), cout
    if not isinstance(out, torch.Tensor) or out.dtype != dtype or tuple(out.shape) != (*lead, cout):
        raise ValueError(f"{who}: out must be a {dtype} tensor of shape {(*lead, cout)}, got "
                         f"{getattr(out, 'dtype', type(out).__name__)} {tuple(getattr(out, 'shape', ()))}")
    if out.device != dev:
        raise RuntimeError(f"{who}: out must be on the inputs' device ({dev}), got {out.device}")
    rs = out.stride(-2) if out.dim() > 1 else cout
    ok = out.stride(-1) == 1 and rs >= cout
    for d in range(out.dim() - 2):  # every leading axis steps whole rows
        ok = ok and (out.shape[d] == 1 or out.stride(d) == rs * math.prod(out.shape[d + 1:-1]))
    if out.numel() and not ok:
        raise ValueError(f"{who}: out must be a channel slice of a contiguous (..., channels) tensor")
    return out, rs


def fp_mlp(xyz1: torch.Tensor, xyz2: torch.Tensor, points1: Optional[torch.Tensor], points2: torch.Tensor, mlp: SharedMLP,
           lengths=None, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """The inference tail of a feature-propagation level as one CUDA op (csrc/fp_mlp.cu): for every row j of cloud i

        row = concat(interpolate(points2[i] at the 3-NN of xyz1[i, j] in xyz2[i]), points1[i, j])
        out[i, j] = mlp(row), its batch norms using their running statistics,

    the row bit-identical to what fp_interpolate_concat writes, and no (B, N1, C2 + C1) tensor in between.  ``xyz1``
    (B, N1, 3) and ``xyz2`` (B, N2, 3) float32; ``points1`` (B, N1, C1) or None; ``points2`` (B, N2, C2) float32 /
    bfloat16 / float16; ``mlp`` a SharedMLP in eval mode, C2 + C1 <= 1536 inputs, whose own parameters and buffers the
    kernel reads on every call.  ``lengths``: optional (B,) per-cloud row counts of xyz1 / points1 (as
    pointnet_fp_module takes them); padding rows are never read and come out 0.  ``out``: an optional (B, N1, C_out)
    tensor to write, which may be a channel slice of a wider contiguous one.

    Arithmetic as in sa_mlp_max: the dtype of points2, or the autocast dtype inside torch.autocast (points1 and points2
    are then cast as the first Linear would cast its input); float32 is FP32 fused multiply-adds in ascending order, the
    16-bit types run on the tensor cores with float32 accumulation and one rounding per layer.  Each output row depends
    on its own row alone: the same bits at every batch size and next to any other cloud.  No gradient.

    Errors as sa_mlp_max: TypeError for a stack that is not a SharedMLP or tensors of the wrong dtype, ValueError for a
    training-mode batch norm, missing running statistics, too many or too wide layers and shapes that do not fit
    together, RuntimeError in grad mode or for tensors off CUDA."""
    stack = _eval_stack(mlp, "fp_mlp", ROW_MLP_MAX_IN)
    xyz1 = require_cuda(xyz1, "xyz1", torch.float32)
    xyz2 = require_cuda(xyz2, "xyz2", torch.float32)
    points2 = require_cuda(points2, "points2", FEATURE_DTYPES)
    if xyz1.dim() != 3 or xyz1.shape[2] != 3 or xyz2.dim() != 3 or xyz2.shape[2] != 3 or xyz2.shape[0] != xyz1.shape[0]:
        raise ValueError(f"fp_mlp expects (batch_size, n1, 3) xyz1 and (batch_size, n2, 3) xyz2, got "
                         f"{tuple(xyz1.shape)} and {tuple(xyz2.shape)}")
    b, n, m = xyz1.shape[0], xyz1.shape[1], xyz2.shape[1]
    if points2.dim() != 3 or points2.shape[:2] != xyz2.shape[:2] or points2.shape[2] < 1:
        raise ValueError(f"points2 must be (batch_size, n2, channel >= 1) matching xyz2, got {tuple(points2.shape)}")
    if m < 1:
        raise ValueError("fp_mlp needs at least one known point (n2 >= 1)")
    tensors = [xyz1, xyz2, points2]
    dtype = sa_mlp_dtype(points2)
    if dtype not in FEATURE_DTYPES:
        raise TypeError(f"fp_mlp computes in float32, bfloat16 or float16, not the autocast dtype {dtype}")
    c1 = 0
    if points1 is not None:
        points1 = require_cuda(points1, "points1", FEATURE_DTYPES)
        if points1.dim() != 3 or points1.shape[:2] != xyz1.shape[:2]:
            raise ValueError(f"points1 must be (batch_size, n1, channel) matching xyz1, got {tuple(points1.shape)}")
        if points1.dtype != points2.dtype and not torch.is_autocast_enabled("cuda"):
            raise TypeError(f"points1 ({points1.dtype}) and points2 ({points2.dtype}) must have one dtype")
        tensors.append(points1)
        c1 = points1.shape[2]
    c2 = points2.shape[2]
    if c2 + c1 != mlp.in_channels:
        raise ValueError(f"the propagated rows have {c2} + {c1} channels, mlp expects {mlp.in_channels}")
    same_device(*tensors)
    dev = xyz1.device
    _check_params(stack, dev)
    lengths = device_lengths(lengths, b, n, dev, "fp_mlp")
    if b > 65535:
        raise ValueError(f"fp_mlp takes at most 65535 clouds, got {b}")
    out, rs = _out_rows(out, (b, n), mlp.out_channels, dtype, dev, "fp_mlp")
    if torch.compiler.is_compiling():
        res = torch.ops.pn2.fp_mlp(xyz1, xyz2, points1, points2, lengths, *_stack_params(stack), dtype)
        return res if out is None else out.copy_(res)
    return fp_mlp_launch(xyz1, xyz2, points1, points2, lengths, *_stack_params(stack), dtype, out, rs)


def fp_mlp_launch(xyz1, xyz2, points1, points2, lengths, params, eps, relu, dtype, out=None, rs=None):
    """fp_mlp on checked arguments (layers as _stack_params gives them); ``out`` None (a new tensor) or checked, with its
    row stride ``rs``."""
    b, n, m = xyz1.shape[0], xyz1.shape[1], xyz2.shape[1]
    c1 = 0 if points1 is None else points1.shape[2]
    c2 = points2.shape[2]
    dev = xyz1.device
    if out is None:
        out, rs = torch.empty((b, n, params[-6].shape[0]), dtype=dtype, device=dev), params[-6].shape[0]
    if b * n == 0:
        return out
    points2 = points2.to(dtype)  # autocast: as the first Linear would cast its input
    if points1 is not None:
        points1 = points1.to(dtype)
    lib = _lib.load()
    with on_device(xyz1):
        wsb = int(lib.pn2_fp_mlp_workspace_bytes(b, n))
        ws = torch.empty(wsb, dtype=torch.uint8, device=dev)
        rc = lib.pn2_fp_mlp_typed(DTYPE_CODES[dtype], b, n, m, c2, c1, ptr(xyz1), ptr(lengths), ptr(xyz2), ptr(points1),
                                  ptr(points2), *_param_args(params, eps, relu), ptr(out), rs, ptr(ws), wsb, stream_ptr(dev))
    _lib.check(rc, "pn2_fp_mlp_typed")
    return out


def mlp_rows(t: torch.Tensor, mlp: SharedMLP, mask: Optional[torch.Tensor] = None) -> torch.Tensor:
    """``mlp`` applied to every row of ``t`` (..., C) as one CUDA op (csrc/fp_mlp.cu), its batch norms using their
    running statistics: what SharedMLP.forward(t, mask) computes in eval mode, with the arithmetic, the errors and the
    batch invariance of fp_mlp.  ``mask``: optional bool tensor of t.shape[:-1] (or as many elements), True on the real
    rows; the others are never read (they may be NaN) and come out 0.  C <= 1536.  Returns (..., C_out) in the
    arithmetic dtype."""
    stack = _eval_stack(mlp, "mlp_rows", ROW_MLP_MAX_IN)
    t = require_cuda(t, "t", FEATURE_DTYPES)
    if t.dim() < 1 or t.shape[-1] != mlp.in_channels:
        raise ValueError(f"mlp_rows: t must be (..., {mlp.in_channels}), got {tuple(t.shape)}")
    lead = tuple(t.shape[:-1])
    rows = math.prod(lead)
    tensors = [t]
    if mask is not None:
        if not isinstance(mask, torch.Tensor) or mask.dtype != torch.bool or mask.numel() != rows:
            raise ValueError(f"mlp_rows expects a bool mask of {rows} rows, got "
                             f"{getattr(mask, 'dtype', type(mask).__name__)} {tuple(getattr(mask, 'shape', ()))}")
        tensors.append(mask)
    dtype = sa_mlp_dtype(t)
    if dtype not in FEATURE_DTYPES:
        raise TypeError(f"mlp_rows computes in float32, bfloat16 or float16, not the autocast dtype {dtype}")
    same_device(*tensors)
    _check_params(stack, t.device)
    if torch.compiler.is_compiling():
        return torch.ops.pn2.mlp_rows(t, None if mask is None else mask.reshape(-1), *_stack_params(stack), dtype)
    return mlp_rows_launch(t, mask, *_stack_params(stack), dtype)


def mlp_rows_launch(t, mask, params, eps, relu, dtype):
    """mlp_rows on checked arguments (layers as _stack_params gives them): a new (..., C_out) tensor."""
    cout = params[-6].shape[0]
    out = torch.empty((*t.shape[:-1], cout), dtype=dtype, device=t.device)
    rows = math.prod(t.shape[:-1])
    if rows == 0:
        return out
    t = t.to(dtype)  # autocast: as the first Linear would cast its input
    keep = None if mask is None else mask.reshape(-1).contiguous().view(torch.uint8)
    with on_device(t):
        rc = _lib.load().pn2_mlp_rows_typed(DTYPE_CODES[dtype], rows, t.shape[-1], ptr(t), ptr(keep),
                                            *_param_args(params, eps, relu), ptr(out), cout, stream_ptr(t.device))
    _lib.check(rc, "pn2_mlp_rows_typed")
    return out


# ---- batch-invariant inference ----------------------------------------------------------------------------------------
_BATCH_INVARIANT = False


def is_batch_invariant() -> bool:
    """Whether the batch-invariant mode (batch_invariant()) is on."""
    return _BATCH_INVARIANT


@contextlib.contextmanager
def batch_invariant(enabled: bool = True):
    """Batch-invariant inference, process-wide (as torch.use_deterministic_algorithms), restored on exit::

        with torch.no_grad(), layers.batch_invariant():
            logits, _ = net.eval()(points, lengths)

    Inside it every learned layer that runs in eval mode (batch norms with running statistics), with grad mode off, on
    CUDA, goes through the fused kernels: set-abstraction tails through sa_mlp_max whatever their width
    (SA_MLP_MAX_MACS does not apply), pointnet_fp_module with a SharedMLP through fp_mlp, and every other SharedMLP call
    (the heads, mlp2, the stacks of non-max poolings) through mlp_rows.  Each output row then depends on its own inputs
    alone, with the same bits at every batch size, chunking and padding, which the cuBLAS products of the torch layers do
    not promise.  A layer the kernels cannot take (more than 4 layers, widths above 1024, inputs above 1536, a module
    converted to 16 bits) raises RuntimeError instead of running the torch layers.  Training steps and grad-mode calls
    are untouched: batch statistics depend on the batch by definition.  Outside the mode nothing changes."""
    global _BATCH_INVARIANT
    prev = _BATCH_INVARIANT
    _BATCH_INVARIANT = bool(enabled)
    try:
        yield
    finally:
        _BATCH_INVARIANT = prev


def invariant_applies(mlp, x: torch.Tensor) -> bool:
    """Whether a call of ``mlp`` on ``x`` falls under batch_invariant(): the mode is on, grad mode is off, x is on CUDA,
    and every batch norm of mlp (when it is a SharedMLP) is in eval mode with running statistics."""
    if not _BATCH_INVARIANT or torch.is_grad_enabled() or not getattr(x, "is_cuda", False):
        return False
    bns = [m for m in mlp.modules() if isinstance(m, nn.modules.batchnorm._BatchNorm)] if isinstance(mlp, nn.Module) else []
    return all(not bn.training and bn.running_mean is not None for bn in bns)


def _invariant_call(fn, *args, **kwargs):
    """fn(...) for a layer that batch_invariant() sends to the kernels; an argument they cannot take is a RuntimeError
    (the mode never falls back to the torch layers)."""
    try:
        return fn(*args, **kwargs)
    except (TypeError, ValueError) as e:
        raise RuntimeError(f"batch_invariant(): the kernels cannot take this layer ({e}); leave the mode to run the "
                           f"torch layers") from e



def set_bn_momentum(model: nn.Module, bn_decay: float) -> None:
    """The reference's bn_decay is the weight of the OLD moving average (train_multi_gpu.py:139-147);
    torch's momentum is the weight of the NEW batch statistic."""
    for mod in model.modules():
        if isinstance(mod, nn.BatchNorm1d):
            mod.momentum = 1.0 - float(bn_decay)


_SCOPES: Dict[str, SharedMLP] = {}


def scoped_mlp(scope: str, name: str, in_channels: int, widths: Sequence[int], bn: bool, device,
               is_training: Optional[bool], bn_decay: Optional[float]) -> SharedMLP:
    """The SharedMLP registered as ``scope/name`` (created on first use), in train/eval mode per ``is_training``
    and with the batch-norm momentum ``bn_decay`` implies."""
    if scope is None:
        raise ValueError("mlp given as a list of widths needs a scope (the reference's variable scope)")
    key = f"{scope}/{name}"
    mod = _SCOPES.get(key)
    if mod is None:
        mod = SharedMLP(in_channels, list(widths), bn).to(device)
        _SCOPES[key] = mod
    elif mod.in_channels != int(in_channels) or [m.out_features for m in mod.body if isinstance(m, nn.Linear)] != [int(w) for w in widths]:
        raise ValueError(f"variable scope {key!r} already holds layers of another shape (TensorFlow would raise too)")
    if is_training is not None:
        mod.train(bool(is_training))
    if bn_decay is not None:
        set_bn_momentum(mod, float(bn_decay))
    return mod


def scope_parameters():
    """Every parameter created through scoped_mlp, e.g. for torch.optim.Adam(scope_parameters())."""
    return [p for m in _SCOPES.values() for p in m.parameters()]


def scope_modules() -> Dict[str, SharedMLP]:
    return dict(_SCOPES)


def reset_scopes() -> None:
    _SCOPES.clear()
