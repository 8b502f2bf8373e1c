"""Learned 1x1-conv stacks and the variable-scope registry behind the reference-form module calls.

The reference builds every learned layer as a 1x1 convolution + batch norm + ReLU on a channels-last
tensor (tf_util.conv2d called from utils/pointnet_util.py:115-121,146-152,187-190,221-226) and finds
its variables by TensorFlow variable scope (``scope='layer1'`` ...).  On a channels-last tensor a 1x1
convolution is a matrix product over the last axis, so ``SharedMLP`` is Linear + BatchNorm1d + ReLU over
the flattened leading axes (cuBLAS through torch: dense layers are outside the hand-written hot path).

``scoped_mlp`` is the registry that lets the reference's own call form run unchanged::

    l1_xyz, l1_points, l1_indices = pointnet_sa_module(l0_xyz, l0_points, npoint=1024, radius=0.1, nsample=32,
        mlp=[32,32,64], mlp2=None, group_all=False, is_training=is_training, bn_decay=bn_decay, scope='layer1')

(models/pointnet2_sem_seg.py:28): the first call under a scope creates the layers (xavier weights, zero
bias, as tf_util does) on the input's device, later calls reuse them; ``scope_parameters()`` hands them to
an optimiser, ``reset_scopes()`` is ``tf.reset_default_graph()``.
"""
from __future__ import annotations

from typing import Dict, Optional, Sequence

import torch
from torch import nn
from torch.autograd.function import once_differentiable

from . import _lib
from ._tensor import DTYPE_CODES, FEATURE_DTYPES, on_device, ptr, stream_ptr


class SharedMLP(nn.Module):
    """conv2d(1x1)+BN+ReLU stack on (..., C) tensors — tf_util.conv2d with xavier weights, zero bias."""

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
                layers.append(nn.BatchNorm1d(int(w)))
            if act:
                layers.append(nn.ReLU(inplace=True))
            c = int(w)
        self.body = nn.Sequential(*layers)
        self.in_channels, self.out_channels = int(in_channels), c

    def forward(self, t: torch.Tensor, mask: Optional[torch.Tensor] = None) -> torch.Tensor:
        """``mask``: optional bool tensor of t.shape[:-1] (or as many elements), True on the real rows of a padded batch
        (see row_mask).  Batch norm then takes its training statistics from the real rows only, and the padding rows of
        every layer's output are 0 (whatever t holds there, NaN included).  Without a mask: the plain stack."""
        lead = t.shape[:-1]
        if mask is None:
            return self.body(t.reshape(-1, t.shape[-1])).reshape(*lead, self.out_channels)
        keep = mask.reshape(-1, 1)
        # torch.where, not a multiply: NaN * 0 is NaN.  This one stays even before the fused op: NaN input rows would
        # reach the Linear's weight gradient through x^T dy.
        x = torch.where(keep, t.reshape(-1, t.shape[-1]), 0)
        mods = list(self.body)
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
                if not _fuses_at(mods, i + 1, x):
                    x = torch.where(keep, x, 0)
            else:
                x = mod(x)  # ReLU keeps the zeros
            i += 1
        return x.reshape(*lead, self.out_channels)


def row_mask(lengths: torch.Tensor, n: int) -> torch.Tensor:
    """(b, n) bool, True on rows j < lengths[i] of a padded batch.  The lengths are clamped to [1, n], as the kernels
    clamp them, and never leave the device."""
    return torch.arange(n, device=lengths.device).unsqueeze(0) < lengths.clamp(1, n).unsqueeze(1)


def masked_batch_norm(bn: nn.BatchNorm1d, x: torch.Tensor, keep: torch.Tensor) -> torch.Tensor:
    """``bn`` on the rows of x (R, C) where keep (R, 1) is True.  Training mode: normalised with the mean and (biased)
    variance of those rows, and the running statistics are updated from them as BatchNorm1d would from a batch made of
    them alone (unbiased variance, momentum or the cumulative average, num_batches_tracked).  Eval mode: the running
    statistics, as bn itself.  The statistics are float32 whatever x's dtype (as torch's batch norm keeps them under
    autocast); the result has x's dtype, and its padding rows are left for the caller to zero.  The padding rows of x
    must be 0 (the caller zeroes them), so the mean is a plain sum over every row.  The variance is a second pass over
    the centred real rows, not E[x^2] - mean^2, which cancels catastrophically once |mean| is large against the
    standard deviation.  The row count stays on the device: nothing synchronises with the host."""
    if not bn.training and bn.running_mean is not None:
        return bn(x)
    xf = x.float()
    cnt = keep.sum(dtype=torch.float32)
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


class _MaskedBatchNormReLU(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, weight, bias, keep, bn):
        rows, c = x.shape
        dev = x.device
        tracking = bn.track_running_stats and bn.running_mean is not None
        momentum = -1.0 if bn.momentum is None else float(bn.momentum)
        y = torch.empty_like(x)
        save_mean = torch.empty(c, dtype=torch.float32, device=dev)
        save_invstd = torch.empty(c, dtype=torch.float32, device=dev)
        lib = _lib.load()
        with on_device(x):
            if tracking:
                bn.num_batches_tracked.add_(1)  # on the device; the kernel reads it for the cumulative average
            wsb = int(lib.pn2_masked_bn_workspace_bytes(rows, c))
            ws = torch.empty(wsb, dtype=torch.uint8, device=dev)
            rc = lib.pn2_masked_bn_relu_forward_typed(
                DTYPE_CODES[x.dtype], rows, c, ptr(x), ptr(keep), ptr(weight), ptr(bias), float(bn.eps), momentum,
                ptr(bn.num_batches_tracked if tracking else None), ptr(bn.running_mean if tracking else None),
                ptr(bn.running_var if tracking else None), ptr(y), ptr(save_mean), ptr(save_invstd), ptr(ws), wsb,
                stream_ptr(dev))
        _lib.check(rc, "pn2_masked_bn_relu_forward_typed")
        ctx.save_for_backward(x, y, keep, weight, save_mean, save_invstd)
        ctx.affine = weight is not None
        return y

    @staticmethod
    @once_differentiable
    def backward(ctx, dy):
        x, y, keep, weight, save_mean, save_invstd = ctx.saved_tensors
        rows, c = x.shape
        dev = x.device
        dy = dy.to(x.dtype).contiguous()
        dx = torch.empty_like(x)
        dgamma = torch.empty(c, dtype=torch.float32, device=dev) if ctx.affine else None
        dbeta = torch.empty(c, dtype=torch.float32, device=dev) if ctx.affine else None
        lib = _lib.load()
        with on_device(x):
            wsb = int(lib.pn2_masked_bn_workspace_bytes(rows, c))
            ws = torch.empty(wsb, dtype=torch.uint8, device=dev)
            rc = lib.pn2_masked_bn_relu_backward_typed(
                DTYPE_CODES[x.dtype], rows, c, ptr(dy), ptr(x), ptr(y), ptr(keep), ptr(weight), ptr(save_mean),
                ptr(save_invstd), ptr(dx), ptr(dgamma), ptr(dbeta), ptr(ws), wsb, stream_ptr(dev))
        _lib.check(rc, "pn2_masked_bn_relu_backward_typed")
        return dx, dgamma, dbeta, None, None


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
    keep = keep.reshape(-1).contiguous().view(torch.uint8)  # the bool mask as bytes, no copy
    weight = bn.weight if bn.affine else None
    bias = bn.bias if bn.affine else None
    return _MaskedBatchNormReLU.apply(x, weight, bias, keep, bn)


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
