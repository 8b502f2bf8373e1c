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
        # torch.where, not a multiply: NaN * 0 is NaN
        x = torch.where(keep, t.reshape(-1, t.shape[-1]), 0)
        for mod in self.body:
            if isinstance(mod, nn.BatchNorm1d):
                x = torch.where(keep, masked_batch_norm(mod, x, keep), 0)
            elif isinstance(mod, nn.Linear):
                x = torch.where(keep, mod(x), 0)
            else:
                x = mod(x)  # ReLU keeps the zeros
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
