"""The reference's PointNet (v1) classifier, models/pointnet_cls_basic.py, restated in float64 on net_oracle's Params /
batch_norm / mlp (tests/test_pointnet_cls_cpu.py, tests/test_pointnet_cls_gpu.py).

Restated from the reference's model file, not from nets.py: conv1-conv5 as 1x1 stacks on the real rows of every cloud
stacked together (so the batch norms take their statistics from the real rows alone), a max over each cloud's real rows,
fc1 / fc2 with batch norm and fc3 without activation.  The dropout is left out: the tests run with p = 0.  The max's
gradient goes to the first maximal row (TF's MaxPoolGrad), which torch's max over a dimension does not promise, so it is
spelled out.

This module must never load the CUDA library: it imports nothing from pointnet2_b200.
"""
from __future__ import annotations

import numpy as np
import torch

import net_oracle as NO

FEAT = [64, 64, 64, 128]


def first_max(x):
    """x (l, C) -> (C,): the maximum over the rows, its gradient to the first row that reaches it"""
    m = x.detach().amax(0, keepdim=True)
    rows = torch.arange(x.shape[0], device=x.device).unsqueeze(1)
    first = torch.where(x.detach() == m, rows, x.shape[0]).amin(0, keepdim=True)
    return x.gather(0, first).squeeze(0)


def cls_basic(P: NO.Params, points, training: bool, lengths=None):
    """logits (b, num_class) of points (b, n, 3) float32 numpy; only rows j < lengths[i] are read"""
    b, n = points.shape[:2]
    ls = NO._lengths(lengths, b, n)
    x = torch.cat([NO._t64(points[i, :l], P.device) for i, l in enumerate(ls)], 0)
    x = NO.mlp(P, "feat", x, FEAT, training)
    x = NO.mlp(P, "conv5", x, [1024], training)
    starts = np.concatenate([[0], np.cumsum(ls)])
    g = torch.stack([first_max(x[starts[i]:starts[i + 1]]) for i in range(b)])
    num_class = P.state["fc3.body.0.weight"].shape[0]
    g = NO.mlp(P, "fc1", g, [512], training)
    g = NO.mlp(P, "fc2", g, [256], training)
    return NO.mlp(P, "fc3", g, [num_class], training, bn=False, last_activation=False)


def run(state, points, *, lengths=None, label=None, training=True, momentum=0.1, device="cpu") -> NO.Result:
    """As net_oracle.run, for the PointNet v1 classifier"""
    P = NO.Params(state, device, momentum)
    logits = cls_basic(P, np.ascontiguousarray(points, dtype=np.float32), training, lengths)
    loss = None if label is None else NO.cls_loss(logits, label)
    res = NO.Result(logits.detach(), None if loss is None else loss.detach(), stats=dict(P.stats), taken=list(P.taken))
    if loss is not None and training:
        names = list(P.leaves)
        grads = torch.autograd.grad(loss, [P.leaves[k] for k in names], allow_unused=True)
        res.grads = {k: torch.zeros_like(P.leaves[k]) if g is None else g for k, g in zip(names, grads)}
    return res
