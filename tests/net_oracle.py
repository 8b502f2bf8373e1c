"""The reference's five PointNet++ models restated in float64, for checking what the networks of nets.py compute as a
whole (tests/test_net_oracle_cpu.py, tests/test_nets_float64_gpu.py).

Restated from the reference's model files (models/pointnet2_{cls_ssg,cls_msg,sem_seg,part_seg,part_seg_msg_one_hot}.py)
and the layers they call (utils/pointnet_util.py, utils/tf_util.py), not from nets.py:

* Geometry decisions come from the C oracle (oracle/oracle.py) on the float32 coordinates: FPS, the gather of the
  centroids, the ball query, kNN and three_nn.  That is exact, not an approximation: the coordinate path only samples
  and gathers, so every level's xyz is a bit-exact copy of input rows, and the oracle's indices are pinned to the
  kernels by the op tests.  A ragged batch runs each call on the truncated cloud.
* Everything continuous is plain float64 torch with autograd: the gathers by integer indexing and the centring, the
  concat orders (SSG [xyz, features], MSG [features, xyz], FP [interpolated, points1]), Linear + batch norm with batch
  statistics and eps 1e-3 (tf.contrib.layers.batch_norm's default, which tf_util.batch_norm_template keeps) + ReLU,
  the poolings, group_all, the inverse squared-distance weights of the interpolation (clamped at 1e-10, computed in
  float64 from the oracle's neighbours) and the three losses.
* Ragged batches (DESIGN §6.8): sa1 sees each cloud's real rows only, the last FP level and fc1 take their batch-norm
  statistics from the real rows only (the restatement computes nothing else), and the padding rows of the logits
  are 0.

Parameters are read from a net's ``state_dict()`` by name, each key exactly once (``Params.taken``), so a layer the
network ignores, or one the restatement does not know, shows up.  The running statistics are updated with torch's
rule (unbiased variance, momentum or the cumulative average), which the project documents; the reference's own moving
variance depends on which TF kernel ran and is not restated.

This module must never load the CUDA library: it imports nothing from pointnet2_b200.
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import Dict, List, Optional, Sequence

import numpy as np
import torch

from oracle import oracle as O

BN_EPS = 1e-3  # tf.contrib.layers.batch_norm's default epsilon; tf_util.batch_norm_template passes none
F64 = torch.float64

NUM_CATEGORIES = 16
NETS = ("cls_ssg", "cls_msg", "sem_seg", "part_seg", "part_seg_msg")


class Params:
    """A state dict read by name.  Every key may be taken once; parameters become float64 leaves on ``device`` (a
    tensor that already is a float64 leaf requiring grad is used as it is, for gradcheck), and batch norms in training
    mode record their updated running statistics in ``stats``."""

    def __init__(self, state, device="cpu", momentum: Optional[float] = 0.1, eps: float = BN_EPS):
        self.state, self.device, self.momentum, self.eps = state, torch.device(device), momentum, eps
        self.taken: List[str] = []
        self.leaves: Dict[str, torch.Tensor] = {}
        self.stats: Dict[str, torch.Tensor] = {}

    def _take(self, name):
        if name in self.taken:
            raise KeyError(f"{name} taken twice")
        if name not in self.state:
            raise KeyError(f"{name} is not in the state dict")
        self.taken.append(name)
        return self.state[name]

    def param(self, name):
        t = self._take(name)
        if not (t.requires_grad and t.dtype == F64 and t.device == self.device):
            t = t.detach().to(self.device, F64).clone().requires_grad_(True)
        self.leaves[name] = t
        return t

    def buffer(self, name):
        return self._take(name).detach().to(self.device)


def _join(prefix, name):
    return f"{prefix}.{name}" if prefix else name


def batch_norm(P: Params, prefix: str, x, training: bool):
    """x (R, C): batch statistics over the R rows in training (biased variance to normalise, torch's update of the
    running statistics), the running statistics otherwise"""
    gamma, beta = P.param(_join(prefix, "weight")), P.param(_join(prefix, "bias"))
    rm, rv = P.buffer(_join(prefix, "running_mean")).to(F64), P.buffer(_join(prefix, "running_var")).to(F64)
    nbt = P.buffer(_join(prefix, "num_batches_tracked"))
    if training:
        r = x.shape[0]
        mean = x.mean(0)
        var = ((x - mean) ** 2).mean(0)
        f = 1.0 / float(nbt + 1) if P.momentum is None else P.momentum
        P.stats[_join(prefix, "running_mean")] = (1 - f) * rm + f * mean.detach()
        P.stats[_join(prefix, "running_var")] = (1 - f) * rv + f * var.detach() * r / max(r - 1, 1)
        P.stats[_join(prefix, "num_batches_tracked")] = nbt + 1
    else:
        mean, var = rm, rv
    return (x - mean) / torch.sqrt(var + P.eps) * gamma + beta


def mlp(P: Params, prefix: str, x, widths: Sequence[int], training: bool, bn: bool = True, last_activation: bool = True):
    """tf_util.conv2d / conv1d / fully_connected with a 1x1 kernel, stacked: x (..., C) -> (..., widths[-1]).  Batch
    norm takes its statistics over every leading row.  The state-dict names follow nets' SharedMLP: ``body.i`` counts
    Linear, BatchNorm1d and ReLU modules in order."""
    lead = x.shape[:-1]
    x = x.reshape(-1, x.shape[-1])
    i = 0
    for k, w in enumerate(widths):
        weight, bias = P.param(_join(prefix, f"body.{i}.weight")), P.param(_join(prefix, f"body.{i}.bias"))
        if tuple(weight.shape) != (int(w), x.shape[1]):
            raise ValueError(f"{prefix} layer {k}: weight {tuple(weight.shape)}, expected ({w}, {x.shape[1]})")
        x = x @ weight.T + bias
        i += 1
        act = last_activation or k + 1 < len(widths)
        if bn and act:
            x = batch_norm(P, _join(prefix, f"body.{i}"), x, training)
            i += 1
        if act:
            x = torch.relu(x)
            i += 1
    return x.reshape(*lead, x.shape[-1])


# ------------------------------------------------------------------------------------------------------- geometry
def _lengths(lengths, b, n):
    return [n] * b if lengths is None else [int(min(max(int(l), 1), n)) for l in lengths]


def _sample(xyz, npoint, lengths):
    """FPS + gather per (truncated) cloud: (b, npoint, 3) float32, bit-exact rows of xyz"""
    out = np.empty((xyz.shape[0], npoint, 3), np.float32)
    for i, l in enumerate(lengths):
        c = np.ascontiguousarray(xyz[i:i + 1, :l])
        out[i] = O.oracle_gather_point(c, O.oracle_fps(npoint, c))[0]
    return out


def _ball(xyz, new_xyz, radius, nsample, lengths):
    idx = np.empty(new_xyz.shape[:2] + (nsample,), np.int64)
    for i, l in enumerate(lengths):
        idx[i] = O.oracle_query_ball_point(radius, nsample, np.ascontiguousarray(xyz[i:i + 1, :l]), new_xyz[i:i + 1])[0][0]
    return idx


def _knn(xyz, new_xyz, nsample):
    return O.oracle_knn_point(nsample, xyz, new_xyz)[1].astype(np.int64)


def _gather(t, idx):
    """t (b, n, c) tensor, idx (b, ...) integer numpy -> (b, ..., c)"""
    idx = torch.from_numpy(np.ascontiguousarray(idx, dtype=np.int64)).to(t.device)
    bidx = torch.arange(t.shape[0], device=t.device).view(-1, *([1] * (idx.dim() - 1)))
    return t[bidx, idx]


def _t64(a, device):
    return torch.from_numpy(np.ascontiguousarray(a)).to(device, F64)


def sa(P, prefix, xyz, feats, npoint, radius, nsample, widths, training, lengths=None, mlp2=None, group_all=False,
       pooling="max", knn=False, use_xyz=True):
    """pointnet_sa_module.  xyz (b, n, 3) float32 numpy, feats (b, n, c) float64 tensor or None.  Returns (new_xyz
    float32 numpy, new_points (b, npoint, C) tensor).  The learned layers are ``prefix.mlp`` / ``prefix.mlp2``."""
    b, n = xyz.shape[:2]
    dev = P.device
    x64 = _t64(xyz, dev)
    if group_all:
        new_xyz = np.zeros((b, 1, 3), np.float32)
        grouped_xyz = x64.unsqueeze(1)  # not centred: the origin is the centroid
        if feats is None:
            new_points = grouped_xyz
        else:
            new_points = torch.cat([x64, feats], -1).unsqueeze(1) if use_xyz else feats.unsqueeze(1)
    else:
        ls = _lengths(lengths, b, n)
        new_xyz = _sample(xyz, npoint, ls)
        idx = _knn(xyz, new_xyz, nsample) if knn else _ball(xyz, new_xyz, radius, nsample, ls)
        grouped_xyz = _gather(x64, idx) - _t64(new_xyz, dev).unsqueeze(2)
        if feats is None:
            new_points = grouped_xyz
        else:
            grouped = _gather(feats, idx)
            new_points = torch.cat([grouped_xyz, grouped], -1) if use_xyz else grouped
    new_points = mlp(P, _join(prefix, "mlp"), new_points, widths, training)
    if pooling == "max":
        new_points = new_points.amax(2)
    elif pooling == "avg":
        new_points = new_points.mean(2)
    elif pooling == "weighted_avg":
        e = torch.exp(-5 * torch.sqrt((grouped_xyz ** 2).sum(-1, keepdim=True)))
        new_points = (new_points * (e / e.sum(2, keepdim=True))).sum(2)
    elif pooling == "max_and_avg":
        new_points = torch.cat([new_points.mean(2), new_points.amax(2)], -1)
    else:
        raise ValueError(pooling)
    if mlp2:
        new_points = mlp(P, _join(prefix, "mlp2"), new_points, mlp2, training)
    return new_xyz, new_points


def sa_msg(P, prefix, xyz, feats, npoint, radii, nsamples, widths_list, training, lengths=None):
    """pointnet_sa_module_msg: one sampling, per scale [grouped features, centred xyz] -> mlp -> max"""
    b, n = xyz.shape[:2]
    dev = P.device
    ls = _lengths(lengths, b, n)
    new_xyz = _sample(xyz, npoint, ls)
    x64, c64 = _t64(xyz, dev), _t64(new_xyz, dev)
    outs = []
    for k, (radius, nsample, widths) in enumerate(zip(radii, nsamples, widths_list)):
        idx = _ball(xyz, new_xyz, radius, nsample, ls)
        gx = _gather(x64, idx) - c64.unsqueeze(2)
        g = gx if feats is None else torch.cat([_gather(feats, idx), gx], -1)
        outs.append(mlp(P, _join(prefix, f"mlps.{k}"), g, widths, training).amax(2))
    return new_xyz, torch.cat(outs, -1)


def interpolation(xyz1, xyz2, lengths=None, device="cpu"):
    """three_nn neighbours of each real row of xyz1 among xyz2 (the oracle's), with float64 weights
    (1/max(d², 1e-10)) / Σ: per cloud (idx (l, 3) int64, weight (l, 3) float64 tensor).  A missing neighbour (fewer
    than three known points) has weight 0."""
    b, n = xyz1.shape[:2]
    out = []
    for i, l in enumerate(_lengths(lengths, b, n)):
        u = np.ascontiguousarray(xyz1[i:i + 1, :l])
        dist, idx = O.oracle_three_nn(u, np.ascontiguousarray(xyz2[i:i + 1]))
        idx = idx[0].astype(np.int64)
        d = ((u[0].astype(np.float64)[:, None, :] - xyz2[i].astype(np.float64)[idx]) ** 2).sum(-1)
        r = np.where(np.isinf(dist[0]), 0.0, 1.0 / np.maximum(d, 1e-10))
        out.append((idx, torch.from_numpy(r / r.sum(1, keepdims=True)).to(device)))
    return out


def fp(P, prefix, xyz1, xyz2, points1, points2, widths, training, lengths=None):
    """pointnet_fp_module: [interpolated points2, points1] -> mlp.  points1 (b, n1, c1) tensor or None, points2
    (b, n2, c2).  Without lengths: (b, n1, C).  With lengths: the real rows of every cloud stacked, (Σ l, C), the batch
    norm's statistics taken over them alone."""
    rows = []
    for i, (idx, w) in enumerate(interpolation(xyz1, xyz2, lengths, P.device)):
        l = idx.shape[0]
        inter = (points2[i][torch.from_numpy(idx).to(P.device)] * w.unsqueeze(-1)).sum(1)
        rows.append(inter if points1 is None else torch.cat([inter, points1[i, :l]], -1))
    x = torch.cat(rows, 0)
    x = mlp(P, _join(prefix, "mlp"), x, widths, training)
    return x if lengths is not None else x.reshape(xyz1.shape[0], xyz1.shape[1], -1)


def _scatter_rows(x, lengths, b, n):
    """stacked real rows (Σ l, C) -> (b, n, C) with zero padding rows"""
    out = x.new_zeros(b, n, x.shape[-1])
    s = 0
    for i, l in enumerate(lengths):
        out[i, :l] = x[s:s + l]
        s += l
    return out


# --------------------------------------------------------------------------------------------------------- models
def _cls_head(P, feat, training):
    num_class = P.state["head.fc3.body.0.weight"].shape[0]
    x = mlp(P, "head.fc1", feat, [512], training)
    x = mlp(P, "head.fc2", x, [256], training)
    return mlp(P, "head.fc3", x, [num_class], training, bn=False, last_activation=False)


def cls_ssg(P, xyz, training, lengths=None):
    """models/pointnet2_cls_ssg.py: logits (b, num_class)"""
    l1_xyz, l1 = sa(P, "sa1", xyz, None, 512, 0.2, 32, [64, 64, 128], training, lengths)
    l2_xyz, l2 = sa(P, "sa2", l1_xyz, l1, 128, 0.4, 64, [128, 128, 256], training)
    _, l3 = sa(P, "sa3", l2_xyz, l2, None, None, None, [256, 512, 1024], training, group_all=True)
    return _cls_head(P, l3.reshape(xyz.shape[0], -1), training)


def cls_msg(P, xyz, training, lengths=None):
    """models/pointnet2_cls_msg.py: logits (b, num_class)"""
    l1_xyz, l1 = sa_msg(P, "sa1", xyz, None, 512, [0.1, 0.2, 0.4], [16, 32, 128],
                        [[32, 32, 64], [64, 64, 128], [64, 96, 128]], training, lengths)
    l2_xyz, l2 = sa_msg(P, "sa2", l1_xyz, l1, 128, [0.2, 0.4, 0.8], [32, 64, 128],
                        [[64, 64, 128], [128, 128, 256], [128, 128, 256]], training)
    _, l3 = sa(P, "sa3", l2_xyz, l2, None, None, None, [256, 512, 1024], training, group_all=True)
    return _cls_head(P, l3.reshape(xyz.shape[0], -1), training)


def _seg_head(P, x, training, lengths, b, n):
    """fc1 (conv1d 128, bn) and fc2 (no bn, no activation) on the stacked real rows, then back to (b, n, num_class)"""
    num_class = P.state["fc2.body.0.weight"].shape[0]
    x = mlp(P, "fc1", x, [128], training)
    x = mlp(P, "fc2", x, [num_class], training, bn=False, last_activation=False)
    return _scatter_rows(x, _lengths(lengths, b, n), b, n)


def _stacked(x, lengths, b, n):
    """(b, n, C) -> its real rows stacked, (Σ l, C)"""
    return torch.cat([x[i, :l] for i, l in enumerate(_lengths(lengths, b, n))], 0)


def sem_seg(P, xyz, training, lengths=None):
    """models/pointnet2_sem_seg.py: logits (b, n, num_class), padding rows 0"""
    b, n = xyz.shape[:2]
    l1_xyz, l1 = sa(P, "sa1", xyz, None, 1024, 0.1, 32, [32, 32, 64], training, lengths)
    l2_xyz, l2 = sa(P, "sa2", l1_xyz, l1, 256, 0.2, 32, [64, 64, 128], training)
    l3_xyz, l3 = sa(P, "sa3", l2_xyz, l2, 64, 0.4, 32, [128, 128, 256], training)
    l4_xyz, l4 = sa(P, "sa4", l3_xyz, l3, 16, 0.8, 32, [256, 256, 512], training)
    l3 = fp(P, "fp1", l3_xyz, l4_xyz, l3, l4, [256, 256], training)
    l2 = fp(P, "fp2", l2_xyz, l3_xyz, l2, l3, [256, 256], training)
    l1 = fp(P, "fp3", l1_xyz, l2_xyz, l1, l2, [256, 128], training)
    l0 = fp(P, "fp4", xyz, l1_xyz, None, l1, [128, 128, 128], training, lengths=_lengths(lengths, b, n))
    return _seg_head(P, l0, training, lengths, b, n)


def part_seg(P, pc, training, lengths=None):
    """models/pointnet2_part_seg.py: pc (b, n, 6) xyz + normals -> logits (b, n, num_part), padding rows 0"""
    b, n = pc.shape[:2]
    xyz, normals = np.ascontiguousarray(pc[..., :3]), _t64(pc[..., 3:], P.device)
    l1_xyz, l1 = sa(P, "sa1", xyz, normals, 512, 0.2, 64, [64, 64, 128], training, lengths)
    l2_xyz, l2 = sa(P, "sa2", l1_xyz, l1, 128, 0.4, 64, [128, 128, 256], training)
    l3_xyz, l3 = sa(P, "sa3", l2_xyz, l2, None, None, None, [256, 512, 1024], training, group_all=True)
    l2 = fp(P, "fp1", l2_xyz, l3_xyz, l2, l3, [256, 256], training)
    l1 = fp(P, "fp2", l1_xyz, l2_xyz, l1, l2, [256, 128], training)
    points1 = torch.cat([_t64(xyz, P.device), normals], -1)
    l0 = fp(P, "fp3", xyz, l1_xyz, points1, l1, [128, 128, 128], training, lengths=_lengths(lengths, b, n))
    return _seg_head(P, l0, training, lengths, b, n)


def part_seg_msg(P, pc, cls_label, training, lengths=None):
    """models/pointnet2_part_seg_msg_one_hot.py: pc (b, n, 6), cls_label (b,) -> logits (b, n, num_part)"""
    b, n = pc.shape[:2]
    xyz, normals = np.ascontiguousarray(pc[..., :3]), _t64(pc[..., 3:], P.device)
    l1_xyz, l1 = sa_msg(P, "sa1", xyz, normals, 512, [0.1, 0.2, 0.4], [32, 64, 128],
                        [[32, 32, 64], [64, 64, 128], [64, 96, 128]], training, lengths)
    l2_xyz, l2 = sa_msg(P, "sa2", l1_xyz, l1, 128, [0.4, 0.8], [64, 128], [[128, 128, 256], [128, 196, 256]], training)
    l3_xyz, l3 = sa(P, "sa3", l2_xyz, l2, None, None, None, [256, 512, 1024], training, group_all=True)
    l2 = fp(P, "fp1", l2_xyz, l3_xyz, l2, l3, [256, 256], training)
    l1 = fp(P, "fp2", l1_xyz, l2_xyz, l1, l2, [256, 128], training)
    one_hot = torch.zeros(b, n, NUM_CATEGORIES, dtype=F64, device=P.device)
    one_hot[torch.arange(b), :, torch.as_tensor(np.asarray(cls_label), dtype=torch.long)] = 1.0
    points1 = torch.cat([one_hot, _t64(xyz, P.device), normals], -1)
    l0 = fp(P, "fp3", xyz, l1_xyz, points1, l1, [128, 128], training, lengths=_lengths(lengths, b, n))
    return _seg_head(P, l0, training, lengths, b, n)


# --------------------------------------------------------------------------------------------------------- losses
def cls_loss(logits, label):
    """mean sparse softmax cross entropy"""
    return torch.nn.functional.cross_entropy(logits, torch.as_tensor(label, device=logits.device).long())


def sem_seg_loss(logits, label, smpw, lengths=None):
    """Σ weight·CE / #(weights ≠ 0) over the real rows (tf.losses' default reduction)"""
    b, n = logits.shape[:2]
    ls = _lengths(lengths, b, n)
    ce = torch.cat([torch.nn.functional.cross_entropy(logits[i, :l], torch.as_tensor(label[i, :l], device=logits.device).long(),
                                                      reduction="none") for i, l in enumerate(ls)])
    w = torch.cat([torch.as_tensor(smpw[i, :l], device=logits.device).to(F64) for i, l in enumerate(ls)])
    return (ce * w).sum() / max(int((w != 0).sum()), 1)


def part_seg_loss(logits, label, lengths=None):
    """mean CE over the real rows"""
    b, n = logits.shape[:2]
    ls = _lengths(lengths, b, n)
    ce = torch.cat([torch.nn.functional.cross_entropy(logits[i, :l], torch.as_tensor(label[i, :l], device=logits.device).long(),
                                                      reduction="none") for i, l in enumerate(ls)])
    return ce.mean()


# ---------------------------------------------------------------------------------------------------------- entry
@dataclass
class Result:
    logits: torch.Tensor
    loss: Optional[torch.Tensor]
    grads: Dict[str, torch.Tensor] = field(default_factory=dict)
    stats: Dict[str, torch.Tensor] = field(default_factory=dict)
    taken: List[str] = field(default_factory=list)


def run(net: str, state, points, *, lengths=None, label=None, smpw=None, cls_label=None, training=True,
        momentum: Optional[float] = 0.1, device="cpu") -> Result:
    """One forward of ``net`` (one of NETS) on ``points`` (b, n, 3) or (b, n, 6) float32 numpy (the padding rows are
    never read) with the parameters and buffers of ``state``.  In training mode with a ``label`` (and ``smpw`` for
    sem_seg) also the loss, the gradient of every parameter and the updated running statistics (by state-dict name).
    In eval mode the batch norms use the running statistics of ``state``."""
    P = Params(state, device, momentum)
    pts = np.ascontiguousarray(points, dtype=np.float32)
    if net == "cls_ssg":
        logits = cls_ssg(P, pts, training, lengths)
    elif net == "cls_msg":
        logits = cls_msg(P, pts, training, lengths)
    elif net == "sem_seg":
        logits = sem_seg(P, pts, training, lengths)
    elif net == "part_seg":
        logits = part_seg(P, pts, training, lengths)
    elif net == "part_seg_msg":
        logits = part_seg_msg(P, pts, cls_label, training, lengths)
    else:
        raise ValueError(net)
    loss = None
    if label is not None:
        if net.startswith("cls"):
            loss = cls_loss(logits, label)
        elif net == "sem_seg":
            loss = sem_seg_loss(logits, label, smpw, lengths)
        else:
            loss = part_seg_loss(logits, label, lengths)
    res = Result(logits.detach(), None if loss is None else loss.detach(), stats=dict(P.stats), taken=list(P.taken))
    if loss is not None and training:
        names = list(P.leaves)
        grads = torch.autograd.grad(loss, [P.leaves[k] for k in names], allow_unused=True)
        res.grads = {k: torch.zeros_like(P.leaves[k]) if g is None else g for k, g in zip(names, grads)}
    return res
