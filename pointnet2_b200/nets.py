"""torch twins of the learned tails around the geometry ops (SURVEY §8f n4 — OUTSIDE the measured
hot path: dense layers belong to cuBLAS/cuDNN through torch, not to hand-written kernels).

The reference builds every learned layer as a 1x1 convolution + batch norm + ReLU on a
channels-last tensor (tf_util.conv2d called from utils/pointnet_util.py:115-121,146-152,187-190,
221-226).  On a channels-last tensor a 1x1 convolution is a matrix product over the last axis, so
``SharedMLP`` is Linear + BatchNorm1d + ReLU applied to the flattened leading axes.

Networks (layer hyper-parameters quoted from the reference's model files):
    PointNet2ClsSSG   models/pointnet2_cls_ssg.py:32-43
    PointNet2ClsMSG   models/pointnet2_cls_msg.py:27-38
    PointNet2SemSeg   models/pointnet2_sem_seg.py:28-46
Geometry goes through pointnet2_b200.pointnet_util (the CUDA ops); there is no CPU path.
"""
from __future__ import annotations

from typing import Optional, Sequence

import torch
from torch import nn

from ._tensor import device_lengths
from .layers import SharedMLP, row_mask, set_bn_momentum  # noqa: F401
from .pointnet_util import pointnet_fp_module, pointnet_sa_module, pointnet_sa_module_msg


class SetAbstraction(nn.Module):
    """pointnet_sa_module (utils/pointnet_util.py:87-154) with its learned tail."""

    def __init__(self, in_channels: int, npoint: Optional[int], radius: Optional[float], nsample: Optional[int],
                 mlp: Sequence[int], mlp2: Optional[Sequence[int]] = None, group_all: bool = False, pooling: str = "max",
                 knn: bool = False, use_xyz: bool = True, bn: bool = True):
        super().__init__()
        self.npoint, self.radius, self.nsample = npoint, radius, nsample
        self.group_all, self.pooling, self.knn, self.use_xyz = group_all, pooling, knn, use_xyz
        cin = in_channels + 3 if (use_xyz or in_channels == 0) else in_channels
        self.mlp = SharedMLP(cin, mlp, bn)
        pooled = self.mlp.out_channels * (2 if pooling == "max_and_avg" else 1)
        self.mlp2 = SharedMLP(pooled, mlp2, bn) if mlp2 else None
        self.out_channels = self.mlp2.out_channels if self.mlp2 else pooled

    def forward(self, xyz, points, lengths=None):
        return pointnet_sa_module(xyz, points, self.npoint, self.radius, self.nsample, self.mlp, self.mlp2,
                                  group_all=self.group_all, pooling=self.pooling, knn=self.knn, use_xyz=self.use_xyz,
                                  lengths=lengths)


class SetAbstractionMSG(nn.Module):
    """pointnet_sa_module_msg (utils/pointnet_util.py:156-196) with its learned tails."""

    def __init__(self, in_channels: int, npoint: int, radius_list: Sequence[float], nsample_list: Sequence[int],
                 mlp_list: Sequence[Sequence[int]], use_xyz: bool = True, bn: bool = True):
        super().__init__()
        self.npoint, self.radius_list, self.nsample_list, self.use_xyz = npoint, list(radius_list), list(nsample_list), use_xyz
        cin = in_channels + 3 if (use_xyz or in_channels == 0) else in_channels
        self.mlps = nn.ModuleList(SharedMLP(cin, w, bn) for w in mlp_list)
        self.out_channels = sum(m.out_channels for m in self.mlps)

    def forward(self, xyz, points, lengths=None):
        return pointnet_sa_module_msg(xyz, points, self.npoint, self.radius_list, self.nsample_list, list(self.mlps),
                                      use_xyz=self.use_xyz, lengths=lengths)


class FeaturePropagation(nn.Module):
    """pointnet_fp_module (utils/pointnet_util.py:199-229) with its learned tail."""

    def __init__(self, in_channels: int, mlp: Sequence[int], bn: bool = True):
        super().__init__()
        self.mlp = SharedMLP(in_channels, mlp, bn)
        self.out_channels = self.mlp.out_channels

    def forward(self, xyz1, xyz2, points1, points2, lengths=None):
        return pointnet_fp_module(xyz1, xyz2, points1, points2, self.mlp, lengths=lengths)


class _ClsHead(nn.Module):
    def __init__(self, in_channels: int, num_class: int, keep_prob: float):
        super().__init__()
        self.fc1 = SharedMLP(in_channels, [512])
        self.dp1 = nn.Dropout(1.0 - keep_prob)
        self.fc2 = SharedMLP(512, [256])
        self.dp2 = nn.Dropout(1.0 - keep_prob)
        self.fc3 = SharedMLP(256, [num_class], bn=False, last_activation=False)

    def forward(self, feat):
        return self.fc3(self.dp2(self.fc2(self.dp1(self.fc1(feat)))))


class PointNet2ClsSSG(nn.Module):
    """Classification net, input (B,N,3) -> logits (B,num_class). models/pointnet2_cls_ssg.py:20-43.
    ``lengths`` (B,), optional: cloud i is ``point_cloud[i, :lengths[i]]`` (variable-size clouds padded to N).  Only
    the first level sees the padding: it samples 512 centroids per cloud from the real points, and every later level
    is dense."""

    def __init__(self, num_class: int = 40):
        super().__init__()
        self.sa1 = SetAbstraction(0, 512, 0.2, 32, [64, 64, 128])
        self.sa2 = SetAbstraction(128, 128, 0.4, 64, [128, 128, 256])
        self.sa3 = SetAbstraction(256, None, None, None, [256, 512, 1024], group_all=True)
        self.head = _ClsHead(1024, num_class, keep_prob=0.5)

    def forward(self, point_cloud, lengths=None):
        end_points = {"l0_xyz": point_cloud}
        l1_xyz, l1_points, _ = self.sa1(point_cloud, None, lengths)
        l2_xyz, l2_points, _ = self.sa2(l1_xyz, l1_points)
        _, l3_points, _ = self.sa3(l2_xyz, l2_points)
        return self.head(l3_points.reshape(point_cloud.shape[0], -1)), end_points


class PointNet2ClsMSG(nn.Module):
    """Multi-scale classification net. models/pointnet2_cls_msg.py:18-38.  ``lengths``: as for PointNet2ClsSSG."""

    def __init__(self, num_class: int = 40):
        super().__init__()
        self.sa1 = SetAbstractionMSG(0, 512, [0.1, 0.2, 0.4], [16, 32, 128], [[32, 32, 64], [64, 64, 128], [64, 96, 128]])
        self.sa2 = SetAbstractionMSG(self.sa1.out_channels, 128, [0.2, 0.4, 0.8], [32, 64, 128],
                                     [[64, 64, 128], [128, 128, 256], [128, 128, 256]])
        self.sa3 = SetAbstraction(self.sa2.out_channels, None, None, None, [256, 512, 1024], group_all=True)
        self.head = _ClsHead(1024, num_class, keep_prob=0.4)

    def forward(self, point_cloud, lengths=None):
        l1_xyz, l1_points = self.sa1(point_cloud, None, lengths)
        l2_xyz, l2_points = self.sa2(l1_xyz, l1_points)
        _, l3_points, _ = self.sa3(l2_xyz, l2_points)
        return self.head(l3_points.reshape(point_cloud.shape[0], -1)), {}


class PointNet2SemSeg(nn.Module):
    """Semantic segmentation net, input (B,N,3) -> logits (B,N,num_class). models/pointnet2_sem_seg.py:20-46.
    ``lengths`` (B,), optional: cloud i is ``point_cloud[i, :lengths[i]]`` (variable-size clouds padded to N).  Only the
    first and the last levels see the padding: sa1 samples 1024 centroids per cloud from the real points (every deeper
    level is dense), and fp4 interpolates onto the real points only.  The batch norms of fp4 and fc1 take their
    statistics from the real rows, and the padding rows of the logits are 0 (sem_seg_loss(..., lengths=) ignores them)."""

    def __init__(self, num_class: int = 21):
        super().__init__()
        self.sa1 = SetAbstraction(0, 1024, 0.1, 32, [32, 32, 64])
        self.sa2 = SetAbstraction(64, 256, 0.2, 32, [64, 64, 128])
        self.sa3 = SetAbstraction(128, 64, 0.4, 32, [128, 128, 256])
        self.sa4 = SetAbstraction(256, 16, 0.8, 32, [256, 256, 512])
        self.fp1 = FeaturePropagation(512 + 256, [256, 256])
        self.fp2 = FeaturePropagation(256 + 128, [256, 256])
        self.fp3 = FeaturePropagation(256 + 64, [256, 128])
        self.fp4 = FeaturePropagation(128, [128, 128, 128])
        self.fc1 = SharedMLP(128, [128])
        self.dp1 = nn.Dropout(0.5)
        self.fc2 = SharedMLP(128, [num_class], bn=False, last_activation=False)

    def forward(self, point_cloud, lengths=None):
        l0_xyz = point_cloud
        mask = None
        if lengths is not None:
            b, n = point_cloud.shape[0], point_cloud.shape[1]
            lengths = device_lengths(lengths, b, n, point_cloud.device, "PointNet2SemSeg")
            mask = row_mask(lengths, n)
        l1_xyz, l1_points, _ = self.sa1(l0_xyz, None, lengths)
        l2_xyz, l2_points, _ = self.sa2(l1_xyz, l1_points)
        l3_xyz, l3_points, _ = self.sa3(l2_xyz, l2_points)
        l4_xyz, l4_points, _ = self.sa4(l3_xyz, l3_points)
        l3_points = self.fp1(l3_xyz, l4_xyz, l3_points, l4_points)
        l2_points = self.fp2(l2_xyz, l3_xyz, l2_points, l3_points)
        l1_points = self.fp3(l1_xyz, l2_xyz, l1_points, l2_points)
        l0_points = self.fp4(l0_xyz, l1_xyz, None, l1_points, lengths)
        feats = self.fc1(l0_points, mask)
        return self.fc2(self.dp1(feats), mask), {"feats": feats}


def cls_loss(pred: torch.Tensor, label: torch.Tensor) -> torch.Tensor:
    """mean sparse softmax cross entropy — models/pointnet2_cls_ssg.py:46-53."""
    return nn.functional.cross_entropy(pred, label.long())


def sem_seg_loss(pred: torch.Tensor, label: torch.Tensor, smpw: torch.Tensor, lengths=None) -> torch.Tensor:
    """sample-weighted cross entropy — models/pointnet2_sem_seg.py:49-56 (tf.losses default reduction:
    sum of weighted losses / number of non-zero weights).  ``lengths`` (B,), optional: the padding rows j >= lengths[i]
    count as weight 0, whatever smpw, label and pred hold there."""
    label = label.reshape(-1).long()
    keep = None
    logits = pred.reshape(-1, pred.shape[-1])
    if lengths is not None:
        b, n = pred.shape[0], pred.shape[1]
        keep = row_mask(device_lengths(lengths, b, n, pred.device, "sem_seg_loss"), n).reshape(-1)
        label = torch.where(keep, label, 0)  # any class: the row's weight is 0
        # select before the softmax, not after: its backward would turn a zero gradient times NaN logits into NaN
        logits = torch.where(keep.unsqueeze(1), logits, 0)
    per = nn.functional.cross_entropy(logits, label, reduction="none")
    w = smpw.reshape(-1).to(per.dtype)
    if keep is not None:
        w = torch.where(keep, w, 0)
    return (per * w).sum() / torch.clamp((w != 0).sum(), min=1)
