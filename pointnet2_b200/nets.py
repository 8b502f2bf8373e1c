"""torch twins of the learned tails around the geometry ops (SURVEY §8f n4).  Training runs them through torch
(cuBLAS / cuDNN, plus the masked batch norm kernel on padded batches); in eval mode under no_grad the set-abstraction
tails run in the library's own kernel (layers.sa_mlp_max), the feature-propagation tails and heads through torch.

The reference builds every learned layer as a 1x1 convolution + batch norm + ReLU on a
channels-last tensor (tf_util.conv2d called from utils/pointnet_util.py:115-121,146-152,187-190,
221-226).  On a channels-last tensor a 1x1 convolution is a matrix product over the last axis, so
``SharedMLP`` is Linear + BatchNorm1d + ReLU applied to the flattened leading axes.

Networks (layer hyper-parameters quoted from the reference's model files):
    PointNet2ClsSSG   models/pointnet2_cls_ssg.py:32-43
    PointNet2ClsMSG   models/pointnet2_cls_msg.py:27-38
    PointNet2SemSeg   models/pointnet2_sem_seg.py:28-46
    PointNet2PartSeg     models/pointnet2_part_seg.py:17-41
    PointNet2PartSegMSG  models/pointnet2_part_seg_msg_one_hot.py:19-47
    PointNetClsBasic  models/pointnet_cls_basic.py:21-60 (PointNet v1, the baseline classifier)
Losses and metrics: cls_loss, sem_seg_loss, part_seg_loss; for part segmentation PART_OFFSETS, part_seg_predict and
part_seg_iou (part_seg/train.py:274-300).
Geometry goes through pointnet2_b200.pointnet_util (the CUDA ops); there is no CPU path.
"""
from __future__ import annotations

import math
from typing import Optional, Sequence

import numpy as np
import torch
from torch import nn

from ._tensor import device_lengths
from .layers import SharedMLP, row_mask, set_bn_momentum, shared_mlp_max  # noqa: F401
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


class PointNetClsBasic(nn.Module):
    """PointNet (v1) classification net, input (B,N,3) -> logits (B,num_class).  models/pointnet_cls_basic.py:21-60:
    conv1-conv5 (64, 64, 64, 128, 1024, each with batch norm and ReLU) on every point, a max over the cloud, fc1 512 and
    fc2 256 with batch norm, dropout (keep 0.7) after fc2 only, fc3 without activation.  No T-nets (the reference has
    none).

    conv1 is a [1, 3] convolution over the (N, 3, 1) image of the cloud (weight [1, 3, 1, 64]), so its xavier bound uses
    fan_in 3 and fan_out 3 * 64 = 192; the other layers are 1x1 and initialise as SharedMLP does.  conv1-conv4 are
    ``feat``, conv5 is ``conv5``: conv5 and the max form one step (layers.shared_mlp_max) that trains through the fused
    masked batch norm + ReLU + max-pool and infers through sa_mlp_max's whole-cloud kernel.

    ``lengths`` (B,), optional: cloud i is ``point_cloud[i, :lengths[i]]`` (variable-size clouds padded to N, as
    shapes.sample_shapes makes them with point dropout).  The padding rows are never read (they may be NaN), the batch
    norms of conv1-conv5 take their statistics from the real rows, and the max runs over the real rows only.  A lengths
    tensor on the GPU is never read back.  On CUDA dense and ragged batches run the same kernels (lengths=None means
    every row is real); on the CPU or in float64 the layers run as the torch composition."""

    def __init__(self, num_class: int = 40):
        super().__init__()
        self.feat = SharedMLP(3, [64, 64, 64, 128])
        bound = math.sqrt(6.0 / (3 + 3 * 64))  # xavier on the [1, 3, 1, 64] kernel: fan_in 3, fan_out 192
        nn.init.uniform_(self.feat.body[0].weight, -bound, bound)
        self.conv5 = SharedMLP(128, [1024])
        self.fc1 = SharedMLP(1024, [512])
        self.fc2 = SharedMLP(512, [256])
        self.dp1 = nn.Dropout(1.0 - 0.7)
        self.fc3 = SharedMLP(256, [num_class], bn=False, last_activation=False)

    def forward(self, point_cloud, lengths=None):
        if not isinstance(point_cloud, torch.Tensor) or point_cloud.dim() != 3 or point_cloud.shape[-1] != 3:
            shape = tuple(point_cloud.shape) if isinstance(point_cloud, torch.Tensor) else type(point_cloud).__name__
            raise ValueError(f"PointNetClsBasic expects a (batch_size, num_point, 3) point cloud, got {shape}")
        b, n = point_cloud.shape[0], point_cloud.shape[1]
        lengths = device_lengths(lengths, b, n, point_cloud.device, "PointNetClsBasic")
        if lengths is None:
            mask = torch.ones(b, n, dtype=torch.bool, device=point_cloud.device)
        else:
            mask = row_mask(lengths, n)
        net = self.feat(point_cloud, mask)
        net = shared_mlp_max(self.conv5, net, lengths)
        return self.fc3(self.dp1(self.fc2(self.fc1(net)))), {}


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


# ShapeNet part labels: category k (the 16 categories in alphabetical order, Airplane .. Table) owns the parts
# PART_OFFSETS[k] <= p < PART_OFFSETS[k + 1] of the 50 (part_seg/part_dataset_all_normal.py:75)
NUM_CATEGORIES = 16
PART_OFFSETS = (0, 4, 6, 8, 12, 16, 19, 22, 24, 28, 30, 36, 38, 41, 44, 47, 50)
_INT_DTYPES = (torch.int8, torch.int16, torch.int32, torch.int64, torch.uint8)


def _check_part_input(point_cloud, op: str) -> None:
    if not isinstance(point_cloud, torch.Tensor) or point_cloud.dim() != 3 or point_cloud.shape[-1] != 6:
        shape = tuple(point_cloud.shape) if isinstance(point_cloud, torch.Tensor) else type(point_cloud).__name__
        raise ValueError(f"{op} expects a (batch_size, num_point, 6) point cloud (xyz, then normals), got {shape}")


def category_labels(cls_label, b: int, device, op: str, num_category: int = NUM_CATEGORIES) -> torch.Tensor:
    """Object categories of a batch as the (b,) int64 tensor on ``device``.  A CPU tensor, numpy array or sequence is
    checked here (shape (b,), integers, 0 <= k < num_category, else ValueError) and then copied.  A CUDA tensor (on
    ``device``) is never read back, so the call stays asynchronous: its shape and dtype are checked and its values
    clamped to [0, num_category), as the kernels clamp lengths."""
    if isinstance(cls_label, torch.Tensor) and cls_label.is_cuda:
        if cls_label.device != device:
            raise RuntimeError(f"all tensors must be on the same device ({device} vs {cls_label.device})")
        if cls_label.dtype not in _INT_DTYPES or tuple(cls_label.shape) != (b,):
            raise ValueError(f"{op} expects (batch_size,) integer cls_label, shape ({b},), got {cls_label.dtype} "
                             f"{tuple(cls_label.shape)}")
        return cls_label.long().clamp(0, num_category - 1)
    arr = (cls_label.detach().cpu().numpy() if isinstance(cls_label, torch.Tensor) else np.asarray(cls_label))
    if tuple(arr.shape) != (b,) or (arr.size and not np.issubdtype(arr.dtype, np.integer)):
        raise ValueError(f"{op} expects (batch_size,) integer cls_label, shape ({b},), got {arr.dtype} {tuple(arr.shape)}")
    if b and (int(arr.min()) < 0 or int(arr.max()) >= num_category):
        raise ValueError(f"{op} expects 0 <= cls_label < {num_category}, got {arr.tolist()}")
    return torch.from_numpy(arr.astype(np.int64)).to(device)


class PointNet2PartSeg(nn.Module):
    """Part segmentation net, input (B,N,6) (xyz, then normals) -> logits (B,N,num_part).
    models/pointnet2_part_seg.py:17-41.

    ``lengths`` (B,), optional: shape i is ``point_cloud[i, :lengths[i]]`` (variable-size shapes padded to N).  Only
    the first and the last levels see the padding: sa1 samples 512 centroids per shape from the real points and groups
    their normals with them (sa2, sa3 and fp1, fp2 are dense), and fp3 interpolates onto the real points only.  The
    batch norms of fp3 and fc1 take their statistics from the real rows, and the padding rows of the logits are 0
    (part_seg_loss(..., lengths=) ignores them).
    Returns (logits, end_points) with end_points["feats"] the (B,N,128) output of fc1 and end_points["l1_xyz"] the
    (B,512,3) centroids of sa1."""

    def __init__(self, num_part: int = 50):
        super().__init__()
        self.sa1 = SetAbstraction(3, 512, 0.2, 64, [64, 64, 128])
        self.sa2 = SetAbstraction(128, 128, 0.4, 64, [128, 128, 256])
        self.sa3 = SetAbstraction(256, None, None, None, [256, 512, 1024], group_all=True)
        self.fp1 = FeaturePropagation(256 + 1024, [256, 256])
        self.fp2 = FeaturePropagation(128 + 256, [256, 128])
        self.fp3 = FeaturePropagation(128 + 6, [128, 128, 128])
        self.fc1 = SharedMLP(128, [128])
        self.dp1 = nn.Dropout(0.5)
        self.fc2 = SharedMLP(128, [num_part], bn=False, last_activation=False)

    def forward(self, point_cloud, lengths=None):
        _check_part_input(point_cloud, "PointNet2PartSeg")
        b, n = point_cloud.shape[0], point_cloud.shape[1]
        lengths = device_lengths(lengths, b, n, point_cloud.device, "PointNet2PartSeg")
        mask = None if lengths is None else row_mask(lengths, n)
        l0_xyz, l0_points = point_cloud[..., :3].contiguous(), point_cloud[..., 3:].contiguous()
        l1_xyz, l1_points, _ = self.sa1(l0_xyz, l0_points, lengths)
        l2_xyz, l2_points, _ = self.sa2(l1_xyz, l1_points)
        l3_xyz, l3_points, _ = self.sa3(l2_xyz, l2_points)
        l2_points = self.fp1(l2_xyz, l3_xyz, l2_points, l3_points)
        l1_points = self.fp2(l1_xyz, l2_xyz, l1_points, l2_points)
        l0_points = self.fp3(l0_xyz, l1_xyz, torch.cat([l0_xyz, l0_points], dim=2), l1_points, lengths)
        feats = self.fc1(l0_points, mask)
        return self.fc2(self.dp1(feats), mask), {"feats": feats, "l1_xyz": l1_xyz}


class PointNet2PartSegMSG(nn.Module):
    """Multi-scale part segmentation net with the object category as a one-hot input, (B,N,6) and (B,) -> logits
    (B,N,num_part).  models/pointnet2_part_seg_msg_one_hot.py:19-47.

    ``cls_label`` (B,) integers in [0, num_category): see category_labels for how a tensor on the GPU is treated.
    fp3 takes [one_hot(cls_label) tiled over N, xyz, normals] (22 channels) as its dense-level features.
    ``lengths``, the padding and the returned end_points: as for PointNet2PartSeg."""

    def __init__(self, num_part: int = 50, num_category: int = NUM_CATEGORIES):
        super().__init__()
        self.num_category = int(num_category)
        self.sa1 = SetAbstractionMSG(3, 512, [0.1, 0.2, 0.4], [32, 64, 128], [[32, 32, 64], [64, 64, 128], [64, 96, 128]])
        self.sa2 = SetAbstractionMSG(self.sa1.out_channels, 128, [0.4, 0.8], [64, 128], [[128, 128, 256], [128, 196, 256]])
        self.sa3 = SetAbstraction(self.sa2.out_channels, None, None, None, [256, 512, 1024], group_all=True)
        self.fp1 = FeaturePropagation(self.sa2.out_channels + 1024, [256, 256])
        self.fp2 = FeaturePropagation(self.sa1.out_channels + 256, [256, 128])
        self.fp3 = FeaturePropagation(128 + self.num_category + 6, [128, 128])
        self.fc1 = SharedMLP(128, [128])
        self.dp1 = nn.Dropout(0.5)
        self.fc2 = SharedMLP(128, [num_part], bn=False, last_activation=False)

    def forward(self, point_cloud, cls_label, lengths=None):
        _check_part_input(point_cloud, "PointNet2PartSegMSG")
        b, n = point_cloud.shape[0], point_cloud.shape[1]
        cls = category_labels(cls_label, b, point_cloud.device, "PointNet2PartSegMSG", self.num_category)
        lengths = device_lengths(lengths, b, n, point_cloud.device, "PointNet2PartSegMSG")
        mask = None if lengths is None else row_mask(lengths, n)
        l0_xyz, l0_points = point_cloud[..., :3].contiguous(), point_cloud[..., 3:].contiguous()
        l1_xyz, l1_points = self.sa1(l0_xyz, l0_points, lengths)
        l2_xyz, l2_points = self.sa2(l1_xyz, l1_points)
        l3_xyz, l3_points, _ = self.sa3(l2_xyz, l2_points)
        l2_points = self.fp1(l2_xyz, l3_xyz, l2_points, l3_points)
        l1_points = self.fp2(l1_xyz, l2_xyz, l1_points, l2_points)
        one_hot = nn.functional.one_hot(cls, self.num_category).to(l0_xyz.dtype)
        points1 = torch.cat([one_hot.unsqueeze(1).expand(b, n, self.num_category), l0_xyz, l0_points], dim=2)
        l0_points = self.fp3(l0_xyz, l1_xyz, points1, l1_points, lengths)
        feats = self.fc1(l0_points, mask)
        return self.fc2(self.dp1(feats), mask), {"feats": feats, "l1_xyz": l1_xyz}


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


def part_seg_loss(pred: torch.Tensor, label: torch.Tensor, lengths=None) -> torch.Tensor:
    """mean softmax cross entropy over the points — models/pointnet2_part_seg.py:44-51.  pred (B,N,num_part), label
    (B,N) part indices.  ``lengths`` (B,), optional: the mean over the real rows j < lengths[i] only, whatever pred and
    label hold in the padding rows (the logits are selected before the softmax, as in sem_seg_loss, so NaN logits there
    give neither a NaN loss nor a NaN gradient).  Every real point then weighs the same, so a shape counts in proportion
    to its length; the reference resamples every shape to N points, which weighs every shape equally."""
    logits = pred.reshape(-1, pred.shape[-1])
    label = label.reshape(-1).long()
    if lengths is None:
        return nn.functional.cross_entropy(logits, label)
    b, n = pred.shape[0], pred.shape[1]
    keep = row_mask(device_lengths(lengths, b, n, pred.device, "part_seg_loss"), n).reshape(-1)
    logits = torch.where(keep.unsqueeze(1), logits, 0)
    label = torch.where(keep, label, 0)
    per = nn.functional.cross_entropy(logits, label, reduction="none")
    return torch.where(keep, per, 0).sum() / keep.sum()


_OFFSETS_ON = {}


def _part_range(cls: torch.Tensor):
    """(first part, one past the last) of each category in cls, from a table copied to the device once"""
    off = _OFFSETS_ON.get(cls.device)
    if off is None:
        off = _OFFSETS_ON[cls.device] = torch.tensor(PART_OFFSETS, dtype=torch.int64, device=cls.device)
    return off[cls], off[cls + 1]


def part_seg_predict(pred: torch.Tensor, cls_label) -> torch.Tensor:
    """(B,N) int64 part labels: per shape, the argmax of pred (B,N,50) over the parts of the shape's own category, plus
    the category's first part — part_seg/train.py:274-280.  cls_label (B,): categories (see category_labels)."""
    if pred.dim() != 3 or pred.shape[-1] != PART_OFFSETS[-1]:
        raise ValueError(f"part_seg_predict expects (batch_size, num_point, {PART_OFFSETS[-1]}) logits, "
                         f"got {tuple(pred.shape)}")
    lo, hi = _part_range(category_labels(cls_label, pred.shape[0], pred.device, "part_seg_predict"))
    parts = torch.arange(pred.shape[-1], device=pred.device)
    own = (parts >= lo.unsqueeze(1)) & (parts < hi.unsqueeze(1))
    # outside the category: -inf, so the argmax (the first maximum, as numpy's) lands in the category's range
    return torch.where(own.unsqueeze(1), pred, float("-inf")).argmax(-1)


def part_seg_iou(pred_parts: torch.Tensor, label: torch.Tensor, cls_label, lengths=None) -> torch.Tensor:
    """(B,) float64: per shape, the mean over the parts of its category of |pred = p and label = p| / |pred = p or
    label = p|, a part absent from both counting 1 — part_seg/train.py:286-300.  pred_parts, label (B,N) part indices
    (part_seg_predict gives the former); cls_label (B,) categories (see category_labels).  ``lengths`` (B,), optional:
    only the rows j < lengths[i] count.  Runs on the tensors' device, with per-shape counts from scatter_add and nothing
    read back to the host.  The reference's two summaries over a test set are plain means of the result::

        ious, cats = torch.cat(per_batch_ious), torch.cat(per_batch_cls_labels)
        instance_miou = ious.mean()                                                       # over shapes
        category_miou = torch.stack([ious[cats == k].mean() for k in cats.unique()]).mean()  # over categories
    """
    if label.dim() != 2 or pred_parts.shape != label.shape:
        raise ValueError(f"part_seg_iou expects (batch_size, num_point) pred_parts and label, got "
                         f"{tuple(pred_parts.shape)} and {tuple(label.shape)}")
    b, n = label.shape
    dev = label.device
    num_part = PART_OFFSETS[-1]
    lo, hi = _part_range(category_labels(cls_label, b, dev, "part_seg_iou"))
    if lengths is None:
        keep = torch.ones(b, n, dtype=torch.bool, device=dev)
    else:
        keep = row_mask(device_lengths(lengths, b, n, dev, "part_seg_iou"), n)
    pred_parts, label = pred_parts.long(), label.long()
    base = (torch.arange(b, device=dev) * num_part).unsqueeze(1)

    def counts(parts, rows):
        """(b, num_part) int64: per shape, how many of the selected rows hold each part (out-of-range parts: none)"""
        ok = rows & (parts >= 0) & (parts < num_part)
        idx = (torch.where(ok, parts, 0) + base).reshape(-1)
        return torch.zeros(b * num_part, dtype=torch.int64, device=dev).scatter_add_(0, idx, ok.reshape(-1).long()).view(b, num_part)

    inter = counts(label, keep & (pred_parts == label))
    union = counts(label, keep) + counts(pred_parts, keep) - inter
    iou = torch.where(union > 0, inter.double() / union.clamp(min=1), 1.0)
    parts = torch.arange(num_part, device=dev)
    own = (parts >= lo.unsqueeze(1)) & (parts < hi.unsqueeze(1))
    return torch.where(own, iou, 0).sum(1) / (hi - lo)
