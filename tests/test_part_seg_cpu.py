"""CPU tests of the part segmentation nets' bookkeeping and of their loss and evaluation helpers (nets.py): parameter
counts, part_seg_loss, part_seg_predict and part_seg_iou against a direct restatement of the reference's evaluation, and
the input checks.  The nets themselves need a GPU (tests/test_part_seg_gpu.py)."""
import numpy as np
import pytest
import torch

from pointnet2_b200 import nets


def lin_bn(cin, cout):
    """one SharedMLP layer with batch norm: weight + bias, then BN gamma + beta"""
    return cin * cout + cout + 2 * cout


def stack(cin, widths):
    total = 0
    for w in widths:
        total += lin_bn(cin, w)
        cin = w
    return total


def test_part_seg_parameter_count():
    """models/pointnet2_part_seg.py:26-39, each SA level's input is its features plus the 3 centred coordinates"""
    sa1 = stack(3 + 3, [64, 64, 128])            # normals + xyz: 576 + 4288 + 8576 = 13440
    sa2 = stack(128 + 3, [128, 128, 256])        # 17152 + 16768 + 33536 = 67456
    sa3 = stack(256 + 3, [256, 512, 1024])       # 67072 + 132608 + 527360 = 727040
    fp1 = stack(256 + 1024, [256, 256])          # 328448 + 66304 = 394752
    fp2 = stack(128 + 256, [256, 128])           # 99072 + 33152 = 132224
    fp3 = stack(128 + 6, [128, 128, 128])        # 17536 + 16768 + 16768 = 51072
    fc1 = lin_bn(128, 128)                       # 16768
    fc2 = 128 * 50 + 50                          # 6450, no batch norm
    want = sa1 + sa2 + sa3 + fp1 + fp2 + fp3 + fc1 + fc2
    assert want == 1409202
    assert sum(p.numel() for p in nets.PointNet2PartSeg(50).parameters()) == want


def test_part_seg_msg_parameter_count():
    """models/pointnet2_part_seg_msg_one_hot.py:28-45; fp3 takes the 16-way one-hot, xyz and normals (22 channels)"""
    sa1 = stack(6, [32, 32, 64]) + stack(6, [64, 64, 128]) + stack(6, [64, 96, 128])  # 3648 + 13440 + 19680 = 36768
    sa2 = stack(320 + 3, [128, 128, 256]) + stack(320 + 3, [128, 196, 256])           # 92032 + 118348 = 210380
    sa3 = stack(512 + 3, [256, 512, 1024])       # 132608 + 132608 + 527360 = 792576
    fp1 = stack(512 + 1024, [256, 256])          # 393984 + 66304 = 460288
    fp2 = stack(320 + 256, [256, 128])           # 148224 + 33152 = 181376
    fp3 = stack(128 + 22, [128, 128])            # 19584 + 16768 = 36352
    fc1 = lin_bn(128, 128)                       # 16768
    fc2 = 128 * 50 + 50                          # 6450
    want = sa1 + sa2 + sa3 + fp1 + fp2 + fp3 + fc1 + fc2
    assert want == 1740958
    net = nets.PointNet2PartSegMSG(50, 16)
    assert (net.sa1.out_channels, net.sa2.out_channels) == (320, 512)
    assert sum(p.numel() for p in net.parameters()) == want


def test_part_offsets_cover_the_50_parts_of_16_categories():
    off = nets.PART_OFFSETS
    assert len(off) == nets.NUM_CATEGORIES + 1 == 17 and off[0] == 0 and off[-1] == 50
    assert all(a < b for a, b in zip(off, off[1:]))


# ------------------------------------------------------------------------------ the reference's evaluation, restated
def seg_classes():
    """category -> its part labels, as part_seg/train.py builds seg_classes from the dataset's mapping"""
    off = nets.PART_OFFSETS
    return {k: list(range(off[k], off[k + 1])) for k in range(nets.NUM_CATEGORIES)}


def ref_predict(logits, cls):
    """part_seg/train.py:277-280"""
    out = np.zeros(logits.shape[:2], np.int64)
    for i in range(logits.shape[0]):
        sc = seg_classes()[int(cls[i])]
        out[i] = np.argmax(logits[i][:, sc], 1) + sc[0]
    return out


def ref_iou(segp_all, segl_all, cls, lengths):
    """part_seg/train.py:290-300 on the first lengths[i] points of each shape"""
    res = []
    for i in range(segp_all.shape[0]):
        segp, segl = segp_all[i, :lengths[i]], segl_all[i, :lengths[i]]
        sc = seg_classes()[int(cls[i])]
        part_ious = [0.0 for _ in range(len(sc))]
        for l in sc:
            if (np.sum(segl == l) == 0) and (np.sum(segp == l) == 0):
                part_ious[l - sc[0]] = 1.0
            else:
                part_ious[l - sc[0]] = np.sum((segl == l) & (segp == l)) / float(np.sum((segl == l) | (segp == l)))
        res.append(np.mean(part_ious))
    return np.array(res)


def random_batch(seed, b=12, n=200):
    rs = np.random.RandomState(seed)
    cls = np.arange(b) % nets.NUM_CATEGORIES
    rs.shuffle(cls)
    logits = rs.randn(b, n, 50).astype(np.float32)
    off = nets.PART_OFFSETS
    label = np.empty((b, n), np.int64)
    for i, k in enumerate(cls):
        # a random subset of the category's parts, so some parts are absent from the label
        parts = rs.choice(np.arange(off[k], off[k + 1]), size=rs.randint(1, off[k + 1] - off[k] + 1), replace=False)
        label[i] = rs.choice(parts, n)
    return cls, logits, label


def test_part_seg_predict_is_the_argmax_within_the_category():
    cls, logits, _ = random_batch(0)
    got = nets.part_seg_predict(torch.from_numpy(logits), torch.from_numpy(cls))
    assert got.dtype == torch.int64
    np.testing.assert_array_equal(got.numpy(), ref_predict(logits, cls))
    # the category may come as a list; a tie picks the first maximum, as numpy's argmax
    logits[:, :, :] = 0
    got = nets.part_seg_predict(torch.from_numpy(logits), cls.tolist())
    np.testing.assert_array_equal(got.numpy(), ref_predict(logits, cls))


@pytest.mark.parametrize("with_lengths", [False, True])
def test_part_seg_iou_matches_the_reference_evaluation(with_lengths):
    b, n = 12, 200
    cls, logits, label = random_batch(1, b, n)
    pred = ref_predict(logits, cls)
    # make some predictions exact and some parts absent from both the label and the prediction
    pred[0] = label[0]
    label[1] = nets.PART_OFFSETS[cls[1]]
    pred[1] = nets.PART_OFFSETS[cls[1]]
    lengths = np.full(b, n)
    if with_lengths:
        lengths = np.array([n, 1, 2, 7, 50, 199, 100, 3, 64, 150, 200, 10])
        rs = np.random.RandomState(2)
        for i, l in enumerate(lengths):  # the padding holds any label, even out of range
            label[i, l:] = rs.randint(-5, 60, n - l)
            pred[i, l:] = rs.randint(0, 50, n - l)
    got = nets.part_seg_iou(torch.from_numpy(pred), torch.from_numpy(label), torch.from_numpy(cls),
                            lengths=lengths.tolist() if with_lengths else None)
    assert got.shape == (b,) and got.dtype == torch.float64
    np.testing.assert_allclose(got.numpy(), ref_iou(pred, label, cls, lengths), rtol=1e-12, atol=1e-12)
    assert float(got[0]) == 1.0


# ----------------------------------------------------------------------------------------------------------- loss
def test_part_seg_loss_without_lengths_is_the_mean_cross_entropy():
    torch.manual_seed(0)
    pred = torch.randn(3, 40, 50)
    label = torch.randint(0, 50, (3, 40))
    per = -torch.log_softmax(pred, -1).gather(-1, label[..., None]).squeeze(-1)
    assert abs(float(nets.part_seg_loss(pred, label)) - float(per.mean())) < 1e-6


def test_part_seg_loss_with_lengths_is_the_mean_over_the_real_rows():
    torch.manual_seed(1)
    lengths = [40, 1, 17]
    pred = torch.randn(3, 40, 50)
    label = torch.randint(0, 50, (3, 40))
    per = -torch.log_softmax(pred, -1).gather(-1, label[..., None]).squeeze(-1)
    want = torch.cat([per[i, :l] for i, l in enumerate(lengths)]).mean()
    for i, l in enumerate(lengths):  # padding: NaN and inf logits, labels out of range
        pred[i, l:, 0::2] = float("nan")
        pred[i, l:, 1::2] = float("inf")
        label[i, l:] = 1000
    p = pred.clone().requires_grad_(True)
    loss = nets.part_seg_loss(p, label, lengths=torch.tensor(lengths))
    torch.testing.assert_close(loss, want, rtol=1e-6, atol=1e-6)
    loss.backward()
    assert torch.isfinite(loss) and bool(torch.isfinite(p.grad).all())
    for i, l in enumerate(lengths):
        assert bool((p.grad[i, l:] == 0).all())


# ----------------------------------------------------------------------------------------------- input validation
@pytest.mark.parametrize("shape", [(2, 64, 3), (2, 64, 7), (64, 6)])
def test_part_nets_refuse_a_point_cloud_without_normals(shape):
    x = torch.zeros(shape)
    with pytest.raises(ValueError, match="6"):
        nets.PointNet2PartSeg()(x)
    with pytest.raises(ValueError, match="6"):
        nets.PointNet2PartSegMSG()(x, torch.zeros(2, dtype=torch.int64))


@pytest.mark.parametrize("cls_label", [[0, 16], [-1, 3], [0, 1, 2], [[0], [1]], [0.5, 1.0], torch.tensor([3, 16])])
def test_part_seg_msg_refuses_bad_categories(cls_label):
    with pytest.raises(ValueError, match="cls_label"):
        nets.PointNet2PartSegMSG()(torch.zeros(2, 64, 6), cls_label)


def test_part_nets_refuse_bad_lengths_before_any_kernel():
    with pytest.raises(ValueError, match="lengths"):
        nets.PointNet2PartSeg()(torch.zeros(2, 64, 6), lengths=[64, 65])
    with pytest.raises(ValueError, match="lengths"):
        nets.PointNet2PartSegMSG()(torch.zeros(2, 64, 6), [0, 1], lengths=[0, 3])


def test_helpers_refuse_bad_shapes():
    with pytest.raises(ValueError):
        nets.part_seg_predict(torch.zeros(2, 8, 13), [0, 1])
    with pytest.raises(ValueError, match="cls_label"):
        nets.part_seg_predict(torch.zeros(2, 8, 50), [0, 17])
    with pytest.raises(ValueError):
        nets.part_seg_iou(torch.zeros(2, 8, dtype=torch.long), torch.zeros(2, 9, dtype=torch.long), [0, 1])
