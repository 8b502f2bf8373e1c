"""CPU tests of the shape batches: the numpy oracle (shape_oracle.py) against a literal restatement of the
utils/provider.py augmentation functions and the loaders' row handling with np.random replaced by the same draws,
pc_normalize against modelnet_dataset.py:15-21, ShapeSet's refusals, the argument errors of sample_shapes / vote_batch
and the C entry's refusals (no launch), cls_accuracy against numpy, and the new kernel's resources."""
import ctypes
import os
import re
import shutil
import subprocess
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import crop_oracle as CO  # noqa: E402
import shape_oracle as SO  # noqa: E402

from pointnet2_b200 import _lib, shapes as SH  # noqa: E402


# ---- literal restatements of provider.py (float64 buffers: the definition rounds once, at the end) ----------------
def rotate_point_cloud(batch_data, angles):
    rotated_data = np.zeros(batch_data.shape, dtype=np.float64)
    for k in range(batch_data.shape[0]):
        cosval, sinval = np.cos(angles[k]), np.sin(angles[k])
        rotation_matrix = np.array([[cosval, 0, sinval], [0, 1, 0], [-sinval, 0, cosval]])
        rotated_data[k, :, 0:3] = np.dot(batch_data[k, :, 0:3].reshape((-1, 3)), rotation_matrix)
        if batch_data.shape[2] == 6:  # rotate_point_cloud_with_normal
            rotated_data[k, :, 3:6] = np.dot(batch_data[k, :, 3:6].reshape((-1, 3)), rotation_matrix)
    return rotated_data


def rotate_perturbation_point_cloud(batch_data, randn3, angle_sigma=0.06, angle_clip=0.18):
    rotated_data = np.zeros(batch_data.shape, dtype=np.float64)
    for k in range(batch_data.shape[0]):
        angles = np.clip(angle_sigma * randn3[k], -angle_clip, angle_clip)
        Rx = np.array([[1, 0, 0], [0, np.cos(angles[0]), -np.sin(angles[0])], [0, np.sin(angles[0]), np.cos(angles[0])]])
        Ry = np.array([[np.cos(angles[1]), 0, np.sin(angles[1])], [0, 1, 0], [-np.sin(angles[1]), 0, np.cos(angles[1])]])
        Rz = np.array([[np.cos(angles[2]), -np.sin(angles[2]), 0], [np.sin(angles[2]), np.cos(angles[2]), 0], [0, 0, 1]])
        R = np.dot(Rz, np.dot(Ry, Rx))
        rotated_data[k, :, 0:3] = np.dot(batch_data[k, :, 0:3].reshape((-1, 3)), R)
        if batch_data.shape[2] == 6:
            rotated_data[k, :, 3:6] = np.dot(batch_data[k, :, 3:6].reshape((-1, 3)), R)
    return rotated_data


def random_scale_point_cloud(batch_data, u, scale_low=0.8, scale_high=1.25):
    scales = scale_low + (scale_high - scale_low) * u  # np.random.uniform(low, high, B)
    for batch_index in range(batch_data.shape[0]):
        batch_data[batch_index, :, :] *= scales[batch_index]
    return batch_data


def shift_point_cloud(batch_data, u, shift_range=0.1):
    shifts = -shift_range + 2 * shift_range * u  # np.random.uniform(-shift_range, shift_range, (B, 3))
    for batch_index in range(batch_data.shape[0]):
        batch_data[batch_index, :, :] += shifts[batch_index, :]
    return batch_data


def jitter_point_cloud(batch_data, randn, sigma=0.01, clip=0.05):
    jittered_data = np.clip(sigma * randn, -1 * clip, clip)
    jittered_data += batch_data
    return jittered_data


def augment_batch_data(batch_data, draws):
    """modelnet_dataset.py:60-72 with each np.random call replaced by the injected draws; shuffle_points becomes one
    permutation per shape."""
    rotated_data = rotate_point_cloud(batch_data, draws["angle"])
    rotated_data = rotate_perturbation_point_cloud(rotated_data, draws["randn3"])
    jittered_data = random_scale_point_cloud(rotated_data[:, :, 0:3], draws["scale_u"])
    jittered_data = shift_point_cloud(jittered_data, draws["shift_u"])
    jittered_data = jitter_point_cloud(jittered_data, draws["jitter_randn"])
    rotated_data[:, :, 0:3] = jittered_data
    return np.stack([rotated_data[k, draws["perm"][k]] for k in range(len(rotated_data))])


def _set_arrays(rs, sizes, normals=True):
    xyz = [rs.standard_normal((n, 3)).astype(np.float32) for n in sizes]
    nrm = [rs.standard_normal((n, 3)).astype(np.float32) for n in sizes]
    lab = rs.randint(0, 40, len(sizes))
    return xyz, nrm if normals else None, lab


def _packed(xyz, nrm):
    off = np.concatenate([[0], np.cumsum([len(x) for x in xyz])])
    return np.concatenate(xyz), (np.concatenate(nrm) if nrm is not None else None), off


@pytest.mark.parametrize("with_normals", [False, True])
@pytest.mark.parametrize("seed", [0, 7, -3, 2 ** 64 - 9])
def test_modelnet_recipe_matches_literal_provider(with_normals, seed):
    rs = np.random.RandomState(5)
    npoints = 64
    sizes = [100, 64, 30]   # above, at and below npoints: the loader's first-npoints truncation
    xyz, nrm, lab = _set_arrays(rs, sizes)
    pxyz, pnrm, off = _packed(xyz, nrm)
    o = SO.oracle_shapes(pxyz, lab, off, np.arange(3), seed, npoints=npoints, with_normals=with_normals, normals=pnrm)
    for e, n in enumerate(sizes):
        m = min(n, npoints)
        order = SO.row_order(seed, e, m)   # output row r is shape row order[r]
        inv = np.argsort(order)            # shape row k lands in output row inv[k]
        pts = xyz[e][:m] if not with_normals else np.concatenate([xyz[e][:m], nrm[e][:m]], 1)
        draws = {"angle": [CO.unit(CO.draw(seed, 4, e, 0)) * 2 * np.pi],
                 "randn3": [SO.normal(seed, 5, e, np.arange(3))],
                 "scale_u": np.array([CO.unit(CO.draw(seed, 6, e, 0))]),
                 "shift_u": CO.unit(CO.draw(seed, 7, e, np.arange(3)))[None],
                 "jitter_randn": SO.normal(seed, 8, e, 3 * inv[:, None] + np.arange(3))[None],
                 "perm": [order]}
        want = augment_batch_data(pts[None].astype(np.float64), draws)[0]
        assert o["lengths"][e] == m
        np.testing.assert_array_equal(o["point_idx"][e, :m], off[e] + order)
        np.testing.assert_allclose(o["points64"][e, :m], want, rtol=0, atol=1e-12)
        assert (o["points"][e, m:] == 0).all() and (o["point_idx"][e, m:] == -1).all()
        assert o["label"][e] == lab[e]


@pytest.mark.parametrize("seed", [1, 99])
def test_part_recipe_matches_literal_loader(seed):
    """part_dataset_all_normal.py:83-112 + part_seg/train.py:200: rows drawn from all P (here without replacement, the
    m smallest keys), jitter on xyz only, normals and part labels carried along."""
    rs = np.random.RandomState(6)
    sizes = [3000, 500]
    xyz, nrm, lab = _set_arrays(rs, sizes)
    part = [rs.randint(0, 50, n) for n in sizes]
    pxyz, pnrm, off = _packed(xyz, nrm)
    npoints = 2048
    o = SO.oracle_shapes(pxyz, lab, off, [0, 1], seed, npoints=npoints, subset="random", rotate=False, perturb=False,
                         scale=None, shift=0, with_normals=True, normals=pnrm, part=np.concatenate(part))
    for e, n in enumerate(sizes):
        m = min(n, npoints)
        choice = SO.row_order(seed, e, n)[:m]
        point_set, normal, seg = xyz[e][choice], nrm[e][choice], part[e][choice]
        jit = jitter_point_cloud(point_set[None].astype(np.float64),
                                 SO.normal(seed, 8, e, 3 * np.arange(m)[:, None] + np.arange(3))[None])[0]
        assert o["lengths"][e] == m
        np.testing.assert_allclose(o["points64"][e, :m, :3], jit, rtol=0, atol=1e-12)
        np.testing.assert_array_equal(o["points"][e, :m, 3:], normal)
        np.testing.assert_array_equal(o["part"][e, :m], seg)
        assert len(np.unique(o["point_idx"][e, :m])) == m   # without replacement
    assert o["lengths"][0] == npoints and o["lengths"][1] == 500


def test_votes_match_rotate_by_angle():
    rs = np.random.RandomState(7)
    xyz, _, lab = _set_arrays(rs, [50, 80], normals=False)
    pxyz, _, off = _packed(xyz, None)
    nv, npoints = 4, 64
    o = SO.oracle_shapes(pxyz, lab, off, [1, 0], 3, npoints=npoints, votes=nv)
    for e in range(2 * nv):
        v, i = e // 2, e % 2
        s = [1, 0][i]
        m = min(len(xyz[s]), npoints)
        order = SO.row_order(3, e, m)
        want = rotate_point_cloud(xyz[s][:m][order][None].astype(np.float64), [v / float(nv) * np.pi * 2])[0]
        np.testing.assert_allclose(o["points64"][e, :m], want, rtol=0, atol=1e-12)
        assert o["label"][e] == lab[s]


def test_dropout_removes_rows():
    """random_point_dropout (provider.py:227-234) with the draws, rows removed instead of overwritten with row 0."""
    rs = np.random.RandomState(8)
    xyz, _, lab = _set_arrays(rs, [500], normals=False)
    pxyz, _, off = _packed(xyz, None)
    for seed in range(6):
        o = SO.oracle_shapes(pxyz, lab, off, [0], seed, npoints=256, max_dropout=0.875)
        order = SO.row_order(seed, 0, 256)
        dropout_ratio = CO.unit(CO.draw(seed, 2, 0, 0)) * 0.875
        drop_idx = np.where(CO.unit(CO.draw(seed, 3, 0, np.arange(256))) <= dropout_ratio)[0]
        keep = np.setdiff1d(np.arange(256), drop_idx[drop_idx > 0])
        assert o["lengths"][0] == len(keep)
        np.testing.assert_array_equal(o["point_idx"][0, :len(keep)], order[keep])


def test_pc_normalize_matches_reference_expression():
    rs = np.random.RandomState(9)
    pc = (rs.standard_normal((1000, 3)) * [3, 1, 2] + 5).astype(np.float32)
    centroid = np.mean(pc, axis=0)   # modelnet_dataset.py:15-21 as written
    ref = pc - centroid
    m = np.max(np.sqrt(np.sum(ref ** 2, axis=1)))
    ref = ref / m
    got = SH.pc_normalize(pc)
    assert got.dtype == np.float32
    np.testing.assert_array_equal(got, ref)
    ss = SH.ShapeSet([pc, pc[:10]], [3, np.int64(4)], device="cpu")
    np.testing.assert_array_equal(ss.xyz.numpy()[:1000], ref)
    np.testing.assert_array_equal(ss.xyz.numpy()[1000:], SH.pc_normalize(pc[:10]))
    raw = SH.ShapeSet([pc], [0], normalize=False, device="cpu")
    np.testing.assert_array_equal(raw.xyz.numpy(), pc)


def test_shape_set_packs_and_refuses():
    a = np.array([[0, 0, 0], [1, 2, 3]], np.float32)
    b = np.array([[5, 5, 1], [6, 7, 2], [5.5, 5, 1.5]], np.float32)
    ss = SH.ShapeSet([a, torch.from_numpy(b)], [1, torch.tensor(2)], normal_list=[a, b], part_list=[[0, 1], [2, 3, 4]],
                     normalize=False, device="cpu")
    assert len(ss) == 2 and ss.offsets.tolist() == [0, 2, 5] and ss.label.tolist() == [1, 2]
    assert ss.part.dtype == torch.int32 and ss.part.tolist() == [0, 1, 2, 3, 4] and ss.normals.shape == (5, 3)
    with pytest.raises(ValueError, match="at least one shape"):
        SH.ShapeSet([], [], device="cpu")
    with pytest.raises(ValueError, match="1 to 16384"):
        SH.ShapeSet([np.zeros((0, 3), np.float32)], [0], device="cpu")
    with pytest.raises(ValueError, match="1 to 16384"):
        SH.ShapeSet([np.zeros((16385, 3), np.float32)], [0], device="cpu")
    with pytest.raises(ValueError, match="NaN or inf"):
        SH.ShapeSet([np.array([[0, 0, 0], [np.nan, 0, 1]], np.float32)], [0], device="cpu")
    with pytest.raises(ValueError, match="NaN or inf normals"):
        SH.ShapeSet([a], [0], normal_list=[np.array([[0, 0, 0], [np.inf, 0, 1]], np.float32)], device="cpu")
    with pytest.raises(ValueError, match="radius 0"):
        SH.ShapeSet([np.ones((4, 3), np.float32)], [0], device="cpu")
    with pytest.raises(ValueError, match="outside"):
        SH.ShapeSet([a], [40], device="cpu")
    with pytest.raises(ValueError, match="outside"):
        SH.ShapeSet([a], [-1], device="cpu")
    with pytest.raises(TypeError, match="one integer"):
        SH.ShapeSet([a], [1.0], device="cpu")
    with pytest.raises(TypeError, match="one integer"):
        SH.ShapeSet([a], [[1, 2]], device="cpu")
    with pytest.raises(ValueError, match="one label per shape"):
        SH.ShapeSet([a, a], [1], device="cpu")
    with pytest.raises(ValueError, match="one normal array per shape"):
        SH.ShapeSet([a, a], [1, 1], normal_list=[a], device="cpu")
    with pytest.raises(ValueError, match="normals of shape"):
        SH.ShapeSet([a], [1], normal_list=[b], device="cpu")
    with pytest.raises(ValueError, match="part labels of shape"):
        SH.ShapeSet([a], [1], part_list=[[1, 2, 3]], device="cpu")
    with pytest.raises(TypeError, match="part labels"):
        SH.ShapeSet([a], [1], part_list=[np.ones(2, np.float32)], device="cpu")
    with pytest.raises(ValueError, match="part labels outside"):
        SH.ShapeSet([a], [1], part_list=[[-1, 0]], device="cpu")
    with pytest.raises(ValueError, match="num_points, 3"):
        SH.ShapeSet([np.zeros((2, 4), np.float32)], [0], device="cpu")
    with pytest.raises(ValueError, match="num_class"):
        SH.ShapeSet([a], [0], num_class=0, device="cpu")


def test_point_count_limit():
    """P >= 2^31 - 1 in all is refused before any shape is converted (broadcast views: no memory behind them)."""
    x = np.broadcast_to(np.float32(1), (16384, 3))
    with pytest.raises(ValueError, match="2\\^31 - 1"):
        SH.ShapeSet([x] * (2 ** 17), [0] * (2 ** 17), device="cpu")


def test_argument_errors_launch_nothing():
    before = _lib.launch_count()
    a = np.array([[0, 0, 0], [1, 2, 3]], np.float32)
    ss = SH.ShapeSet([a], [1], device="cpu")
    idx = torch.zeros(4, dtype=torch.int64)
    with pytest.raises(RuntimeError, match="no CPU path"):
        SH.sample_shapes(ss, idx, 0)
    with pytest.raises(TypeError, match="ShapeSet"):
        SH.sample_shapes(object(), idx, 0)
    with pytest.raises(ValueError, match="npoints"):
        SH.sample_shapes(ss, idx, 0, npoints=0)
    with pytest.raises(ValueError, match="16384"):
        SH.sample_shapes(ss, idx, 0, npoints=16385)
    with pytest.raises(ValueError, match="normals"):
        SH.sample_shapes(ss, idx, 0, with_normals=True)
    for kw, err, pat in [(dict(subset="all"), ValueError, "subset"), (dict(rotate=1), TypeError, "rotate"),
                         (dict(scale=(1.2, 0.8)), ValueError, "scale"), (dict(scale=0.8), TypeError, "scale"),
                         (dict(jitter=(0.01, 0)), ValueError, "jitter"), (dict(shift=-0.1), ValueError, "shift"),
                         (dict(shift=float("inf")), ValueError, "shift"), (dict(max_dropout=1.5), ValueError, "max_dropout"),
                         (dict(max_dropout=float("nan")), ValueError, "max_dropout")]:
        with pytest.raises(err, match=pat):
            SH.sample_shapes(ss, idx, 0, **kw)
    # the checks that need a CUDA set: a fake one whose tensors are on the CPU but claims a CUDA device
    fake = SH.ShapeSet([a], [1], normal_list=[a], device="cpu")
    fake.device = torch.device("cuda", 0)
    with pytest.raises(RuntimeError, match="no CPU path"):
        SH.sample_shapes(fake, idx, 0)                                     # shape_idx on the CPU
    with pytest.raises(TypeError, match="integer"):
        SH.sample_shapes(fake, idx.float(), 0)
    with pytest.raises(ValueError, match="shape_idx"):
        SH.sample_shapes(fake, torch.zeros(2, 2, dtype=torch.int64), 0)
    with pytest.raises(TypeError, match="shape_idx"):
        SH.sample_shapes(fake, [0, 1], 0)
    with pytest.raises(ValueError, match="num_votes"):
        SH.vote_batch(fake, idx, 0, 0)
    with pytest.raises(ValueError, match="chunk"):
        SH.classify_votes(None, fake, idx, 2, 0, chunk=0)
    assert _lib.launch_count() == before


def test_abi_refusals():
    lib = _lib.load()
    before = _lib.launch_count()
    null = ctypes.c_void_p(0)
    one = ctypes.c_void_p(256)  # never dereferenced: every call below is refused first

    def call(s=2, p=1000, max_shape=600, b=4, votes=0, npoints=1024, subset=0, rotate=1, perturb=1, scale_on=1,
             scale=(0.8, 1.25), shift=0.1, jitter_on=1, jitter=(0.01, 0.05), max_dropout=0.0, with_normals=0, ptrs=None):
        q = ptrs or {}
        g = lambda k: q.get(k, one)  # noqa: E731
        return lib.pn2_shape_batch(s, p, max_shape, g("xyz"), g("nrm"), g("label"), g("part"), g("off"), b, g("idx"), 5,
                                   null, votes, npoints, subset, rotate, perturb, scale_on, scale[0], scale[1], shift,
                                   jitter_on, jitter[0], jitter[1], max_dropout, with_normals, g("pts"), g("lab"),
                                   g("opart"), g("len"), g("pi"), null)
    assert call(s=0) == 1
    assert call(p=0) == 1
    assert call(p=2 ** 31 - 1) == 1
    assert call(max_shape=0) == 1
    assert call(max_shape=1001) == 1
    assert call(p=20000, max_shape=16385) == 1
    assert call(b=0) == 1
    assert call(votes=-1) == 1
    assert call(npoints=0) == 1
    assert call(npoints=16385) == 1
    assert call(b=60000, npoints=16384) == 1           # E * npoints * 3 >= 2^31
    assert call(b=30000, npoints=16384, with_normals=1) == 1
    assert call(subset=2) == 1
    assert call(rotate=2) == 1
    assert call(scale=(1.3, 1.2)) == 1
    assert call(scale=(float("nan"), 1.2)) == 1
    assert call(shift=-0.1) == 1
    assert call(shift=float("inf")) == 1
    assert call(jitter=(0.01, 0.0)) == 1
    assert call(jitter=(-0.01, 0.05)) == 1
    assert call(max_dropout=1.01) == 1
    assert call(max_dropout=float("nan")) == 1
    assert call(votes=3) == 1                            # a vote takes no augmentation
    for k in ("xyz", "label", "off", "idx", "pts", "lab", "len", "pi"):
        assert call(ptrs={k: null}) == 1, k
    assert call(with_normals=1, ptrs={"nrm": null}) == 1
    assert call(ptrs={"part": null}) == 1                # part output without part labels
    assert _lib.launch_count() == before


def test_cls_accuracy_matches_numpy():
    rs = np.random.RandomState(10)
    nc = 7
    label = rs.randint(0, nc, 500)
    pred = np.where(rs.random_sample(500) < 0.6, label, rs.randint(0, nc, 500))
    acc, cacc = SH.cls_accuracy(torch.from_numpy(pred), torch.from_numpy(label), nc)
    seen = np.array([np.sum(label == c) for c in range(nc)])
    correct = np.array([np.sum((pred == label) & (label == c)) for c in range(nc)])
    assert acc.item() == np.sum(pred == label) / float(len(label))
    assert cacc.item() == np.mean(correct / seen.astype(np.float64))
    _, cnan = SH.cls_accuracy(torch.tensor([0, 1]), torch.tensor([0, 1]), 3)  # class 2 unseen: NaN, as numpy's 0 / 0
    assert np.isnan(cnan.item())


def test_shape_kernel_does_not_spill():
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(cuobjdump):
        pytest.skip("cuobjdump not available")
    out = subprocess.run([cuobjdump, "-res-usage", _lib.lib_path()], capture_output=True, text=True).stdout
    found = re.findall(r"Function (\S*shape_batch_kernel\S*):\s*\n\s*REG:(\d+) STACK:(\d+)", out)
    assert len(found) == 1, found
    assert all(stack == "0" for _, _, stack in found), found
