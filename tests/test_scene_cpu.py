"""CPU tests of whole-scene segmentation: the numpy oracle of the block partition against the reference's own loop
(scannet_dataset.py:94-103), grid planning, the sub-block split, the torch voxel restatement against pc_util.py:39-51,
the whole-scene metric accumulation and the argument errors (no launch)."""
import ctypes
import math
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import scene_oracle as SO  # noqa: E402

from pointnet2_b200 import _lib, scene, workloads as W  # noqa: E402


def _scenes():
    rs = np.random.RandomState(3)
    yield "room", W.scene_room(30000, 1)[0]
    yield "uniform", (rs.random_sample((20000, 3)) * [7.3, 4.1, 2.5]).astype(np.float32)
    # coordinates on block boundaries and one float32 ulp either side
    base = np.array([0.0, 1.5, 3.0, 4.5, 1.7, 1.3, 1.499, 1.501], np.float32)
    edge = np.concatenate([base, np.nextafter(base, np.float32(-1)), np.nextafter(base, np.float32(9))])
    g = np.stack(np.meshgrid(edge, edge, [0.0, 1.0]), -1).reshape(-1, 3).astype(np.float32)
    yield "edges", g
    yield "offset", (rs.random_sample((5000, 3)) * [4, 4, 1] + [1000.25, -371.5, 3]).astype(np.float32)


@pytest.mark.parametrize("name,xyz", list(_scenes()), ids=[n for n, _ in _scenes()])
def test_oracle_matches_reference_loop(name, xyz):
    """For every block the oracle keeps (stride = size = 1.5, padding 0.2, no split), the context set and core mask
    equal the reference's for the same (i, j); every block the reference forms and the oracle drops has no core."""
    ref = SO.reference_blocks(xyz)
    o = SO.oracle_scene_blocks(xyz, max_points=len(xyz))
    assert (o["block"][:, 2] == 0).all()
    kept = set()
    for s in range(len(o["lengths"])):
        i, j, _ = o["block"][s]
        kept.add((i, j))
        assert (i, j) in ref, (name, i, j)
        members, core = ref[(i, j)]
        c = o["lengths"][s]
        np.testing.assert_array_equal(o["point_idx"][s, :c], members)
        np.testing.assert_array_equal(o["core"][s, :c], core)
    for key, (_, core) in ref.items():
        if key not in kept:
            assert not core.any(), (name, key)
    assert (np.diff(o["occ_off"]) >= 1).all()  # every point is scored somewhere


def test_grid_planning():
    gs = scene.grid_size
    assert gs(0.0, 3.0, 1.5, 1.5) == 2            # extent an exact multiple of the stride
    assert gs(0.0, 4.5, 1.5, 1.5) == 3
    assert gs(0.0, 3.0, 1.5, 0.5) == 4
    assert gs(0.0, 3.0000001, 1.5, 1.5) == 3
    assert gs(2.0, 2.0, 1.5, 1.5) == 1            # extent 0
    assert gs(-7.25, -7.25, 1.5, 0.5) == 1
    assert gs(0.0, 1.5, 1.5, 0.25) == 1
    rs = np.random.RandomState(0)
    for _ in range(2000):
        lo = float(np.float32(rs.uniform(-100, 100)))
        hi = float(np.float32(lo + rs.choice([0, rs.uniform(0, 40), 1.5 * rs.randint(0, 20)])))
        s = float(rs.choice([1.5, 1.0, 2.0]))
        t = float(rs.choice([s, s / 3, 0.5]))
        assert gs(lo, hi, s, t) == SO.plan_axis(lo, hi, s, t)
    # a single point: one block, the point is its core
    o = SO.oracle_scene_blocks(np.array([[3.0, -2.0, 1.0]], np.float32))
    assert o["lengths"].tolist() == [1] and o["occ_row"].tolist() == [0] and o["occ_off"].tolist() == [0, 1]


def test_split_arithmetic():
    ctx = np.array([0, 5, 64, 65, 200, 1000, 7], np.int64)
    core = np.array([0, 1, 3, 0, 9, 1, 7], np.int64)
    sub_begin, k, lengths, sub = scene.split_plan(ctx, core, 64)
    assert k.tolist() == [0, 1, 1, 0, 4, 16, 1]
    assert sub_begin.tolist() == [0, 0, 1, 2, 2, 6, 22]
    for blk in range(len(ctx)):
        rows = np.arange(ctx[blk])
        got = lengths[sub_begin[blk]:sub_begin[blk] + k[blk]]
        want = [len(rows[q::k[blk]]) for q in range(k[blk])]
        assert got.tolist() == want
        assert all(v <= 64 for v in got) and got.sum() == (ctx[blk] if k[blk] else 0)
        assert sub[sub_begin[blk]:sub_begin[blk] + k[blk], 0].tolist() == [blk] * k[blk]
        assert sub[sub_begin[blk]:sub_begin[blk] + k[blk], 1].tolist() == list(range(k[blk]))
    # the oracle with splits: every member in exactly one sub-block, rank r at sub-block r mod k, row r div k
    xyz = W.scene_room(20000, 4)[0]
    whole = SO.oracle_scene_blocks(xyz, max_points=len(xyz))
    split = SO.oracle_scene_blocks(xyz, max_points=300)
    for s in range(len(whole["lengths"])):
        i, j, _ = whole["block"][s]
        members = whole["point_idx"][s, :whole["lengths"][s]]
        sel = np.nonzero((split["block"][:, 0] == i) & (split["block"][:, 1] == j))[0]
        k = len(sel)
        assert k == math.ceil(len(members) / 300)
        for q, t in enumerate(sel):
            assert split["block"][t, 2] == q
            np.testing.assert_array_equal(split["point_idx"][t, :split["lengths"][t]], members[q::k])
    assert split["occ_row"].shape == whole["occ_row"].shape


def _voxel_cases():
    rs = np.random.RandomState(5)
    room, lab = W.scene_room(20000, 2)
    yield room, lab, 0.02
    yield room, np.stack([lab, rs.randint(0, 21, len(lab))], 1), 0.0484
    # on the maximum of every axis: index == nvox, which aliases the next row's key
    pts = (rs.randint(0, 6, (3000, 3)) * 0.0484).astype(np.float32)
    yield pts, rs.randint(0, 21, (3000, 2)), 0.0484
    # keys above 2^24: float32 rounds neighbouring keys together
    big = (rs.random_sample((40000, 3)) * [40, 30, 3]).astype(np.float32)
    yield big, rs.randint(0, 21, 40000), 0.01


@pytest.mark.parametrize("case", range(4))
def test_voxel_labels_match_pc_util(case):
    pts, lab, res = list(_voxel_cases())[case]
    want_k, want_l, want_n = SO.reference_voxel_labels(pts, lab, res)
    assert want_k.dtype == np.float32  # numpy keeps float32 input in float32
    keys, labels, nvox = scene.surface_voxel_labels(torch.from_numpy(pts), torch.from_numpy(lab), res)
    assert keys.dtype == torch.float32 and nvox.dtype == torch.float32
    np.testing.assert_array_equal(nvox.numpy(), want_n)
    np.testing.assert_array_equal(keys.numpy(), want_k)
    np.testing.assert_array_equal(labels.numpy(), want_l)
    if case == 3:
        assert want_k.max() > 2 ** 24


def test_voxel_accuracy_matches_train_loop():
    """VoxelAccuracy against train.py:401-419 restated on one scene (all points scored)."""
    rs = np.random.RandomState(8)
    acc = scene.VoxelAccuracy()
    seen = np.zeros(21)
    correct = np.zeros(21)
    tc = ts = 0
    for seed in range(3):
        pts, lab = W.scene_room(15000, seed)
        pred = np.where(rs.random_sample(len(lab)) < 0.7, lab, rs.randint(0, 21, len(lab)))
        acc.update(torch.from_numpy(pts), torch.from_numpy(lab), torch.from_numpy(pred))
        _, uv, _ = SO.reference_voxel_labels(pts, np.stack([lab, pred], 1), res=0.02)
        tc += np.sum((uv[:, 0] == uv[:, 1]) & (uv[:, 0] > 0))
        ts += np.sum(uv[:, 0] > 0)
        for c in range(21):
            seen[c] += np.sum(uv[:, 0] == c)
            correct[c] += np.sum((uv[:, 0] == c) & (uv[:, 1] == c))
    r = acc.results()
    assert r["accuracy"] == pytest.approx(tc / ts, rel=1e-12)
    per = correct[1:] / (seen[1:] + 1e-6)
    assert r["class_accuracy"] == pytest.approx(per.mean(), rel=1e-12)
    w = np.array(scene.CALIBRATION_WEIGHTS)
    assert len(w) == 20
    assert r["calibrated_accuracy"] == pytest.approx(np.average(per, weights=w), rel=1e-12)


def test_scene_room_is_seeded_and_labelled():
    a, la = W.scene_room(50000, 7)
    b, lb = W.scene_room(50000, 7)
    assert a.shape == (50000, 3) and a.dtype == np.float32 and la.dtype == np.int64
    np.testing.assert_array_equal(a, b)
    np.testing.assert_array_equal(la, lb)
    assert la.min() >= 0 and la.max() <= 20 and {0, 1, 2} <= set(la.tolist())
    assert len(np.unique(a, axis=0)) < len(a)  # duplicates
    assert np.isfinite(a).all() and a[:, 2].min() >= 0


def test_argument_errors_launch_nothing():
    before = _lib.launch_count()
    x = torch.zeros(10, 3)
    with pytest.raises(RuntimeError, match="no CPU path"):
        scene.scene_blocks(x)
    with pytest.raises(TypeError):
        scene.scene_blocks(x.double())
    with pytest.raises(TypeError):
        scene.scene_blocks(np.zeros((10, 3), np.float32))
    with pytest.raises(ValueError, match="num_points, 3"):
        scene.scene_blocks(torch.zeros(10, 4))
    with pytest.raises(ValueError, match="num_points, 3"):
        scene.scene_blocks(torch.zeros(0, 3))
    with pytest.raises(ValueError, match="stride"):
        scene.scene_blocks(x, block_size=1.0, stride=1.5)   # gaps between blocks
    with pytest.raises(ValueError, match="stride"):
        scene.scene_blocks(x, stride=0.0)
    with pytest.raises(ValueError, match="block_size"):
        scene.scene_blocks(x, block_size=-1.0)
    with pytest.raises(ValueError, match="padding"):
        scene.scene_blocks(x, padding=-0.1)
    with pytest.raises(ValueError, match="finite"):
        scene.scene_blocks(x, padding=float("inf"))
    with pytest.raises(ValueError, match="max_points"):
        scene.scene_blocks(x, max_points=0)
    with pytest.raises(TypeError, match="max_points"):
        scene.scene_blocks(x, max_points=8192.0)
    with pytest.raises(ValueError, match="batch_size"):
        scene.predict_scene(lambda *a: None, x, batch_size=0)
    i32 = lambda *s: torch.zeros(*s, dtype=torch.int32)  # noqa: E731
    blocks = scene.SceneBlocks(torch.zeros(2, 4, 3), i32(2), i32(2, 4), torch.zeros(2, 4, dtype=torch.bool), i32(2, 3),
                               i32(6), i32(5))
    with pytest.raises(ValueError, match="logits"):
        scene.merge_block_logits(blocks, torch.zeros(2, 5, 3), torch.zeros(5, 3))
    with pytest.raises(ValueError, match="accum"):
        scene.merge_block_logits(blocks, torch.zeros(2, 4, 3), torch.zeros(5, 4))
    with pytest.raises(ValueError, match="row_begin"):
        scene.merge_block_logits(blocks, torch.zeros(1, 4, 3), torch.zeros(5, 3), row_begin=2)
    with pytest.raises(ValueError, match="row_begin"):
        scene.merge_block_logits(blocks, torch.zeros(2, 4, 3), torch.zeros(5, 3), row_begin=4)
    with pytest.raises(RuntimeError, match="no CPU path"):
        scene.merge_block_logits(blocks, torch.zeros(2, 4, 3), torch.zeros(5, 3))
    with pytest.raises(TypeError):
        scene.merge_block_logits(blocks, torch.zeros(2, 4, 3, dtype=torch.float64), torch.zeros(5, 3))
    assert _lib.launch_count() == before


def test_scene_kernels_do_not_spill():
    import re
    import shutil
    import subprocess
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(cuobjdump):
        pytest.skip("cuobjdump not available")
    out = subprocess.run([cuobjdump, "-res-usage", _lib.lib_path()], capture_output=True, text=True).stdout
    found = re.findall(r"Function (\S*scene_\w+_kernel\S*):\s*\n\s*REG:\d+ STACK:(\d+)", out)
    assert len(found) == 6, found  # count, scan, fill and the merge in three dtypes
    assert all(stack == "0" for _, stack in found), found


def test_abi_refusals():
    lib = _lib.load()
    before = _lib.launch_count()
    null = ctypes.c_void_p(0)
    one = ctypes.c_void_p(256)  # never dereferenced: every call below is refused first
    assert lib.pn2_scene_blocks_workspace_bytes(0, 1, 1) == 0
    assert lib.pn2_scene_blocks_workspace_bytes(10, 200, 200) == 0  # more than 16384 blocks
    assert lib.pn2_scene_blocks_workspace_bytes(10**7, 60, 60) >= 4 * 60 * 60 * 1024
    ws = lib.pn2_scene_blocks_workspace_bytes(1000, 2, 2)
    geo = (0.0, 0.0, 1.5, 1.5, 0.2)
    assert lib.pn2_scene_blocks_count(1000, null, *geo, 2, 2, one, one, ws, null) == 1
    assert lib.pn2_scene_blocks_count(1000, one, *geo, 2, 2, one, one, ws - 1, null) == 1
    assert lib.pn2_scene_blocks_count(1000, one, 0.0, 0.0, 1.5, 2.0, 0.2, 2, 2, one, one, ws, null) == 1  # stride > size
    assert lib.pn2_scene_blocks_count(1000, one, 0.0, 0.0, 1.5, 1.5, -0.2, 2, 2, one, one, ws, null) == 1
    assert lib.pn2_scene_blocks_count(0, one, *geo, 2, 2, one, one, ws, null) == 1
    assert lib.pn2_scene_blocks_fill(1000, one, *geo, 2, 2, one, one, 4, 1 << 29, one, one, one, one, one, one, ws, null) == 1
    assert lib.pn2_scene_blocks_fill(1000, one, *geo, 2, 2, one, null, 4, 8, one, one, one, one, one, one, ws, null) == 1
    assert lib.pn2_scene_merge_typed(3, 10, 4, 2, 8, 0, 16, one, one, one, one, one, one, null) == 1      # dtype
    assert lib.pn2_scene_merge_typed(0, 10, 4, 2, 8, 0, 17, one, one, one, one, one, one, null) == 1      # past b*n
    assert lib.pn2_scene_merge_typed(0, 10, 4, 2, 8, 9, 8, one, one, one, one, one, one, null) == 1       # reversed
    assert lib.pn2_scene_merge_typed(0, 10, 4, 2, 8, 0, 16, one, one, one, null, one, one, null) == 1
    assert lib.pn2_scene_merge_typed(0, 10, 4, 2, 8, 8, 8, one, one, one, one, one, one, null) == 0       # empty range
    assert _lib.launch_count() == before
