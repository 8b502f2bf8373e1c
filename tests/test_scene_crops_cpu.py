"""CPU tests of the training crops: the counter-based draws against values worked out from the definition, the numpy
oracle (crop_oracle.py) against a literal restatement of scannet_dataset.py:30-59, train.py:192-196 and
provider.py:60-69 with np.random replaced by the draws, the label weights of scannet_dataset.py:17-24, SceneSet's
refusals, sample_crops' argument errors and the C entries' refusals (no launch), and the new kernels' resources."""
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

from pointnet2_b200 import _lib, scene, workloads as W  # noqa: E402

M = (1 << 64) - 1


def _mix_int(x):
    x ^= x >> 30
    x = (x * 0xBF58476D1CE4E5B9) & M
    x ^= x >> 27
    x = (x * 0x94D049BB133111EB) & M
    return x ^ (x >> 31)


def test_draw_known_answers():
    # SplitMix64 seeded with 0 yields mix(G), mix(2G), mix(3G): its published first outputs
    g = 0x9E3779B97F4A7C15
    assert [int(CO.mix(np.uint64((k * g) & M))) for k in (1, 2, 3)] == [0xE220A8397B1DCDAF, 0x6E789E6AA1B965F4,
                                                                         0x06C45D188009454F]
    # draw(0, 0, 0, 0) = mix(mix(mix(0))) = 0: the finaliser fixes 0
    assert int(CO.draw(0, 0, 0, 0)) == 0
    # draw(seed, s, b, i) with Python integers, wrap-around by masking
    for seed, s, b, i in [(0, 1, 0, 0), (12345, 2, 7, 99), (-1, 5, 31, 0), (2 ** 63, 4, 65534, 16383), (M, 3, 1, 1)]:
        h = _mix_int(((seed & M) + s * g) & M)
        h = _mix_int((h + b * g) & M)
        h = _mix_int((h + i * g) & M)
        assert int(CO.draw(seed, s, b, i)) == h
        assert CO.unit(h) == (h >> 11) / 2.0 ** 53
    v = CO.draw(7, 4, 3, np.arange(1000))
    assert v.dtype == np.uint64 and len(np.unique(v)) == 1000
    u = CO.unit(v)
    assert (u >= 0).all() and (u < 1).all()


def literal_crop(pts, labels, class_w, seed, b, npoints, max_dropout, rotate):
    """One crop restated expression by expression from scannet_dataset.py:30-59, train.py:192-196 and
    provider.py:60-69, in Python 3 and with the random calls replaced by the draws: the centre index is
    draw(seed, 1, b, attempt) % P, the resampling with replacement becomes the npoints members of smallest key in key
    order, and dropped rows are removed instead of overwritten with row 0.  Every comparison and the voxel key keep
    numpy's float32-against-float64 evaluation of the reference."""
    top, bottom = np.max(pts, axis=0), np.min(pts, axis=0)
    half = [0.75, 0.75, 1.5]
    attempt, accepted = 0, False
    while attempt < 10:
        mid = pts[int(CO.draw(seed, 1, b, attempt)) % len(labels), :]
        box_lo, box_hi = mid - half, mid + half
        box_lo[2], box_hi[2] = bottom[2], top[2]
        sel = np.sum((pts >= (box_lo - 0.2)) * (pts <= (box_hi + 0.2)), axis=1) == 3
        sub, sub_lab = pts[sel, :], labels[sel]
        if len(sub_lab) > 0:
            near = np.sum((sub >= (box_lo - 0.01)) * (sub <= (box_hi + 0.01)), axis=1) == 3
            cell = np.ceil((sub[near, :] - box_lo) / (box_hi - box_lo) * [31.0, 31.0, 62.0])
            cells = np.unique(cell[:, 0] * 31.0 * 62.0 + cell[:, 1] * 62.0 + cell[:, 2])
            accepted = np.sum(sub_lab > 0) / len(sub_lab) >= 0.7 and len(cells) / 31.0 / 31.0 / 62.0 >= 0.02
            if accepted:
                break
        attempt += 1
    attempt = min(attempt, 9)
    members = np.nonzero(sel)[0]
    rank = [int(CO.draw(seed, 2, b, j)) >> 32 for j in members]
    rows = sorted(range(len(members)), key=lambda r: (rank[r], members[r]))[:npoints]
    row_lab, row_core = sub_lab[rows], near[rows]
    w = class_w[row_lab] * row_core
    cut = CO.unit(CO.draw(seed, 3, b, 0)) * max_dropout
    gone = CO.unit(CO.draw(seed, 4, b, np.arange(len(rows)))) <= cut
    w = np.where(gone, np.float32(0), w).astype(np.float32)
    stay = ~gone
    stay[0] = True
    out = sub[rows, :].astype(np.float64)
    if rotate:
        angle = CO.unit(CO.draw(seed, 5, b, 0)) * 2 * np.pi
        cs, sn = np.cos(angle), np.sin(angle)
        out = out.reshape((-1, 3)) @ np.array([[cs, sn, 0], [-sn, cs, 0], [0, 0, 1]])
    return {"attempt": attempt, "valid": bool(accepted), "members": members, "core": near, "nvox": len(cells),
            "rows": members[rows][stay], "xyz": out[stay], "label": row_lab[stay], "weight": w[stay],
            "core_rows": row_core[stay]}


def _boundary_scene():
    """A grid scene whose points sit on the 0.2 / 0.01 boundaries of crops centred on its grid points, and 1 ulp
    either side; every row is a candidate centre, so many attempts land on boundaries."""
    base = np.array([0.0, 0.75, 0.95, 0.76, 1.5, -0.75, -0.95, -0.76, 0.3], np.float32)
    ax = np.concatenate([base, np.nextafter(base, np.float32(-9)), np.nextafter(base, np.float32(9))])
    g = np.stack(np.meshgrid(ax, ax, [0.0, 0.5, 2.0]), -1).reshape(-1, 3).astype(np.float32)
    lab = (np.arange(len(g)) % 7 != 0).astype(np.int64)
    return g, lab


def _alias_scene():
    """Points at the voxel edges of a crop: keys with vy = 32 or vz = 62 collide with neighbouring rows' keys."""
    rs = np.random.RandomState(4)
    c = np.array([2.0, 2.0], np.float32)
    k = rs.randint(0, 33, (4000, 2)).astype(np.float64)
    xy = (c - 0.75 + k / 31.0 * 1.5).astype(np.float32)
    z = (rs.randint(0, 63, 4000) / 62.0 * 2.5).astype(np.float32)
    pts = np.concatenate([np.c_[xy, z], [[2.0, 2.0, 0.0], [2.0, 2.0, 2.5]]]).astype(np.float32)
    return pts, np.ones(len(pts), np.int64)


def _literal_cases():
    rs = np.random.RandomState(2)
    room, lab = W.scene_room(20000, 3)
    yield "room", room, lab, 8192, 0.875, True
    yield "room_small_n", room, lab, 300, 0.0, True
    g, gl = _boundary_scene()
    yield "boundaries", g, gl, 100, 0.875, False
    a, al = _alias_scene()
    yield "alias", a, al, 8192, 0.5, True
    dup = np.repeat((rs.random_sample((300, 3)) * [2.0, 2.0, 1.0]).astype(np.float32), 5, axis=0)
    yield "duplicates", dup, rs.randint(0, 3, len(dup)), 64, 0.875, True
    yield "unlabelled", room, np.zeros_like(lab), 512, 0.875, True


@pytest.mark.parametrize("case", list(_literal_cases()), ids=[c[0] for c in _literal_cases()])
def test_oracle_matches_literal_restatement(case):
    name, pts, lab, npoints, max_dropout, rotate = case
    lw = (1.0 + np.arange(21)).astype(np.float32) / 7
    offsets = np.array([0, len(pts)])
    lo, hi = pts.min(0)[None], pts.max(0)[None]
    seen_invalid = 0
    for seed in (0, 1, -5, 2 ** 63 + 11):
        for b in (0, 3):
            o = CO.oracle_crops(pts, lab, offsets, lo, hi, lw, np.zeros(b + 1, np.int64), seed, npoints, max_dropout,
                                rotate)
            ref = literal_crop(pts, lab, lw, seed, b, npoints, max_dropout, rotate)
            att = CO.crop_attempts(pts, lab, lo[0][2], hi[0][2], seed, b)
            a = int(o["attempt"][b])
            assert a == ref["attempt"] and bool(o["valid"][b]) == ref["valid"], (name, seed, b)
            np.testing.assert_array_equal(att[a]["members"], ref["members"])
            np.testing.assert_array_equal(att[a]["core"], ref["core"])
            assert att[a]["nvox"] == ref["nvox"]
            n = int(o["lengths"][b])
            assert n == len(ref["rows"]) >= 1
            np.testing.assert_array_equal(o["point_idx"][b, :n], ref["rows"])
            np.testing.assert_array_equal(o["label"][b, :n], ref["label"])
            np.testing.assert_array_equal(o["weight"][b, :n], ref["weight"])
            np.testing.assert_array_equal(o["core"][b, :n], ref["core_rows"])
            np.testing.assert_allclose(o["xyz64"][b, :n], ref["xyz"], rtol=0, atol=1e-12)
            assert (o["point_idx"][b, n:] == -1).all() and (o["xyz"][b, n:] == 0).all()
            seen_invalid += not ref["valid"]
    if name == "unlabelled":
        assert seen_invalid == 8  # no attempt can pass: attempt 9 is taken every time
    if name == "alias":
        keys = np.concatenate([t["keys"] for t in CO.crop_attempts(pts, lab, lo[0][2], hi[0][2], 0, 0)])
        assert keys.max() > 31 * 31 * 62  # vx = 32 or beyond: the aliased range is exercised


def test_train_label_weights_match_reference():
    rs = np.random.RandomState(9)
    labels = [rs.randint(0, 21, n) for n in (1000, 5000, 37)] + [W.scene_room(8000, 1)[1]]
    pts = [rs.random_sample((len(l), 3)).astype(np.float32) for l in labels]
    ss = scene.SceneSet(pts, labels, device="cpu")
    # the expression of scannet_dataset.py:17-24 with its dtypes: float64 histogram counts over the 21 unit bins,
    # then float32 frequencies and 1 / log(1.2 + freq) in float32
    counts = sum(np.histogram(l, bins=np.arange(22))[0] for l in labels).astype(np.float64)
    freq = counts.astype(np.float32)
    want = 1 / np.log(1.2 + freq / np.sum(freq))
    w = ss.train_label_weights()
    assert w.dtype == torch.float32 and tuple(w.shape) == (21,)
    assert want.dtype == np.float32
    np.testing.assert_array_equal(w.numpy(), want)


def test_scene_set_packs_and_refuses():
    a = np.array([[0, 0, 0], [1, 2, 3]], np.float32)
    b = np.array([[5, 5, 1], [6, 7, 2], [5.5, 5, 1.5]], np.float32)
    ss = scene.SceneSet([a, torch.from_numpy(b)], [np.array([1, 2]), torch.tensor([0, 3, 4])], device="cpu")
    assert len(ss) == 2 and ss.offsets.tolist() == [0, 2, 5] and ss.label.dtype == torch.int32
    np.testing.assert_array_equal(ss.lo.numpy(), np.stack([a.min(0), b.min(0)]))
    np.testing.assert_array_equal(ss.hi.numpy(), np.stack([a.max(0), b.max(0)]))
    ok = np.ones(2, np.int64)
    with pytest.raises(ValueError, match="at least one scene"):
        scene.SceneSet([], [], device="cpu")
    with pytest.raises(ValueError, match="empty"):
        scene.SceneSet([a, np.zeros((0, 3), np.float32)], [ok, ok[:0]], device="cpu")
    with pytest.raises(ValueError, match="NaN or inf"):
        scene.SceneSet([np.array([[0, 0, 0], [np.nan, 0, 1]], np.float32)], [ok], device="cpu")
    with pytest.raises(ValueError, match="NaN or inf"):
        scene.SceneSet([np.array([[0, 0, 0], [np.inf, 0, 1]], np.float32)], [ok], device="cpu")
    with pytest.raises(ValueError, match="zero z extent"):
        scene.SceneSet([np.array([[0, 0, 1], [3, 2, 1]], np.float32)], [ok], device="cpu")
    with pytest.raises(ValueError, match="outside"):
        scene.SceneSet([a], [np.array([1, 21])], device="cpu")
    with pytest.raises(ValueError, match="outside"):
        scene.SceneSet([a], [np.array([-1, 2])], device="cpu")
    with pytest.raises(ValueError, match="outside"):
        scene.SceneSet([a], [np.array([1, 5])], num_class=5, device="cpu")
    with pytest.raises(ValueError, match="one label array per scene"):
        scene.SceneSet([a, a], [ok], device="cpu")
    with pytest.raises(ValueError, match="labels of shape"):
        scene.SceneSet([a], [np.ones(3, np.int64)], device="cpu")
    with pytest.raises(TypeError, match="labels"):
        scene.SceneSet([a], [np.ones(2, np.float32)], device="cpu")
    with pytest.raises(ValueError, match="num_points, 3"):
        scene.SceneSet([np.zeros((2, 4), np.float32)], [ok], device="cpu")
    with pytest.raises(ValueError, match="num_class"):
        scene.SceneSet([a], [ok], num_class=0, device="cpu")
    with pytest.raises(ValueError, match="1e9"):
        scene.SceneSet([np.array([[0, 0, 0], [2e9, 0, 1]], np.float32)], [ok], device="cpu")


def test_point_count_limit():
    """P >= 2^31 - 1 is refused before any scene is converted (broadcast views: no memory behind them)."""
    x = np.broadcast_to(np.float32(1), (2 ** 30, 3))
    lab = np.broadcast_to(np.int64(1), (2 ** 30,))
    with pytest.raises(ValueError, match="2\\^31 - 1"):
        scene.SceneSet([x, x], [lab, lab], device="cpu")


def test_sample_crops_argument_errors_launch_nothing():
    before = _lib.launch_count()
    a = np.array([[0, 0, 0], [1, 2, 3]], np.float32)
    ss = scene.SceneSet([a], [np.array([1, 2])], device="cpu")
    lw = torch.ones(21)
    cs = torch.zeros(4, dtype=torch.int64)
    with pytest.raises(RuntimeError, match="no CPU path"):
        scene.sample_crops(ss, cs, 0, lw)
    with pytest.raises(TypeError, match="SceneSet"):
        scene.sample_crops(object(), cs, 0, lw)
    with pytest.raises(ValueError, match="npoints"):
        scene.sample_crops(ss, cs, 0, lw, npoints=0)
    with pytest.raises(ValueError, match="16384"):
        scene.sample_crops(ss, cs, 0, lw, npoints=16385)
    with pytest.raises(TypeError, match="npoints"):
        scene.sample_crops(ss, cs, 0, lw, npoints=8192.0)
    with pytest.raises(ValueError, match="max_dropout"):
        scene.sample_crops(ss, cs, 0, lw, max_dropout=1.5)
    with pytest.raises(ValueError, match="max_dropout"):
        scene.sample_crops(ss, cs, 0, lw, max_dropout=float("nan"))
    with pytest.raises(TypeError, match="rotate"):
        scene.sample_crops(ss, cs, 0, lw, rotate=1)
    # the checks that need a CUDA set: a fake one whose tensors are on the CPU but claims a CUDA device
    fake = scene.SceneSet([a], [np.array([1, 2])], device="cpu")
    fake.device = torch.device("cuda", 0)
    with pytest.raises(RuntimeError, match="no CPU path"):
        scene.sample_crops(fake, cs, 0, lw)                                  # crop_scene on the CPU
    with pytest.raises(TypeError, match="integer"):
        scene.sample_crops(fake, cs.float(), 0, lw)
    with pytest.raises(ValueError, match="crop_scene"):
        scene.sample_crops(fake, torch.zeros(2, 2, dtype=torch.int64), 0, lw)
    with pytest.raises(ValueError, match="crop_scene"):
        scene.sample_crops(fake, torch.zeros(0, dtype=torch.int64), 0, lw)
    with pytest.raises(TypeError, match="crop_scene"):
        scene.sample_crops(fake, [0, 1], 0, lw)
    assert _lib.launch_count() == before


def test_abi_refusals():
    lib = _lib.load()
    before = _lib.launch_count()
    null = ctypes.c_void_p(0)
    one = ctypes.c_void_p(256)  # never dereferenced: every call below is refused first
    assert lib.pn2_scene_crops_workspace_bytes(0, 8192) == 0
    assert lib.pn2_scene_crops_workspace_bytes(4, 0) == 0
    assert lib.pn2_scene_crops_workspace_bytes(4, 16385) == 0
    assert lib.pn2_scene_crops_workspace_bytes(65536, 16) == 0
    ws = lib.pn2_scene_crops_workspace_bytes(4, 8192)
    assert ws >= 4 * 10 * (2 + 1986) * 4 and ws % 256 == 0
    assert lib.pn2_scene_crops_workspace_bytes(4, 16384) == ws  # sized by the batch, not the rows or the scenes

    def call(s=2, p=1000, max_scene=600, num_class=21, b=4, npoints=8192, max_dropout=0.875, ptrs=None, wsb=ws, wsp=one):
        q = ptrs or {}
        g = lambda k: q.get(k, one)  # noqa: E731
        return lib.pn2_scene_crops(s, p, max_scene, g("xyz"), g("label"), g("off"), g("lo"), g("hi"), num_class, g("lw"), b,
                                   g("cs"), 5, null, npoints, max_dropout, 1, g("ox"), g("ol"), g("ow"), g("len"), g("pi"),
                                   g("core"), g("att"), g("valid"), wsp, wsb, null)
    assert call(s=0) == 1
    assert call(p=0) == 1
    assert call(p=2 ** 31 - 1) == 1
    assert call(max_scene=1001) == 1
    assert call(max_scene=0) == 1
    assert call(num_class=0) == 1
    assert call(b=0) == 1
    assert call(b=65536, npoints=1) == 1
    assert call(npoints=0) == 1
    assert call(npoints=16385) == 1
    assert call(b=50000, npoints=16384) == 1        # b * npoints * 3 >= 2^31
    assert call(max_dropout=-0.1) == 1
    assert call(max_dropout=1.01) == 1
    assert call(max_dropout=float("nan")) == 1
    for k in ("xyz", "label", "off", "lo", "hi", "lw", "cs", "ox", "ol", "ow", "len", "pi", "core", "att", "valid"):
        assert call(ptrs={k: null}) == 1, k
    assert call(wsb=ws - 1) == 1
    assert call(wsp=ctypes.c_void_p(264)) == 1      # workspace not 256-byte aligned
    assert call(wsp=null) == 1
    assert _lib.launch_count() == before


def test_crop_kernels_do_not_spill():
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(cuobjdump):
        pytest.skip("cuobjdump not available")
    out = subprocess.run([cuobjdump, "-res-usage", _lib.lib_path()], capture_output=True, text=True).stdout
    found = re.findall(r"Function (\S*crop_\w+_kernel\S*):\s*\n\s*REG:(\d+) STACK:(\d+)", out)
    assert len(found) == 2, found  # the attempt and select passes
    assert all(stack == "0" for _, _, stack in found), found
    assert not re.findall(r"scene_crop|scene_\w*crop", out)  # crop kernels stay outside the scene_*_kernel names
