"""CPU tests of the virtual scans: the numpy oracle (scan_oracle.py) against a literal Python 3 restatement of
scannet/scene_util.py virtual_scan on float64 input (the same visible set) and on float32 input (the reference's own
dtypes: at most 1 % of the visible set differs), ScannetDatasetVirtualScan.__getitem__ restated (it keeps exactly the
scans the oracle marks valid), SceneSet.mean, sample_virtual_scans' argument errors and the C entries' refusals (no
launch), and the new kernels' resources."""
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
import scan_oracle as SO  # noqa: E402

from pointnet2_b200 import _lib, scene, workloads as W  # noqa: E402


def literal_virtual_scan(xyz, mode=-1, random=None):
    """scene_util.py:11-63 expression by expression in Python 3 (range for xrange), np.random.random replaced by
    ``random``.  The nearest ray comes from scikit-learn's kd-tree, as in the reference."""
    neighbors = pytest.importorskip("sklearn.neighbors")

    def cart2sph(xyz):
        xy = xyz[:, 0] ** 2 + xyz[:, 1] ** 2
        aer = np.zeros(xyz.shape)
        aer[:, 2] = np.sqrt(xy + xyz[:, 2] ** 2)
        aer[:, 1] = np.arctan2(xyz[:, 2], np.sqrt(xy))
        aer[:, 0] = np.arctan2(xyz[:, 1], xyz[:, 0])
        return aer

    camloc = np.mean(xyz, axis=0)
    camloc[2] = 1.5
    if mode == -1:
        view_dr = np.array([2 * np.pi * random(), np.pi / 10 * (random() - 0.75)])
        camloc[:2] -= (0.8 + 0.7 * random()) * np.array([np.cos(view_dr[0]), np.sin(view_dr[0])])
    else:
        view_dr = np.array([np.pi / 4 * mode, 0])
        camloc[:2] -= np.array([np.cos(view_dr[0]), np.sin(view_dr[0])])
    ct_ray_dr = np.array([np.cos(view_dr[1]) * np.cos(view_dr[0]), np.cos(view_dr[1]) * np.sin(view_dr[0]),
                          np.sin(view_dr[1])])
    hr_dr = np.cross(ct_ray_dr, np.array([0, 0, 1]))
    hr_dr /= np.linalg.norm(hr_dr)
    vt_dr = np.cross(hr_dr, ct_ray_dr)
    vt_dr /= np.linalg.norm(vt_dr)
    xx = np.linspace(-0.6, 0.6, 200)
    yy = np.linspace(-0.45, 0.45, 150)
    xx, yy = np.meshgrid(xx, yy)
    xx = xx.reshape(-1, 1)
    yy = yy.reshape(-1, 1)
    rays = xx * hr_dr.reshape(1, -1) + yy * vt_dr.reshape(1, -1) + ct_ray_dr.reshape(1, -1)
    rays_aer = cart2sph(rays)
    local_xyz = xyz - camloc.reshape(1, -1)
    local_aer = cart2sph(local_xyz)
    nbrs = neighbors.NearestNeighbors(n_neighbors=1, algorithm="kd_tree").fit(rays_aer[:, :2])
    mindd, minidx = nbrs.kneighbors(local_aer[:, :2])
    mindd = mindd.reshape(-1)
    minidx = minidx.reshape(-1)
    sub_idx = mindd < 0.01
    if sum(sub_idx) < 100:
        return np.ones(0)
    sub_r = local_aer[sub_idx, 2]
    sub_minidx = minidx[sub_idx]
    min_r = float("inf") * np.ones(np.max(sub_minidx) + 1)
    for i in range(len(sub_r)):
        if sub_r[i] < min_r[sub_minidx[i]]:
            min_r[sub_minidx[i]] = sub_r[i]
    sub_smpidx = np.ones(len(sub_r))
    for i in range(len(sub_r)):
        if sub_r[i] > min_r[sub_minidx[i]]:
            sub_smpidx[i] = 0
    smpidx = np.where(sub_idx)[0]
    smpidx = smpidx[sub_smpidx == 1]
    return smpidx


def literal_getitem(point_set_ini, semantic_seg_ini, labelweights, npoints, virtual_scan, choice):
    """scannet_dataset.py:141-165 in Python 3, with virtual_scan and np.random.choice injected.  Also returns the
    views it kept."""
    sample_weight_ini = labelweights[semantic_seg_ini]
    point_sets, semantic_segs, sample_weights, kept = [], [], [], []
    for i in range(8):
        smpidx = virtual_scan(point_set_ini, mode=i)
        if len(smpidx) < 300:
            continue
        point_set = point_set_ini[smpidx, :]
        semantic_seg = semantic_seg_ini[smpidx]
        sample_weight = sample_weight_ini[smpidx]
        c = choice(len(semantic_seg), npoints)
        point_sets.append(np.expand_dims(point_set[c, :], 0))
        semantic_segs.append(np.expand_dims(semantic_seg[c], 0))
        sample_weights.append(np.expand_dims(sample_weight[c], 0))
        kept.append(i)
    return (np.concatenate(point_sets, axis=0), np.concatenate(semantic_segs, axis=0),
            np.concatenate(sample_weights, axis=0), kept)


class _Draws:
    """np.random.random() replaced by the u1, u2, u3 of a random view, in the reference's call order."""

    def __init__(self, u):
        self.u = list(u)

    def __call__(self):
        return self.u.pop(0)


def _room(p, seed):
    x, lab = W.scene_room(p, seed)
    return x, lab, np.mean(x.astype(np.float64), axis=0)


@pytest.mark.parametrize("p,seed", [(150000, 0), (20000, 3)])
def test_oracle_matches_reference_on_float64_input(p, seed):
    x, _, mean = _room(p, seed)
    x64 = x.astype(np.float64)
    for b, mode in enumerate(list(range(8)) + [-1, -1, -1]):
        draws = SO.view_draws(seed, b) if mode == -1 else None
        want = SO.scan(x, mean, mode, draws)
        assert want["margin"] > 1e-12, (mode, want["margin"])
        got = literal_virtual_scan(x64, mode, _Draws(draws) if draws else None)
        np.testing.assert_array_equal(np.asarray(got, np.int64), want["smpidx"], err_msg=str(mode))
        assert len(want["smpidx"]) > 0


def test_oracle_against_reference_on_float32_input():
    """The reference's own dtypes (float32 camera and local coordinates) change at most 1 % of a scan."""
    x, _, mean = _room(150000, 0)
    for mode in range(8):
        want = SO.scan(x, mean, mode)["smpidx"]
        got = np.asarray(literal_virtual_scan(x, mode), np.int64)
        diff = len(np.setxor1d(got, want))
        assert diff <= 0.01 * len(want), (mode, diff, len(want))


def test_dataset_keeps_the_valid_scans():
    """A small room: some of its eight views see fewer than 300 points.  The restated __getitem__ keeps exactly the
    views the oracle marks valid, and every row it returns is a point of that view's visible set."""
    x, lab, mean = _room(2600, 1)
    x64 = x.astype(np.float64)
    lw = np.ones(21)
    rs = np.random.RandomState(0)
    pts, segs, wts, kept = literal_getitem(x64, lab.astype(np.int32), lw, 512, literal_virtual_scan,
                                           lambda n, k: rs.choice(n, k, replace=True))
    got = SO.oracle_scans(x, lab, np.array([0, len(x)]), mean[None], lw.astype(np.float32), np.zeros(8, np.int64),
                          np.arange(8), 0, npoints=512)
    assert (got["margin"] > 1e-12).all()
    valid = np.nonzero(got["valid"])[0].tolist()
    assert kept == valid and 0 < len(valid) < 8, (kept, got["visible"])
    for k, view in enumerate(kept):
        vis = x64[got["smpidx"][view]]
        assert (pts[k][:, None, :] == vis[None]).all(-1).any(-1).all()
        assert (wts[k] == 1).all() and segs[k].shape == (512,)


def test_oracle_edge_cases():
    rs = np.random.RandomState(2)
    x, _, mean = _room(20000, 4)
    # behind the camera only: nothing is near
    cam, rays = SO.view(mean, 0)
    behind = (cam + np.array([-1.0, 0.0, 0.0]) + rs.uniform(-0.3, 0.3, (500, 3))).astype(np.float32)
    assert len(SO.scan(behind, mean, 0)["smpidx"]) == 0
    # exact duplicates are both visible
    d = np.concatenate([x, x[:50]])
    got = SO.scan(d, mean, 0)["smpidx"]
    dup = np.intersect1d(got, np.arange(50))
    assert len(dup) and np.isin(dup + len(x), got).all()


def test_scene_set_mean():
    a = (np.random.RandomState(0).random_sample((1001, 3)) * 7).astype(np.float32)
    b = np.array([[1, 2, 3], [2, 3, 5]], np.float32)
    ss = scene.SceneSet([a, b], [np.zeros(1001, np.int64), np.zeros(2, np.int64)], device="cpu")
    assert ss.mean.dtype == torch.float64 and tuple(ss.mean.shape) == (2, 3)
    np.testing.assert_array_equal(ss.mean.numpy()[0], np.mean(a.astype(np.float64), axis=0))
    np.testing.assert_array_equal(ss.mean.numpy()[1], [1.5, 2.5, 4.0])


def test_sample_virtual_scans_argument_errors_launch_nothing():
    before = _lib.launch_count()
    a = np.array([[0, 0, 0], [1, 2, 3]], np.float32)
    ss = scene.SceneSet([a], [np.array([1, 2])], device="cpu")
    lw = torch.ones(21)
    cs = torch.zeros(4, dtype=torch.int64)
    cm = torch.arange(4)
    f = scene.sample_virtual_scans
    with pytest.raises(RuntimeError, match="no CPU path"):
        f(ss, cs, cm, 0, lw)
    with pytest.raises(TypeError, match="SceneSet"):
        f(object(), cs, cm, 0, lw)
    with pytest.raises(ValueError, match="npoints"):
        f(ss, cs, cm, 0, lw, npoints=0)
    with pytest.raises(ValueError, match="16384"):
        f(ss, cs, cm, 0, lw, npoints=16385)
    with pytest.raises(TypeError, match="npoints"):
        f(ss, cs, cm, 0, lw, npoints=8192.0)
    with pytest.raises(ValueError, match="min_points"):
        f(ss, cs, cm, 0, lw, min_points=-1)
    with pytest.raises(TypeError, match="min_points"):
        f(ss, cs, cm, 0, lw, min_points=True)
    # the checks that need a CUDA set: a fake one whose tensors are on the CPU but claims a CUDA device
    fake = scene.SceneSet([a], [np.array([1, 2])], device="cpu")
    fake.device = torch.device("cuda", 0)
    with pytest.raises(RuntimeError, match="no CPU path"):
        f(fake, cs, cm, 0, lw)                                      # scan_scene on the CPU
    with pytest.raises(TypeError, match="scan_scene"):
        f(fake, cs.float(), cm, 0, lw)
    with pytest.raises(TypeError, match="scan_mode"):
        f(fake, cs, cm.bool(), 0, lw)
    with pytest.raises(ValueError, match="scan_scene"):
        f(fake, torch.zeros(2, 2, dtype=torch.int64), cm, 0, lw)
    with pytest.raises(ValueError, match="scan_scene"):
        f(fake, torch.zeros(0, dtype=torch.int64), cm, 0, lw)
    with pytest.raises(ValueError, match="4096"):
        f(fake, torch.zeros(4097, dtype=torch.int64), cm, 0, lw)
    with pytest.raises(TypeError, match="scan_scene"):
        f(fake, [0, 1], cm, 0, lw)
    with pytest.raises(TypeError, match="scan_mode"):
        f(fake, cs, [0, 1], 0, lw)
    with pytest.raises(ValueError, match="one scan_mode per scan_scene"):
        f(fake, cs, cm[:3], 0, lw)
    assert _lib.launch_count() == before


def test_abi_refusals():
    lib = _lib.load()
    before = _lib.launch_count()
    null = ctypes.c_void_p(0)
    one = ctypes.c_void_p(256)  # never dereferenced: every call below is refused first
    assert lib.pn2_virtual_scans_workspace_bytes(0, 1000, 8192) == 0
    assert lib.pn2_virtual_scans_workspace_bytes(4097, 1000, 16) == 0
    assert lib.pn2_virtual_scans_workspace_bytes(4, 0, 8192) == 0
    assert lib.pn2_virtual_scans_workspace_bytes(4, 1000, 0) == 0
    assert lib.pn2_virtual_scans_workspace_bytes(4, 1000, 16385) == 0
    ws = lib.pn2_virtual_scans_workspace_bytes(4, 1000, 8192)
    assert ws > 4 * 30000 * (4 * 8 + 4 + 8) and ws % 256 == 0
    assert lib.pn2_virtual_scans_workspace_bytes(4, 1000, 16) == ws             # not sized by the rows
    assert lib.pn2_virtual_scans_workspace_bytes(4, 1000 + 32 * 64, 16) == ws + 4 * 4 * 64  # one bit per point

    def call(s=2, p=2000, max_scene=1000, num_class=21, b=4, npoints=8192, min_points=300, ptrs=None, wsb=ws, wsp=one):
        q = ptrs or {}
        g = lambda k: q.get(k, one)  # noqa: E731
        return lib.pn2_virtual_scans(s, p, max_scene, g("xyz"), g("label"), g("off"), g("mean"), num_class, g("lw"), b,
                                     g("cs"), g("cm"), 5, null, npoints, min_points, g("ox"), g("ol"), g("ow"), g("len"),
                                     g("pi"), g("vis"), g("valid"), wsp, wsb, null)
    assert call(s=0) == 1
    assert call(p=0) == 1
    assert call(p=2 ** 31 - 1) == 1
    assert call(p=999) == 1                          # max_scene > p
    assert call(max_scene=0) == 1
    assert call(num_class=0) == 1
    assert call(b=0) == 1
    assert call(b=4097, npoints=1) == 1
    assert call(npoints=0) == 1
    assert call(npoints=16385) == 1
    assert call(min_points=-1) == 1
    for k in ("xyz", "label", "off", "mean", "lw", "cs", "cm", "ox", "ol", "ow", "len", "pi", "vis", "valid"):
        assert call(ptrs={k: null}) == 1, k
    assert call(wsb=ws - 1) == 1
    assert call(wsp=ctypes.c_void_p(264)) == 1      # workspace not 256-byte aligned
    assert call(wsp=null) == 1
    assert _lib.launch_count() == before


def test_scan_kernels_do_not_spill():
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(cuobjdump):
        pytest.skip("cuobjdump not available")
    out = subprocess.run([cuobjdump, "-res-usage", _lib.lib_path()], capture_output=True, text=True).stdout
    found = re.findall(r"Function (\S*vscan_\w+_kernel\S*):\s*\n\s*REG:(\d+) STACK:(\d+)", out)
    assert len(found) == 4, found  # ray, cell, point and select
    assert all(stack == "0" for _, _, stack in found), found
