"""GPU tests of the virtual scans (scene.sample_virtual_scans): every output field against the numpy oracle
(scan_oracle.py) bit for bit, after checking that every decision of the oracle has a margin above 1e-12; subsets when
npoints < visible; an adversarial scene (points along rays at several depths, exact duplicates, the +-pi seam of view 4,
a point at a camera); scenes that see nothing or too little; determinism and a device seed replayed through a CUDA
graph; an out-of-range scene; and a ragged training step fed by the scans."""
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import scan_oracle as SO  # noqa: E402

from pointnet2_b200 import _lib, nets, scene, workloads as W  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
FIELDS = ("xyz", "label", "weight", "lengths", "point_idx", "visible", "valid")
Q = 2.0 ** -14  # grid of the adversarial scene's coordinates: every float64 sum over it is exact


def _set(scenes, num_class=21):
    return scene.SceneSet([p for p, _ in scenes], [l for _, l in scenes], num_class=num_class, device=DEV)


def _run(ss, scan_scene, scan_mode, seed, lw=None, **kw):
    lw = ss.train_label_weights() if lw is None else lw
    cs = torch.as_tensor(np.asarray(scan_scene, np.int64), device=DEV)
    cm = torch.as_tensor(np.asarray(scan_mode, np.int64), device=DEV)
    want = SO.oracle_scans(ss.xyz.cpu().numpy(), ss.label.cpu().numpy(), ss.offsets.cpu().numpy(), ss.mean.cpu().numpy(),
                           lw.cpu().numpy(), scan_scene, scan_mode, seed, **kw)
    assert (want["margin"] > 1e-12).all(), want["margin"]  # the precondition of an exact comparison
    return scene.sample_virtual_scans(ss, cs, cm, seed, lw, **kw), want


def _check(got, want):
    for f in FIELDS:
        g = getattr(got, f).cpu().numpy()
        assert g.dtype == want[f].dtype, f
        np.testing.assert_array_equal(g, want[f], err_msg=f)
    # weight 0 on every row of an invalid entry
    assert (got.weight[~got.valid] == 0).all()


def _rooms(sizes, seed0=0):
    return [W.scene_room(int(n), seed0 + k) for k, n in enumerate(sizes)]


def test_full_scans_match_oracle():
    """Rooms small enough that every scan fits in npoints: the rows are the whole visible set in (key, index) order."""
    ss = _set(_rooms((40000, 25000)) + [W.scene_room(2600, 1)])
    modes = list(range(8)) + [8, -2, -1, -1, -1, -1]
    cs = [k % 3 for k in range(len(modes))] + [2] * 8
    cm = modes + list(range(8))
    for seed in (3, -11, 2 ** 64 - 5):
        got, want = _run(ss, cs, cm, seed, npoints=16384)
        _check(got, want)
        assert (want["visible"] < 16384).all() and (want["lengths"] == want["visible"]).all()
    assert not want["valid"].all() and want["valid"].any()  # the 2600-point room has views below 300 points


def test_subsets_are_the_smallest_keys():
    ss = _set(_rooms((150000, 60000), seed0=3))
    cs, cm = [0] * 8 + [1, 1, 0, 0], list(range(8)) + [-1, 3, -1, 5]
    for npoints in (1000, 4096, 7000):
        got, want = _run(ss, cs, cm, 21, npoints=npoints, min_points=300)
        _check(got, want)
        assert (want["visible"] > npoints).all() and (want["lengths"] == npoints).all()


def _adversarial():
    """A quantised room plus points placed from the cameras of views 0, 2 and 4, and one last point that makes the
    scene's float64 mean exactly mu, so that every camera is exactly where the points assume.  The room lies on a grid
    of 2Q and mu on the odd multiples of Q, so no room point lies in a camera's plane of symmetry, where the two middle
    rays tie."""
    room, lab = W.scene_room(20000, 7)
    room = np.round(room.astype(np.float64) / (2 * Q)) * (2 * Q)
    mu = np.round(room.mean(axis=0) / (2 * Q)) * (2 * Q) + Q
    c0 = np.array([mu[0] - 1, mu[1], 1.5])
    xx, yy = np.linspace(-0.6, 0.6, 200), np.linspace(-0.45, 0.45, 150)
    extra, kinds = [], []
    for i, j in [(10, 20), (100, 75), (150, 140), (199, 0), (0, 149)]:
        for t in (0.3, 0.6, 0.9):  # one ray of view 0 (direction (1, -xx_i, yy_j)) at three depths
            extra.append(c0 + t * np.array([1.0, -xx[i], yy[j]]))
            kinds.append(("ray", (i, j), t))
    dup = c0 + 0.2 * np.array([1.0, -xx[50], yy[50]])
    extra += [dup, dup]
    kinds += [("dup", 0, 0), ("dup", 1, 0)]
    extra.append(np.array([mu[0], mu[1] - 1, 1.5]))  # at the camera of view 2
    kinds.append(("camera", 2, 0))
    c4 = np.array([mu[0] + 1, mu[1], 1.5])
    for dy, dz in [(0.012, 0.03), (-0.012, 0.03), (0.0, 0.06), (0.009, -0.09), (-0.009, -0.09)]:
        extra.append(c4 + np.array([-3.0, dy, dz]))  # both sides of the +-pi seam of view 4, behind the view-0 camera
        kinds.append(("seam", dy, dz))
    extra = np.round(np.array(extra) / Q) * Q
    pts = np.concatenate([room, extra])
    last = (len(pts) + 1) * mu - pts.sum(axis=0)
    pts = np.concatenate([pts, last[None]]).astype(np.float32)
    assert (pts.astype(np.float64) == np.concatenate([room, extra, last[None]])).all()
    assert (np.mean(pts.astype(np.float64), axis=0) == mu).all()
    labels = np.concatenate([lab, np.full(len(extra) + 1, 5)])
    return pts, labels, len(room), kinds


def test_adversarial_scene():
    pts, labels, n_room, kinds = _adversarial()
    # a scene behind and beside the view-0 camera (nothing near), and one with 100 <= visible < 300
    rs = np.random.RandomState(4)
    blobs = [np.array(c) + rs.uniform(-0.2, 0.2, (400, 3)) for c in ((-3, 0, 1.5), (1.5, 6, 1.5), (1.5, -6, 1.5))]
    away = np.concatenate(blobs).astype(np.float32)
    small, small_lab = W.scene_room(2600, 1)
    ss = _set([(pts, labels), (away, np.ones(len(away), np.int64)), (small, small_lab)])
    # the views whose cameras the points were placed from, and a random one (the diagonal views, and view 6 with the
    # view-2 camera straight ahead, hold points in exact ties between rays)
    cs = [0, 0, 0, 0, 1, 1, 2]
    cm = [0, 2, 4, -1, 0, -1, 0]
    got, want = _run(ss, cs, cm, 5, npoints=16384)
    _check(got, want)
    vis0 = set(want["smpidx"][0].tolist())
    ray_pts = [k for k, kd in enumerate(kinds) if kd[0] == "ray"]
    for k in ray_pts:  # the nearest of the three depths is what view 0 sees of each ray
        assert ((n_room + k) in vis0) == (kinds[k][2] == 0.3), kinds[k]
    assert {n_room + k for k, kd in enumerate(kinds) if kd[0] == "dup"} <= vis0  # both duplicates
    seam = {n_room + k for k, kd in enumerate(kinds) if kd[0] == "seam"}
    assert seam <= set(want["smpidx"][2].tolist())
    assert (n_room + kinds.index(("camera", 2, 0))) not in set(want["smpidx"][1].tolist())  # r = 0, az = el = 0
    assert want["visible"][4] == 0 and want["near"][4] < 100 and got.lengths[4].item() == 0
    assert 100 <= want["visible"][6] < 300 and not want["valid"][6] and got.lengths[6].item() == want["visible"][6]
    assert (got.weight[6] == 0).all()


def test_same_seed_same_bits_and_device_seed():
    ss = _set(_rooms((100000, 50000)))
    cs = torch.tensor([0, 1, 0, 1, 1, 0, 0, 1], device=DEV)
    cm = torch.tensor([-1, -1, 0, 4, -1, 7, -1, -1], device=DEV)
    lw = ss.train_label_weights()
    a = scene.sample_virtual_scans(ss, cs, cm, 123, lw)
    b = scene.sample_virtual_scans(ss, cs, cm, 123, lw)
    c = scene.sample_virtual_scans(ss, cs, cm, 124, lw)
    for f in a._fields:
        assert torch.equal(getattr(a, f), getattr(b, f)), f
    assert not torch.equal(a.point_idx, c.point_idx)
    d = scene.sample_virtual_scans(ss, cs, cm, torch.tensor([123], device=DEV), lw)
    for f in a._fields:
        assert torch.equal(getattr(a, f), getattr(d, f)), f
    e = scene.sample_virtual_scans(ss, cs.to(torch.int32), cm.to(torch.int16), 123, lw)
    assert torch.equal(a.point_idx, e.point_idx)


def test_device_seed_in_cuda_graph():
    ss = _set(_rooms((60000, 30000)))
    cs = torch.tensor([0, 1, 1, 0], device=DEV)
    cm = torch.tensor([-1, -1, 2, -1], device=DEV)
    lw = ss.train_label_weights()
    seed = torch.tensor([1], device=DEV)
    scene.sample_virtual_scans(ss, cs, cm, seed, lw)  # loads the library and sets the kernels' attributes
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        with torch.cuda.graph(g, stream=s):
            out = scene.sample_virtual_scans(ss, cs, cm, seed, lw)
    torch.cuda.current_stream().wait_stream(s)
    for v in (99, -4, 2 ** 40):
        seed.fill_(v)
        g.replay()
        want = scene.sample_virtual_scans(ss, cs, cm, v, lw)
        torch.cuda.synchronize()
        for f in want._fields:
            assert torch.equal(getattr(out, f), getattr(want, f)), (v, f)


def test_out_of_range_scene_gives_empty_entry():
    ss = _set(_rooms((20000,)))
    got = scene.sample_virtual_scans(ss, torch.tensor([0, 5, -1], device=DEV), torch.tensor([0, 0, -1], device=DEV), 1,
                                     ss.train_label_weights(), npoints=512)
    assert got.lengths.tolist()[1:] == [0, 0] and got.visible.tolist()[1:] == [-1, -1]
    assert not got.valid[1:].any() and (got.point_idx[1:] == -1).all() and (got.xyz[1:] == 0).all()
    assert (got.label[1:] == 0).all() and (got.weight[1:] == 0).all()
    assert got.lengths[0].item() >= 1


def test_launches_and_no_host_sync():
    ss = _set(_rooms((20000,)))
    cs = torch.zeros(3, dtype=torch.int64, device=DEV)
    cm = torch.tensor([0, -1, 3], device=DEV)
    lw = ss.train_label_weights()
    scene.sample_virtual_scans(ss, cs, cm, 0, lw)
    seed = torch.tensor([4], device=DEV)
    torch.cuda.synchronize()
    before = _lib.launch_count()
    torch.cuda.set_sync_debug_mode("error")
    try:
        scene.sample_virtual_scans(ss, cs, cm, seed, lw)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    assert _lib.launch_count() == before + 5


def test_training_step_on_scans():
    torch.manual_seed(0)
    ss = _set(_rooms((80000, 40000, 2600), seed0=5))
    net = nets.PointNet2SemSeg(21).to(DEV).train()
    scans = scene.sample_virtual_scans(ss, torch.tensor([0, 1, 2, 0], device=DEV), torch.tensor([0, 3, 1, -1], device=DEV),
                                       3, ss.train_label_weights(), npoints=4096)
    assert scans.lengths.min().item() < 4096  # a ragged batch
    pred, _ = net(scans.xyz, scans.lengths)
    loss = nets.sem_seg_loss(pred, scans.label, scans.weight, lengths=scans.lengths)
    assert torch.isfinite(loss)
    loss.backward()
    assert all(p.grad is None or torch.isfinite(p.grad).all() for p in net.parameters())
    assert any(p.grad is not None and p.grad.abs().sum() > 0 for p in net.parameters())
