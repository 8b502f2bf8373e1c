"""GPU tests of the training crops (scene.sample_crops): every output field against the numpy oracle
(crop_oracle.py) bit for bit, the rotated coordinates within one float32 ulp of its float64 evaluation; determinism and
seed dependence; a device seed replayed through a CUDA graph; the uniformity of the rows; and a ragged training step
fed by the crops."""
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import crop_oracle as CO  # noqa: E402

from pointnet2_b200 import _lib, nets, scene, workloads as W  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
FIELDS = ("label", "weight", "lengths", "point_idx", "core", "attempt", "valid")


def _set(scenes, num_class=21):
    return scene.SceneSet([p for p, _ in scenes], [l for _, l in scenes], num_class=num_class, device=DEV)


def _run(ss, crop_scene, seed, lw=None, **kw):
    lw = ss.train_label_weights() if lw is None else lw
    cs = torch.as_tensor(np.asarray(crop_scene, np.int64), device=DEV)
    got = scene.sample_crops(ss, cs, seed, lw, **kw)
    want = CO.oracle_crops(ss.xyz.cpu().numpy(), ss.label.cpu().numpy(), ss.offsets.cpu().numpy(), ss.lo.cpu().numpy(),
                           ss.hi.cpu().numpy(), lw.cpu().numpy(), crop_scene, seed, **kw)
    return got, want


def _check(got, want, rotate=True):
    for f in FIELDS:
        g = getattr(got, f).cpu().numpy()
        assert g.dtype == want[f].dtype or f in ("core", "valid"), f
        np.testing.assert_array_equal(g, want[f], err_msg=f)
    xyz = got.xyz.cpu().numpy()
    if rotate:
        # one float32 ulp, plus an absolute 1e-12 for the ~1e-16 difference between the kernel's sincospi(2u) and
        # numpy's cos / sin of the rounded angle, which can matter where x cos - y sin cancels to almost 0
        ulp = np.spacing(np.abs(want["xyz64"]).astype(np.float32)).astype(np.float64)
        assert (np.abs(xyz.astype(np.float64) - want["xyz64"]) <= ulp + 1e-12).all()
        assert (xyz.view(np.int32) != want["xyz"].view(np.int32)).mean() < 1e-3  # nearly always the same rounding
    else:
        np.testing.assert_array_equal(xyz, want["xyz"])


def _rooms(sizes, seed0=0):
    return [W.scene_room(int(n), seed0 + k) for k, n in enumerate(sizes)]


@pytest.mark.parametrize("sizes,b", [((150000,), 8), ((30000, 150000, 4000), 12), (tuple(np.linspace(3000, 60000, 20)), 24),
                                     ((1000000, 20000), 6)], ids=["one", "three", "twenty", "million"])
def test_crops_match_oracle(sizes, b):
    ss = _set(_rooms(sizes))
    rs = np.random.RandomState(len(sizes))
    cs = rs.randint(0, len(sizes), b)
    for seed, kw in [(11, {}), (-3, dict(max_dropout=0.0, rotate=False)), (2 ** 64 - 7, dict(npoints=2048))]:
        got, want = _run(ss, cs, seed, **kw)
        _check(got, want, kw.get("rotate", True))
        assert (want["lengths"] >= 1).all()


def test_crop_sizes_around_npoints():
    """c < npoints, c = npoints and c >> npoints, npoints 1 and the cap."""
    ss = _set(_rooms((200000,)))
    cs = np.zeros(4, np.int64)
    probe = CO.oracle_crops(ss.xyz.cpu().numpy(), ss.label.cpu().numpy(), ss.offsets.cpu().numpy(), ss.lo.cpu().numpy(),
                            ss.hi.cpu().numpy(), np.ones(21, np.float32), cs, 5, npoints=16384, max_dropout=0.0)
    c = int(probe["context"][0])
    assert c > 1000
    for n in (c, c - 1, c + 1, 1, 16384, 64):
        if n > 16384:
            continue
        got, want = _run(ss, cs, 5, npoints=n, max_dropout=0.0)
        _check(got, want)
        if n == c:
            assert want["lengths"][0] == c
    got, want = _run(ss, cs, 5, npoints=16384, max_dropout=0.875)
    _check(got, want)
    assert (want["context"] > 16384).any() or (want["context"] < 16384).any()


def test_unlabelled_and_duplicate_scenes():
    rs = np.random.RandomState(1)
    room, lab = W.scene_room(40000, 3)
    dup = np.repeat((rs.random_sample((2000, 3)) * [2.5, 2.5, 1.0]).astype(np.float32), 20, axis=0)
    ss = _set([(room, np.zeros_like(lab)), (dup, rs.randint(0, 21, len(dup)))])
    got, want = _run(ss, [0, 0, 1, 1, 0, 1], 77, npoints=4096)
    _check(got, want)
    assert (want["attempt"][[0, 1, 4]] == 9).all() and not want["valid"][[0, 1, 4]].any()
    assert (want["label"][[0, 1, 4]] == 0).all()
    # equal points get different keys: duplicates land in different rows
    pi = want["point_idx"][2, :want["lengths"][2]]
    assert len(np.unique(dup[pi - len(room)], axis=0)) < len(pi)


def test_same_seed_same_bits_other_seed_other_crops():
    ss = _set(_rooms((100000, 50000)))
    cs = torch.tensor([0, 1, 0, 1, 1, 0, 0, 1], device=DEV)
    lw = ss.train_label_weights()
    a = scene.sample_crops(ss, cs, 123, lw)
    b = scene.sample_crops(ss, cs, 123, lw)
    c = scene.sample_crops(ss, cs, 124, lw)
    for f in a._fields:
        assert torch.equal(getattr(a, f), getattr(b, f)), f
    assert not torch.equal(a.point_idx, c.point_idx)
    # a (1,) device seed gives the bits of the same int seed
    d = scene.sample_crops(ss, cs, torch.tensor([123], device=DEV), lw)
    for f in a._fields:
        assert torch.equal(getattr(a, f), getattr(d, f)), f
    # an int32 crop_scene is the same request
    e = scene.sample_crops(ss, cs.to(torch.int32), 123, lw)
    assert torch.equal(a.point_idx, e.point_idx)


def test_out_of_range_scene_gives_empty_crop():
    ss = _set(_rooms((20000,)))
    got = scene.sample_crops(ss, torch.tensor([0, 5, -1], device=DEV), 1, ss.train_label_weights(), npoints=512)
    assert got.lengths.tolist()[1:] == [0, 0] and got.attempt.tolist()[1:] == [-1, -1]
    assert (got.point_idx[1:] == -1).all() and (got.xyz[1:] == 0).all() and got.lengths[0].item() >= 1


def test_device_seed_in_cuda_graph():
    ss = _set(_rooms((60000, 30000)))
    cs = torch.tensor([0, 1, 1, 0], device=DEV)
    lw = ss.train_label_weights()
    seed = torch.tensor([1], device=DEV)
    scene.sample_crops(ss, cs, seed, lw)  # loads the library and sets the kernels' attributes outside the capture
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        with torch.cuda.graph(g, stream=s):
            out = scene.sample_crops(ss, cs, seed, lw)
    torch.cuda.current_stream().wait_stream(s)
    for v in (99, -4, 2 ** 40):
        seed.fill_(v)
        g.replay()
        want = scene.sample_crops(ss, cs, v, lw)
        torch.cuda.synchronize()
        for f in want._fields:
            assert torch.equal(getattr(out, f), getattr(want, f)), (v, f)


def test_rows_are_uniform():
    """In a crop of c > npoints members, each member is a row with probability npoints / c, and row 0 is spread
    over the members."""
    rs = np.random.RandomState(0)
    # in [0, 0.9]^2 x [0, 1]: every attempt's box (centre +- 0.95 in x and y) holds all 3000 points, so c = 3000
    pts = (rs.random_sample((3000, 3)) * [0.9, 0.9, 1.0]).astype(np.float32)
    ss = _set([(pts, np.ones(3000, np.int64))])
    lw = ss.train_label_weights()
    n, trials, b = 300, 200, 32
    counts = np.zeros(3000)
    first = np.zeros(3000)
    for t in range(trials):
        got = scene.sample_crops(ss, torch.zeros(b, dtype=torch.int64, device=DEV), 1000 + t, lw, npoints=n,
                                 max_dropout=0.0)
        pi = got.point_idx.cpu().numpy()
        assert (got.lengths.cpu().numpy() == n).all()
        np.add.at(counts, pi.reshape(-1), 1)
        np.add.at(first, pi[:, 0], 1)
    draws = trials * b
    p = n / 3000
    sd = np.sqrt(draws * p * (1 - p))
    assert np.abs(counts - draws * p).max() < 6 * sd
    assert (first > 0).sum() > 0.8 * (1 - np.exp(-draws / 3000)) * 3000  # row 0 reaches most members
    assert first.max() < 20


def test_training_step_on_crops():
    torch.manual_seed(0)
    ss = _set(_rooms((80000, 40000), seed0=5))
    net = nets.PointNet2SemSeg(21).to(DEV).train()
    crops = scene.sample_crops(ss, torch.tensor([0, 1, 0, 1], device=DEV), 3, ss.train_label_weights(), npoints=4096)
    captured = []
    h = net.sa1.register_forward_hook(lambda m, i, o: captured.append(o[2].clone()))
    try:
        pred, _ = net(crops.xyz, crops.lengths)
        loss = nets.sem_seg_loss(pred, crops.label, crops.weight, lengths=crops.lengths)
        assert torch.isfinite(loss)
        loss.backward()
        assert all(p.grad is None or torch.isfinite(p.grad).all() for p in net.parameters())
        assert any(p.grad is not None and p.grad.abs().sum() > 0 for p in net.parameters())
        sa1 = captured[0]
        lengths = crops.lengths.cpu().tolist()
        assert min(lengths) < 4096  # dropout made the batch ragged
        net.eval()
        for bi, ln in enumerate(lengths):
            captured.clear()
            with torch.no_grad():
                net(crops.xyz[bi:bi + 1, :ln].contiguous())
            assert torch.equal(captured[0][0], sa1[bi]), bi
    finally:
        h.remove()


def test_set_on_default_cuda_device():
    """A set built with device="cuda" (no index) samples crops with its own label weights."""
    room, lab = W.scene_room(20000, 2)
    for dev in ("cuda", torch.device("cuda")):
        ss = scene.SceneSet([room], [lab], device=dev)
        assert ss.device == ss.xyz.device and ss.device.index is not None
        got = scene.sample_crops(ss, torch.zeros(2, dtype=torch.int64, device=dev), 3, ss.train_label_weights(),
                                 npoints=1024)
        assert (got.lengths >= 1).all()
    ss = scene.SceneSet([room], [lab])  # the default: the current CUDA device
    scene.sample_crops(ss, torch.zeros(2, dtype=torch.int64, device="cuda"), 3, ss.train_label_weights(), npoints=64)


def test_launches_and_no_host_sync():
    ss = _set(_rooms((20000,)))
    cs = torch.zeros(3, dtype=torch.int64, device=DEV)
    lw = ss.train_label_weights()
    scene.sample_crops(ss, cs, 0, lw)
    seed = torch.tensor([4], device=DEV)
    torch.cuda.synchronize()
    before = _lib.launch_count()
    torch.cuda.set_sync_debug_mode("error")
    try:
        scene.sample_crops(ss, cs, seed, lw)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    assert _lib.launch_count() == before + 2
