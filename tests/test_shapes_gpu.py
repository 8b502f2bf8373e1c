"""GPU tests of the shape batches (shapes.sample_shapes / vote_batch / classify_votes): every output field against the
numpy oracle (shape_oracle.py), lengths / rows / labels / parts bit for bit and the points within one float32 ulp of
its float64 evaluation; exact gathers with every step off; determinism, seed dependence and a device seed replayed
through a CUDA graph; the distributions of the draws; voted classification; and ragged training steps on the batches."""
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import shape_oracle as SO  # noqa: E402

from pointnet2_b200 import _lib, nets, shapes as SH  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
OFF = dict(rotate=False, perturb=False, scale=None, shift=0, jitter=None)


def _shapes(sizes, seed=0, num_class=40, parts=True):
    rs = np.random.RandomState(seed)
    xyz = [rs.standard_normal((n, 3)).astype(np.float32) for n in sizes]
    nrm = [rs.standard_normal((n, 3)).astype(np.float32) for n in sizes]
    nrm = [n / np.linalg.norm(n, axis=1, keepdims=True) for n in nrm]
    part = [rs.randint(0, 50, n) for n in sizes] if parts else None
    return SH.ShapeSet(xyz, rs.randint(0, num_class, len(sizes)), nrm, part, num_class=num_class, normalize=False,
                       device=DEV)


def _host(ss):
    return dict(xyz=ss.xyz.cpu().numpy(), label=ss.label.cpu().numpy(), offsets=ss.offsets.cpu().numpy(),
                normals=ss.normals.cpu().numpy() if ss.normals is not None else None,
                part=ss.part.cpu().numpy() if ss.part is not None else None)


def _check(got, want):
    for f in ("lengths", "point_idx", "label") + (("part",) if "part" in want else ()):
        g = getattr(got, f).cpu().numpy()
        assert g.dtype == want[f].dtype, f
        np.testing.assert_array_equal(g, want[f], err_msg=f)
    pts = got.points.cpu().numpy()
    # one float32 ulp of the float64 value, plus 1e-12 absolute for the ~1e-16 differences between the kernel's and
    # numpy's sin / cos / log where a sum cancels to almost 0
    ulp = np.spacing(np.abs(want["points64"]).astype(np.float32)).astype(np.float64)
    assert (np.abs(pts.astype(np.float64) - want["points64"]) <= ulp + 1e-12).all()


def _run(ss, idx, seed, **kw):
    got = SH.sample_shapes(ss, torch.as_tensor(np.asarray(idx, np.int64), device=DEV), seed, **kw)
    h = _host(ss)
    want = SO.oracle_shapes(h["xyz"], h["label"], h["offsets"], idx, seed, normals=h["normals"], part=h["part"], **kw)
    return got, want


SIZES = [10000, 2048, 3000, 700, 1024, 1, 5000, 16384]


@pytest.mark.parametrize("b", [1, 7, 64])
@pytest.mark.parametrize("recipe", ["modelnet", "modelnet_normals", "part", "dropout_random", "first_off"])
def test_matches_oracle(recipe, b):
    ss = _shapes(SIZES, seed=b)
    idx = np.random.RandomState(b).randint(0, len(SIZES), b)
    kw = {"modelnet": {}, "modelnet_normals": dict(with_normals=True),
          "part": dict(subset="random", rotate=False, perturb=False, scale=None, shift=0, with_normals=True),
          "dropout_random": dict(subset="random", max_dropout=0.875),
          "first_off": dict(max_dropout=0.5, **OFF)}[recipe]
    for seed, npoints in [(3, 1024), (-11, 2048), (2 ** 64 - 5, 16384), (12, 100)]:
        got, want = _run(ss, idx, seed, npoints=npoints, **kw)
        _check(got, want)
        assert (want["lengths"] >= 1).all()


def test_shapes_without_parts_or_normals():
    ss = _shapes([500, 3000], parts=False)
    got, want = _run(ss, [0, 1, 1], 5, npoints=1024)
    assert got.part is None and "part" not in want
    _check(got, want)
    raw = SH.ShapeSet([np.random.RandomState(1).standard_normal((300, 3)).astype(np.float32)], [2], device=DEV)
    with pytest.raises(ValueError, match="normals"):
        SH.sample_shapes(raw, torch.zeros(1, dtype=torch.int64, device=DEV), 0, with_normals=True)


def test_every_step_off_is_an_exact_gather():
    ss = _shapes(SIZES)
    idx = torch.arange(len(SIZES), device=DEV)
    for subset in ("first", "random"):
        got = SH.sample_shapes(ss, idx, 9, npoints=4096, subset=subset, with_normals=True, **OFF)
        pi = got.point_idx.long()
        real = pi >= 0
        assert torch.equal(real.sum(1).int(), got.lengths)
        src = torch.cat([ss.xyz, ss.normals], 1)[pi.clamp(min=0)]
        assert torch.equal(got.points[real], src[real])
        assert torch.equal(got.part[real], ss.part[pi[real]].long())
        assert (got.points[~real] == 0).all() and (got.part[~real] == 0).all()
    # a single vote is a permuted copy of the first npoints rows
    v = SH.vote_batch(ss, idx, 1, 4, npoints=2048)
    off = ss.offsets.cpu().numpy()
    for e, n in enumerate(SIZES):
        m = min(n, 2048)
        rows = v.point_idx[e, :m].cpu().numpy()
        assert sorted(rows.tolist()) == list(range(off[e], off[e] + m))
        assert torch.equal(v.points[e, :m], ss.xyz[torch.from_numpy(rows).long().to(DEV)])


def test_votes_match_oracle():
    ss = _shapes(SIZES[:5])
    h = _host(ss)
    idx = np.array([4, 0, 2])
    for nv, kw in [(12, {}), (3, dict(with_normals=True, npoints=2048))]:
        got = SH.vote_batch(ss, torch.as_tensor(idx, device=DEV), nv, 21, **kw)
        want = SO.oracle_shapes(h["xyz"], h["label"], h["offsets"], idx, 21, votes=nv, normals=h["normals"],
                                part=h["part"], **kw)
        _check(got, want)
        assert got.points.shape[0] == nv * len(idx)


def test_same_seed_same_bits_other_seed_other_batch():
    ss = _shapes([3000, 10000, 600])
    idx = torch.tensor([0, 1, 2, 1, 0], device=DEV)
    a = SH.sample_shapes(ss, idx, 123, max_dropout=0.5)
    b = SH.sample_shapes(ss, idx, 123, max_dropout=0.5)
    c = SH.sample_shapes(ss, idx, 124, max_dropout=0.5)
    for f in ("points", "label", "part", "lengths", "point_idx"):
        assert torch.equal(getattr(a, f), getattr(b, f)), f
    assert not torch.equal(a.point_idx, c.point_idx) and not torch.equal(a.points, c.points)
    d = SH.sample_shapes(ss, idx, torch.tensor([123], device=DEV), max_dropout=0.5)
    e = SH.sample_shapes(ss, idx.to(torch.int32), 123, max_dropout=0.5)
    for f in ("points", "label", "part", "lengths", "point_idx"):
        assert torch.equal(getattr(a, f), getattr(d, f)), f
        assert torch.equal(getattr(a, f), getattr(e, f)), f


def test_out_of_range_shape_gives_empty_entry():
    ss = _shapes([500, 800])
    got = SH.sample_shapes(ss, torch.tensor([1, 2, -1], device=DEV), 1, npoints=512, with_normals=True)
    assert got.lengths.tolist() == [512, 0, 0] and got.label.tolist()[1:] == [0, 0]
    assert (got.point_idx[1:] == -1).all() and (got.points[1:] == 0).all() and (got.part[1:] == 0).all()


def test_device_seed_in_cuda_graph():
    ss = _shapes([3000, 10000])
    idx = torch.tensor([0, 1, 1, 0], device=DEV)
    seed = torch.tensor([1], device=DEV)
    kw = dict(max_dropout=0.875, with_normals=True, subset="random")
    SH.sample_shapes(ss, idx, seed, **kw)  # loads the library and sets the kernel's attributes outside the capture
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        with torch.cuda.graph(g, stream=s):
            out = SH.sample_shapes(ss, idx, seed, **kw)
    torch.cuda.current_stream().wait_stream(s)
    for v in (99, -4, 2 ** 40):
        seed.fill_(v)
        g.replay()
        want = SH.sample_shapes(ss, idx, v, **kw)
        torch.cuda.synchronize()
        for f in ("points", "label", "part", "lengths", "point_idx"):
            assert torch.equal(getattr(out, f), getattr(want, f)), (v, f)


def test_launches_and_no_host_sync():
    ss = _shapes([3000, 600])
    idx = torch.zeros(3, dtype=torch.int64, device=DEV)
    SH.sample_shapes(ss, idx, 0)
    seed = torch.tensor([4], device=DEV)
    model = nets.PointNet2ClsSSG(40).to(DEV).eval()
    SH.classify_votes(model, ss, idx, 2, 0)
    torch.cuda.synchronize()
    before = _lib.launch_count()
    torch.cuda.set_sync_debug_mode("error")
    try:
        SH.sample_shapes(ss, idx, seed, max_dropout=0.5, with_normals=True)
        SH.vote_batch(ss, idx, 3, seed)
        got = SH.sample_shapes(ss, idx, seed)
        SH.cls_accuracy(got.label, torch.zeros_like(got.label), 40)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    assert _lib.launch_count() == before + 3


def test_distributions():
    """Rows uniform over the pool, theta uniform, jitter clipped at 0.05 with about the expected spread, scale and
    shift inside their ranges."""
    rs = np.random.RandomState(0)
    pts = rs.standard_normal((400, 3)).astype(np.float32)
    ss = SH.ShapeSet([pts], [0], normalize=False, device=DEV)
    b, n, trials = 64, 40, 100
    counts = np.zeros(400)
    for t in range(trials):
        got = SH.sample_shapes(ss, torch.zeros(b, dtype=torch.int64, device=DEV), 1000 + t, npoints=n, subset="random",
                               **OFF)
        np.add.at(counts, got.point_idx.cpu().numpy().reshape(-1), 1)
    draws, p = trials * b, n / 400
    assert np.abs(counts - draws * p).max() < 6 * np.sqrt(draws * p * (1 - p))
    # theta: the rotation of the unit x axis about y lands at angle theta in the xz plane
    e = np.array([[1, 0, 0], [0, 0, 1], [0, 1, 0]], np.float32)
    ss3 = SH.ShapeSet([e], [0], normalize=False, device=DEV)
    th = []
    for t in range(20):
        got = SH.sample_shapes(ss3, torch.zeros(256, dtype=torch.int64, device=DEV), t, npoints=3, perturb=False,
                               scale=None, shift=0, jitter=None)
        p = got.points.cpu().numpy()
        rows = got.point_idx.cpu().numpy()
        x = p[np.arange(len(p)), np.argmax(rows == 0, axis=1)]
        th.append(np.arctan2(x[:, 2], x[:, 0]) % (2 * np.pi))  # (1, 0, 0) Ry = (cos, 0, sin)
    th = np.concatenate(th)
    hist = np.histogram(th, bins=16, range=(0, 2 * np.pi))[0]
    assert np.abs(hist - len(th) / 16).max() < 6 * np.sqrt(len(th) / 16)
    # jitter alone: the offsets from the source rows
    got = SH.sample_shapes(ss, torch.zeros(256, dtype=torch.int64, device=DEV), 5, npoints=400, rotate=False,
                           perturb=False, scale=None, shift=0)
    d = (got.points - ss.xyz[got.point_idx.long()]).cpu().numpy().reshape(-1)
    assert np.abs(d).max() <= 0.05 + 1e-6
    assert 0.0095 < d.std() < 0.0105 and abs(d.mean()) < 2e-4
    # scale and shift alone: one affine map per entry, inside (0.8, 1.25) and [-0.1, 0.1)
    got = SH.sample_shapes(ss, torch.zeros(512, dtype=torch.int64, device=DEV), 6, npoints=400, rotate=False,
                           perturb=False, jitter=None)
    src = ss.xyz[got.point_idx.long()].double().cpu().numpy()
    q = got.points.double().cpu().numpy()
    dq, ds = q - q.mean(1, keepdims=True), src - src.mean(1, keepdims=True)
    s = (dq * ds).sum((1, 2)) / (ds * ds).sum((1, 2))     # the least-squares scale of each entry
    t = q.mean(1) - src.mean(1) * s[:, None]
    assert (s > 0.8 - 1e-5).all() and (s < 1.25 + 1e-5).all() and s.min() < 0.85 and s.max() > 1.2
    assert (np.abs(t) <= 0.1 + 1e-5).all() and np.abs(t).max() > 0.09


def test_classify_votes_and_accuracy():
    torch.manual_seed(0)
    ss = _shapes([1024, 3000, 2048, 1500, 800], seed=3, num_class=10)
    idx = torch.tensor([0, 1, 2, 3, 4, 1], device=DEV)
    model = nets.PointNet2ClsSSG(10).to(DEV).eval()
    a = SH.classify_votes(model, ss, idx, 4, 7)
    b = SH.classify_votes(model, ss, idx, 4, 7)
    assert a.dtype == torch.float32 and a.shape == (6, 10) and torch.equal(a, b)
    c = SH.classify_votes(model, ss, idx, 4, 7, chunk=3)
    votes = SH.vote_batch(ss, idx, 4, 7)
    want = torch.zeros(6, 10, device=DEV)
    with torch.no_grad():
        for v in range(4):
            want += model(votes.points[v * 6:(v + 1) * 6], votes.lengths[v * 6:(v + 1) * 6])[0]
    torch.testing.assert_close(a, want, rtol=1e-4, atol=1e-4)
    torch.testing.assert_close(c, want, rtol=1e-4, atol=1e-4)
    pred = a.argmax(1)
    label = ss.label[idx].long()
    acc, cacc = SH.cls_accuracy(pred, label, 10)
    p, l = pred.cpu().numpy(), label.cpu().numpy()
    assert acc.item() == np.sum(p == l) / float(len(l))
    seen = np.array([np.sum(l == k) for k in range(10)], np.float64)
    correct = np.array([np.sum((p == l) & (l == k)) for k in range(10)])
    with np.errstate(invalid="ignore"):
        np.testing.assert_array_equal(cacc.item(), np.mean(correct / seen))


def test_training_steps_on_shape_batches():
    torch.manual_seed(0)
    ss = _shapes([10000, 3000, 2048, 700], seed=4)
    idx = torch.tensor([0, 1, 2, 3, 0, 1], device=DEV)
    net = nets.PointNet2ClsSSG(40).to(DEV).train()
    batch = SH.sample_shapes(ss, idx, 3, max_dropout=0.875)
    assert batch.lengths.min() < 1024 and batch.lengths.min() >= 1  # dropout made the batch ragged
    pred, _ = net(batch.points, batch.lengths)
    loss = nets.cls_loss(pred, batch.label)
    assert torch.isfinite(loss)
    loss.backward()
    assert all(p.grad is None or torch.isfinite(p.grad).all() for p in net.parameters())
    assert any(p.grad is not None and p.grad.abs().sum() > 0 for p in net.parameters())
    part_net = nets.PointNet2PartSeg().to(DEV).train()
    pb = SH.sample_shapes(ss, idx, 4, npoints=2048, subset="random", rotate=False, perturb=False, scale=None, shift=0,
                          with_normals=True)
    pred, _ = part_net(pb.points, pb.lengths)
    loss = nets.part_seg_loss(pred, pb.part, lengths=pb.lengths)
    assert torch.isfinite(loss)
    loss.backward()
    assert all(p.grad is None or torch.isfinite(p.grad).all() for p in part_net.parameters())
    assert any(p.grad is not None and p.grad.abs().sum() > 0 for p in part_net.parameters())
