"""GPU tests of per-cloud lengths for kNN: knn_point(lengths=, query_lengths=), sample_knn(lengths=) on both layer
paths, and pointnet_sa_module(knn=True, lengths=) (sample_and_group keeps refusing lengths with knn).

The ops are held to the contract's restatement on the C oracle (tests/knn_ragged_oracle.py), the layers to per-cloud
b = 1 calls.  Every case runs twice, once with poisoned padding (NaN, +inf and a far point) and once with padding that
copies real points, and the two runs must agree bit for bit."""
import numpy as np
import pytest
import torch

from knn_ragged_oracle import oracle_knn_ragged, oracle_sample_knn_ragged
from pointnet2_b200 import _lib, layers, workloads as W
from pointnet2_b200.pointnet_util import pointnet_sa_module, sample_and_group
from pointnet2_b200.sa_layer import sample_knn
from pointnet2_b200.tf_grouping import knn_point

pytestmark = pytest.mark.gpu

FAR = np.float32(50.0)
KS = [1, 31, 32, 33, 64, 65, 128]


def pad(x, lengths, kind):
    """x (b, n, c) with the rows of cloud i from lengths[i] on overwritten: 'poison' or 'copy'"""
    x = x.copy()
    for i, ln in enumerate(lengths):
        rows = np.arange(ln, x.shape[1])
        if kind == "poison":
            x[i, rows[0::3]] = np.nan
            x[i, rows[1::3]] = np.inf
            x[i, rows[2::3]] = FAR
        else:
            x[i, rows] = x[i, rows % ln]
    return x


def T(a, dev):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


def N(t):
    return t.detach().cpu().numpy()


def bits_equal(a, b):
    a, b = np.asarray(a), np.asarray(b)
    if a.dtype == np.float32:
        a, b = a.view(np.int32), np.asarray(b, np.float32).view(np.int32)
    return a.shape == b.shape and np.array_equal(a, b)


def both_paddings(fn, arrays, lengths_list, dev):
    """fn(*padded device tensors) for both paddings (array j padded with lengths_list[j], None = dense); the results
    must be bit-identical"""
    outs = []
    for kind in ("poison", "copy"):
        ts = [T(a if ls is None else pad(a, ls, kind), dev) for a, ls in zip(arrays, lengths_list)]
        outs.append([None if o is None else N(o) for o in fn(*ts)])
    for a, b in zip(*outs):
        assert (a is None and b is None) or bits_equal(a, b), "padding changed the result"
    return outs[0]


def data_lengths(n, k):
    return sorted({min(max(ln, 1), n) for ln in (1, k - 1, k, k + 1, 1023, 1024, 1025, n)})


# --------------------------------------------------------------------------------------------------------- knn_point
@pytest.mark.parametrize("k", KS)
@pytest.mark.parametrize("mode", ["data", "query", "both"])
def test_knn_point_ragged_matches_the_oracle(dev, k, mode):
    n, m = 1100, 37
    lens = data_lengths(n, k)
    b = len(lens)
    x = W.cloud_uniform(b, n, 100 + k)
    x[b // 2] = W.cloud_duplicates(1, n, 7 + k)[0]  # ties everywhere
    q = np.concatenate([x[:, :20], W.cloud_uniform(b, m - 20, 200 + k)], 1)  # copies of cloud points and free points
    qlens = [1 + (7 * i) % m for i in range(b)]
    use_l, use_q = mode in ("data", "both"), mode in ("query", "both")
    kw = lambda lt, qt: dict(lengths=lt if use_l else None, query_lengths=qt if use_q else None)  # noqa: E731
    lt, qt = torch.tensor(lens, dtype=torch.int32, device=dev), torch.tensor(qlens, dtype=torch.int32, device=dev)
    val, idx = both_paddings(lambda a, c: knn_point(k, a, c, **kw(lt, qt)), [x, q],
                             [lens if use_l else None, qlens if use_q else None], dev)
    wv, wi = oracle_knn_ragged(k, x, q, lens if use_l else None, qlens if use_q else None)
    assert np.array_equal(idx, wi)
    assert bits_equal(val, wv)


@pytest.mark.parametrize("k", KS)
def test_self_knn_of_a_ragged_batch(dev, k):
    n = 1030
    lens = data_lengths(n, k)
    x = W.cloud_surface(len(lens), n, 300 + k)
    lt = torch.tensor(lens, dtype=torch.int32, device=dev)
    val, idx = both_paddings(lambda a: knn_point(k, a, a, lengths=lt, query_lengths=lt), [x], [lens], dev)
    wv, wi = oracle_knn_ragged(k, x, x, lens, lens)
    assert np.array_equal(idx, wi) and bits_equal(val, wv)
    for i, ln in enumerate(lens):
        assert idx[i, :ln].max() < ln and np.all(idx[i, ln:] == 0) and np.all(np.isinf(val[i, ln:]))


# -------------------------------------------------------------------------------------------------------- sample_knn
@pytest.mark.parametrize("path", [1, 2])
@pytest.mark.parametrize("k", [16, 33, 64])
@pytest.mark.parametrize("center", [False, True])
def test_sample_knn_ragged_matches_the_oracle_chain(dev, path, k, center):
    n, m = 1500, 96
    lens = [n, 1, k - 1, k, k + 1, 1025, 700]
    b = len(lens)
    x = W.cloud_uniform(b, n, 400 + k)
    x[-1] = W.cloud_duplicates(1, n, 401 + k)[0]
    lib = _lib.load()
    try:
        lib.pn2_set_sa_knn_path(path)
        assert (int(lib.pn2_sa_knn_layer_workspace_bytes(b, n, m, k)) == 0) == (path == 1)
        lt = torch.tensor(lens, dtype=torch.int32, device=dev)
        got = both_paddings(lambda a: sample_knn(m, k, a, center=center, want_dist=True, lengths=lt), [x], [lens], dev)
    finally:
        lib.pn2_set_sa_knn_path(0)
    want = oracle_sample_knn_ragged(m, k, x, lens, center)
    for name, a, w in zip(("fps_idx", "new_xyz", "idx", "dist", "grouped_xyz"), got, want):
        assert bits_equal(a, w), name


def test_sample_knn_paths_agree_without_grouped_or_dist(dev):
    n, m, k = 2048, 256, 32
    lens = [n, 5, 31, 32, 33, 1500]
    x = T(pad(W.cloud_surface(len(lens), n, 500), lens, "poison"), dev)
    lib = _lib.load()
    outs = []
    try:
        for path in (1, 2):
            lib.pn2_set_sa_knn_path(path)
            outs.append(sample_knn(m, k, x, want_grouped=False, lengths=lens))
    finally:
        lib.pn2_set_sa_knn_path(0)
    for a, b in zip(*outs):
        assert (a is None and b is None) or torch.equal(a, b)


# ------------------------------------------------------------------------------------------ sample_and_group, SA module
def per_cloud(fn, x, feats, lens, k, grouped):
    """fn(xyz, points, nsample) on each truncated cloud alone (b = 1, nsample = min(k, length)), the outputs numbered
    in ``grouped`` with their nsample axis padded to k by repeating column 0"""
    outs = []
    for i, ln in enumerate(lens):
        kk = min(k, ln)
        o = fn(x[i:i + 1, :ln], None if feats is None else feats[i:i + 1, :ln], kk)
        fill = []
        for j, t in enumerate(o):
            if j in grouped and kk < k:
                t = torch.cat([t, t[:, :, :1].expand(*t.shape[:2], k - kk, *t.shape[3:])], 2)
            fill.append(t)
        outs.append(fill)
    return [torch.cat(ts, 0) for ts in zip(*outs)]


@pytest.mark.parametrize("fused", [True, False])
@pytest.mark.parametrize("points", ["none", "xyz_first", "features_only"])
def test_grouped_knn_features_equal_each_truncated_cloud(dev, fused, points):
    """the (b, npoint, nsample, channels) groups pointnet_sa_module(knn=True, lengths=) hands its mlp"""
    n, m, k = 1200, 64, 32
    lens = [n, 1, 31, 32, 33, 1024, 1025]
    x = W.cloud_uniform(len(lens), n, 600)
    f = W.features(len(lens), n, 5, 601)

    def groups(a, p, kk, lengths=None):
        seen = []

        def mlp(t):
            seen.append(t)
            return t
        new_xyz, _, idx = pointnet_sa_module(a, None if points == "none" else p, m, 0.2, kk, mlp, knn=True,
                                             use_xyz=points != "features_only", fused=fused, lengths=lengths)
        return new_xyz, seen[0], idx

    with torch.no_grad():
        got = both_paddings(lambda a, p: groups(a, p, k, lens), [x, f], [lens, lens], dev)
        want = per_cloud(groups, T(x, dev), T(f, dev), lens, k, grouped=(1, 2))
    for name, a, w in zip(("new_xyz", "groups", "idx"), got, want):
        assert bits_equal(a, N(w)), name


def test_sample_and_group_keeps_refusing_knn_lengths(dev):
    x = T(W.cloud_uniform(2, 64, 650), dev)
    for fused in (True, False):
        with pytest.raises(ValueError, match="knn"):
            sample_and_group(8, 0.2, 4, x, None, knn=True, fused=fused, lengths=[64, 10])


@pytest.mark.parametrize("tail", ["kernel", "torch"])
@pytest.mark.parametrize("fused", [True, False])
def test_pointnet_sa_module_knn_ragged_equals_each_truncated_cloud(dev, tail, fused):
    n, m, k = 1100, 48, 33
    lens = [n, 2, 32, 33, 34, 1025]
    x = W.cloud_surface(len(lens), n, 700)
    f = W.features(len(lens), n, 6, 701)
    torch.manual_seed(0)
    # kernel: an eval-mode SharedMLP, which the fused call hands to sa_mlp_max (fused=False keeps the torch layers);
    # torch: mlp=None, the grouped tensor max-pooled as is
    mlp = layers.SharedMLP(9, [16, 32]).to(dev).eval() if tail == "kernel" else None
    with torch.no_grad():
        got = both_paddings(lambda a, p: pointnet_sa_module(a, p, m, 0.2, k, mlp, knn=True, fused=fused, lengths=lens),
                            [x, f], [lens, lens], dev)
        want = per_cloud(lambda a, p, kk: pointnet_sa_module(a, p, m, 0.2, kk, mlp, knn=True, fused=fused),
                         T(x, dev), T(f, dev), lens, k, grouped=(2,))
    for name, a, w in zip(("new_xyz", "new_points", "idx"), got, want):
        if name == "new_points" and mlp is not None and not fused:  # cuBLAS may sum in another order for another b
            np.testing.assert_allclose(a, N(w), rtol=1e-5, atol=1e-6)
        else:
            assert bits_equal(a, N(w)), name
    assert not np.isnan(got[1]).any()


# ------------------------------------------------------------------------------------------------- lengths handling
def test_lengths_dtypes_and_clamping(dev):
    n, m, k = 600, 40, 20
    x = T(pad(W.cloud_uniform(4, n, 800), [n, 10, 300, 1], "copy"), dev)
    q = T(W.cloud_uniform(4, m, 801), dev)
    want = knn_point(k, x, q, lengths=torch.tensor([n, 10, 300, 1], dtype=torch.int32, device=dev))
    for lens in ([n, 10, 300, 1], np.array([n, 10, 300, 1], np.int64), torch.tensor([n, 10, 300, 1]),
                 torch.tensor([n, 10, 300, 1], dtype=torch.int64, device=dev),
                 torch.tensor([n + 50, 10, 300, -7], dtype=torch.int32, device=dev)):  # out of range on the device: clamped
        got = knn_point(k, x, q, lengths=lens)
        assert torch.equal(got[1], want[1]) and torch.equal(got[0], want[0])
    qgot = knn_point(k, x, q, query_lengths=torch.tensor([0, m + 9, 5, m], dtype=torch.int32, device=dev))
    qwant = knn_point(k, x, q, query_lengths=[1, m, 5, m])
    assert torch.equal(qgot[1], qwant[1]) and torch.equal(qgot[0], qwant[0])
    for bad in ([0, 5, 5, 5], [5, n + 1, 5, 5], [5, 5, 5]):
        with pytest.raises(ValueError):
            knn_point(k, x, q, lengths=bad)
        with pytest.raises(ValueError):
            sample_knn(16, k, x, lengths=bad)
    with pytest.raises(ValueError):
        knn_point(k, x, q, query_lengths=[1, m + 1, 1, 1])


def test_the_composite_path_refuses_lengths(dev):
    x4 = torch.zeros(2, 50, 4, device=dev)
    with pytest.raises(ValueError, match="lengths"):
        knn_point(4, x4, x4[:, :5].contiguous(), lengths=[50, 10])
    x = torch.zeros(2, 200, 3, device=dev)
    with pytest.raises(ValueError, match="lengths"):
        knn_point(129, x, x[:, :5].contiguous(), lengths=[200, 10])


@pytest.mark.parametrize("path", [1, 2])
def test_sample_knn_in_a_cuda_graph_follows_rewritten_lengths(dev, path):
    n, m, k = 2048, 256, 32
    x = T(pad(W.cloud_uniform(5, n, 900), [n] * 5, "copy"), dev)
    lens = torch.tensor([n, 1500, 31, 700, 1025], dtype=torch.int32, device=dev)
    lib = _lib.load()
    try:
        lib.pn2_set_sa_knn_path(path)
        st = torch.cuda.Stream(dev)
        st.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(st):
            sample_knn(m, k, x, want_dist=True, lengths=lens)  # warm-up outside the capture
        st.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=st):
            out = sample_knn(m, k, x, want_dist=True, lengths=lens)
        for new in ([n, 1500, 31, 700, 1025], [3, 2048, 1024, 32, 33], [n] * 5):
            lens.copy_(torch.tensor(new, dtype=torch.int32))  # an in-place write; the graph is not re-captured
            g.replay()
            torch.cuda.synchronize(dev)
            want = sample_knn(m, k, x, want_dist=True, lengths=new)
            for j, (a, w) in enumerate(zip(out, want)):
                assert torch.equal(a, w), (new, j)
    finally:
        lib.pn2_set_sa_knn_path(0)
