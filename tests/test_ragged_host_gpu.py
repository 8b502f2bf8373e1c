"""GPU tests of the host-buffer layer on packed variable-size clouds (pn2_sa_layer_host_ragged, SetAbstractionHost /
SetAbstractionPipeline with ragged=True) and of SetAbstractionDevice with lengths.

Every cloud must get, bit for bit, what pn2_sa_layer_device_ragged computes on the same clouds padded to the capacity
(and through that what the dense layer computes on the cloud alone), whatever the capacity."""
import numpy as np
import pytest
import torch

from oracle import oracle as O
from pointnet2_b200 import _lib, workloads as W
from pointnet2_b200.host import SetAbstractionHost, SetAbstractionPipeline
from pointnet2_b200.sa_layer import SetAbstractionDevice, sample_group

pytestmark = pytest.mark.gpu


def lattice(b, n, seed):
    """points of a shuffled integer lattice: many exactly equal distances"""
    side = int(np.ceil(n ** (1 / 3)))
    g = np.stack(np.meshgrid(*[np.arange(side)] * 3, indexing="ij"), -1).reshape(-1, 3).astype(np.float32) / side
    rng = np.random.default_rng(seed)
    return np.stack([g[rng.permutation(len(g))[:n]] for _ in range(b)])


GEN = {"U": W.cloud_uniform, "S": W.cloud_surface, "D": W.cloud_duplicates, "L": lattice}


def clouds_of(x, lengths):
    return [np.ascontiguousarray(x[i, :l]) for i, l in enumerate(lengths)]


def padded(clouds, n):
    """the clouds padded to n rows with poison (NaN, +inf, a far point) that no kernel may read"""
    x = np.empty((len(clouds), n, 3), np.float32)
    x[:, 0::3], x[:, 1::3], x[:, 2::3] = np.nan, np.inf, 50.0
    for i, c in enumerate(clouds):
        x[i, :len(c)] = c
    return x


def bits(a):
    a = np.asarray(a)
    return a.view(np.int32) if a.dtype == np.float32 else a


def assert_same(got, want, what=""):
    for name, a, w in zip(("new_xyz", "idx", "pts_cnt", "grouped_xyz"), got, want):
        if a is None or w is None:
            assert a is None and w is None, name
            continue
        np.testing.assert_array_equal(bits(a), bits(w), err_msg=f"{what} {name}")


def device_reference(clouds, n, m, r, s, dev, want_grouped=True):
    """pn2_sa_layer_device_ragged on the clouds padded to n, as host arrays in the host layer's order"""
    x = torch.from_numpy(padded(clouds, n)).to(dev)
    _, nx, idx, cnt, g = sample_group(m, r, s, x, center=False, want_grouped=want_grouped, lengths=[len(c) for c in clouds])
    return nx.cpu().numpy(), idx.cpu().numpy(), cnt.cpu().numpy(), (g.cpu().numpy() if g is not None else None)


CASES = [
    # gen, capacity n, npoint, radius, nsample, lengths: the stride is max(lengths)
    ("U", 4096, 1024, 0.1, 32, [1500, 1, 700, 2047, 513, 3, 1024]),           # stride < 2048: brute-force ball query
    ("D", 4096, 512, 0.1, 32, [4096, 4095, 1, 2, 3000, 511]),                  # duplicate-heavy, full stride
    ("L", 4096, 256, 0.15, 16, [2197, 1000, 7, 2048]),                         # lattice ties, stride 2197 >= 2048
    ("S", 16384, 512, 0.1, 32, [9700, 5000, 1, 2049, 600]),                    # stride 9700: the largest overlapped grid
    ("U", 20000, 256, 0.05, 32, [16384, 9701, 3, 12000]),                      # stride > 9700: the sequential layer
]


@pytest.mark.parametrize("gen,n,m,r,s,lengths", CASES)
def test_equals_the_padded_device_layer(dev, gen, n, m, r, s, lengths):
    x = GEN[gen](len(lengths), max(lengths), 101)
    x[0, min(5, lengths[0] - 1), 1] = np.nan  # a NaN coordinate inside a real row
    clouds = clouds_of(x, lengths)
    sess = SetAbstractionHost(len(lengths), n, m, r, s, device=dev, ragged=True)
    got = sess.run(clouds)
    assert sess.h2d_bytes == 4 * len(lengths) + 12 * sum(lengths)
    assert_same(got, device_reference(clouds, n, m, r, s, dev), gen)


@pytest.mark.parametrize("gen,n,m,r,s,lengths", [CASES[0], CASES[2]])
def test_equals_the_oracle_on_each_truncated_cloud(dev, gen, n, m, r, s, lengths):
    x = GEN[gen](len(lengths), max(lengths), 102)
    clouds = clouds_of(x, lengths)
    new_xyz, idx, cnt, grouped = SetAbstractionHost(len(lengths), n, m, r, s, device=dev, ragged=True).run(clouds)
    for i, c in enumerate(clouds):
        c = c[None]
        o_new = O.oracle_gather_point(c, O.oracle_fps(m, c))
        o_idx, o_cnt = O.oracle_query_ball_point(r, s, c, o_new)
        np.testing.assert_array_equal(bits(new_xyz[i:i + 1]), bits(o_new), err_msg=f"cloud {i}")
        np.testing.assert_array_equal(idx[i:i + 1], o_idx, err_msg=f"cloud {i}")
        np.testing.assert_array_equal(cnt[i:i + 1], o_cnt, err_msg=f"cloud {i}")
        np.testing.assert_array_equal(bits(grouped[i:i + 1]), bits(O.oracle_group_point(c, o_idx)), err_msg=f"cloud {i}")


@pytest.mark.parametrize("gen,n,m,r,s,lengths", [CASES[0], CASES[1], CASES[3]])
def test_the_capacity_does_not_change_a_bit(dev, gen, n, m, r, s, lengths):
    clouds = clouds_of(GEN[gen](len(lengths), max(lengths), 103), lengths)
    a = SetAbstractionHost(len(lengths), n, m, r, s, device=dev, ragged=True).run(clouds)
    b = SetAbstractionHost(len(lengths), 4 * n, m, r, s, device=dev, ragged=True).run(clouds)
    assert_same(a, b, "capacity 4n")


@pytest.mark.parametrize("b,n,m", [(4, 1024, 256), (32, 4096, 1024), (2, 16384, 512)])
def test_full_lengths_equal_the_dense_host_layer(dev, b, n, m):
    x = W.cloud_uniform(b, n, 104)
    want = SetAbstractionHost(b, n, m, 0.1, 32, device=dev).run(x)
    got = SetAbstractionHost(b, n, m, 0.1, 32, device=dev, ragged=True).run(list(x))
    assert_same(got, want, "dense")


@pytest.mark.parametrize("n,lengths", [(4096, [3000, 4096, 10]), (20000, [16384, 12000, 3])])  # overlapped, sequential
def test_no_grouping_launch_without_grouped_xyz(dev, n, lengths):
    m, r, s = 256, 0.1, 16
    clouds = clouds_of(W.cloud_uniform(len(lengths), max(lengths), 105), lengths)
    full = SetAbstractionHost(len(lengths), n, m, r, s, device=dev, ragged=True)
    lean = SetAbstractionHost(len(lengths), n, m, r, s, device=dev, ragged=True, want_grouped=False)
    want = full.run(clouds)  # warm-up: every function attribute is set
    lean.run(clouds)
    ref = device_reference(clouds, max(lengths), m, r, s, dev, want_grouped=False)

    def launches(fn):
        torch.cuda.synchronize(dev)
        before = _lib.launch_count()
        out = fn()
        torch.cuda.synchronize(dev)
        return _lib.launch_count() - before, out

    k_full, _ = launches(lambda: full.run(clouds))
    k_lean, got = launches(lambda: lean.run(clouds))
    k_dev, _ = launches(lambda: device_reference(clouds, max(lengths), m, r, s, dev, want_grouped=False))
    assert got[3] is None
    assert_same(got[:3], want[:3], "lean")
    assert_same(got[:3], ref[:3], "device")
    assert k_lean == k_dev + 1  # the unpack kernel, then the device layer at the stride of the longest cloud
    sequential = max(lengths) > 9700
    assert k_full - k_lean == (1 if sequential else 0)  # the grouping kernel of the sequential layer; fused otherwise


def random_lengths(rng, b, lo, hi):
    return [int(v) for v in rng.integers(lo, hi + 1, b)]


@pytest.mark.parametrize("depth", [1, 3])
def test_pipeline_returns_mixed_batches_in_order(dev, depth):
    b, n, m, r, s = 8, 4096, 512, 0.1, 32
    rng = np.random.default_rng(106 + depth)
    batches = []
    for k in range(6):
        lens = random_lengths(rng, b, n // 2, n) if k % 2 == 0 else random_lengths(rng, b, 1, n // 3)
        batches.append(clouds_of(W.cloud_uniform(b, max(lens), 200 + k), lens))
    wants = [device_reference(c, n, m, r, s, dev) for c in batches]
    pipe = SetAbstractionPipeline(b, n, m, r, s, depth=depth, device=dev, ragged=True)
    got = []
    for k, clouds in enumerate(batches):
        if pipe.full():
            got.append([a.copy() if a is not None else None for a in pipe.collect()])
        if k % 3 == 2:  # the caller packs into the slot's pinned buffer itself
            buf = pipe.input_buffer()
            assert buf.shape == (b * n, 3)
            buf[:sum(map(len, clouds))] = np.concatenate(clouds)
            pipe.submit(lengths=[len(c) for c in clouds])
        else:
            pipe.submit(clouds)
        assert pipe.h2d_bytes == 4 * b + 12 * sum(map(len, clouds))
    while pipe.pending():
        got.append([a.copy() if a is not None else None for a in pipe.collect()])
    assert len(got) == len(batches)
    for k, (g, w) in enumerate(zip(got, wants)):
        assert_same(g, w, f"batch {k}")
    with pytest.raises(ValueError):
        pipe.submit()  # a ragged submit needs clouds or lengths
    with pytest.raises(ValueError):
        pipe.submit([np.zeros((n + 1, 3), np.float32)] * b)


def test_device_pipeline_with_lengths_equals_sample_group(dev):
    b, n, m, r, s = 6, 4096, 512, 0.1, 32
    lens = [4096, 3000, 1, 700, 2049, 4095]
    xs = [torch.from_numpy(padded(clouds_of(W.cloud_surface(b, n, 300 + k), lens), n)).to(dev) for k in range(4)]
    dl = torch.tensor(lens, dtype=torch.int32, device=dev)
    wants = [sample_group(m, r, s, x, center=False, lengths=lens) for x in xs]
    sa = SetAbstractionDevice(b, n, m, r, s, depth=2, center=False, device=dev)
    got = []
    for k, x in enumerate(xs):
        if sa.full():
            got.append([t.clone() for t in sa.collect(sync=True)])
        sa.submit(x, lengths=dl if k % 2 else lens)
    while sa.pending():
        got.append([t.clone() for t in sa.collect(sync=True)])
    for g, w in zip(got, wants):
        for a, v in zip(g, w):
            assert torch.equal(a, v)


def test_device_layer_with_lengths_in_a_cuda_graph(dev):
    b, n, m, r, s = 6, 4096, 512, 0.1, 32
    x = torch.from_numpy(W.cloud_uniform(b, n, 301)).to(dev)
    lens = torch.tensor([n, 3000, 513, 1000, 7, 2049], dtype=torch.int32, device=dev)
    sa = SetAbstractionDevice(b, n, m, r, s, depth=1, center=False, device=dev)
    slot = sa.slots[0]
    st = torch.cuda.Stream(dev)
    st.wait_stream(torch.cuda.current_stream(dev))
    with torch.cuda.stream(st):
        sa.enqueue(slot, x, st, lens)  # warm-up outside the capture (function attributes)
    st.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=st):
        sa.enqueue(slot, x, torch.cuda.current_stream(dev), lens)
    for new in ([n, 3000, 513, 1000, 7, 2049], [5, 4096, 1111, 2, 4000, 600], [n] * 6):
        lens.copy_(torch.tensor(new, dtype=torch.int32))  # an in-place write; the graph is not re-captured
        for k in ("fps_idx", "new_xyz", "idx", "pts_cnt", "grouped"):
            slot[k].zero_()
        g.replay()
        torch.cuda.synchronize(dev)
        want = sample_group(m, r, s, x, center=False, lengths=new)
        for k, w in zip(("fps_idx", "new_xyz", "idx", "pts_cnt", "grouped"), want):
            assert torch.equal(slot[k], w), (new, k)
