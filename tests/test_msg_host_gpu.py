"""GPU tests of the multi-scale host-buffer layer (pn2_sa_layer_msg_host, pn2_sa_layer_msg_host_ragged, and
SetAbstractionHost / SetAbstractionPipeline with radius and nsample sequences).

Every output must be, bit for bit, what sa_layer.sample_group_msg(center=False) computes on the same clouds on the
device, and each scale what the single-scale host layer computes for that scale alone, since the sampling is shared.
The layer's path depends on n only: up to 8192 points the sampling runs one CTA per cloud and every scale's ball query
overlaps it; 16384 points take clustered sampling and the sequential ops.  A radius of 1.5 or 2.0 puts most of the
unit cloud in every ball, the ball query's dense-ball case."""
import numpy as np
import pytest
import torch

from oracle import oracle as O
from pointnet2_b200 import _lib, workloads as W
from pointnet2_b200.host import SetAbstractionHost, SetAbstractionPipeline
from pointnet2_b200.sa_layer import sample_group_msg
from test_ragged_host_gpu import GEN, bits, clouds_of, padded

pytestmark = pytest.mark.gpu

WANTS = {"all": True, "none": False, "some": "some"}


def want_flags(want, k):
    """want_grouped for k scales: True, False, or every other scale from the first"""
    return [j % 2 == 0 for j in range(k)] if want == "some" else want


def device_reference(x, m, radii, nsamples, dev, lengths=None):
    """sample_group_msg(center=False) on the dense or padded batch x, as host arrays in the host layer's order"""
    _, nx, idx, cnt, g = sample_group_msg(m, radii, nsamples, torch.from_numpy(x).to(dev), center=False, lengths=lengths)
    return nx.cpu().numpy(), [t.cpu().numpy() for t in idx], [t.cpu().numpy() for t in cnt], [t.cpu().numpy() for t in g]


def assert_same(got, want, wants, what=""):
    """got: the host layer's (new_xyz, [idx], [cnt], [grouped] or None); want: a full reference; wants: the flags"""
    k = len(want[1])
    flags = [wants] * k if isinstance(wants, bool) else list(wants)
    np.testing.assert_array_equal(bits(got[0]), bits(want[0]), err_msg=f"{what} new_xyz")
    assert len(got[1]) == len(got[2]) == k
    for j in range(k):
        np.testing.assert_array_equal(got[1][j], want[1][j], err_msg=f"{what} idx scale {j}")
        np.testing.assert_array_equal(got[2][j], want[2][j], err_msg=f"{what} pts_cnt scale {j}")
    if not any(flags):
        assert got[3] is None, what
        return
    assert len(got[3]) == k
    for j in range(k):
        if flags[j]:
            np.testing.assert_array_equal(bits(got[3][j]), bits(want[3][j]), err_msg=f"{what} grouped_xyz scale {j}")
        else:
            assert got[3][j] is None, (what, j)


def d2h_bytes(b, m, nsamples, flags):
    return 4 * b * m * 3 + sum(4 * b * m * (s + 1) + (12 * b * m * s if w else 0) for s, w in zip(nsamples, flags))


DENSE = [
    # gen, b, n, npoint, radii, nsamples
    ("U", 8, 1024, 512, [0.1, 0.2, 0.4], [16, 32, 128]),     # the cls_msg level-1 layer, overlapped
    ("S", 4, 4096, 1024, [0.1, 0.2, 0.4], [16, 32, 128]),
    ("D", 3, 2048, 256, [0.05, 0.3], [8, 40]),                # duplicate-heavy
    ("L", 4, 2197, 300, [0.15, 1.5], [16, 64]),               # lattice ties; a ball holding most of the cloud
    ("U", 2, 16384, 512, [0.1, 0.2, 0.4], [16, 32, 128]),     # clustered sampling: the sequential layer
    ("S", 2, 16384, 256, [0.05, 2.0], [8, 128]),              # sequential, with a ball holding most of the cloud
]


@pytest.mark.parametrize("want", list(WANTS))
@pytest.mark.parametrize("gen,b,n,m,radii,nsamples", DENSE)
def test_dense_equals_the_device_layer(dev, gen, b, n, m, radii, nsamples, want):
    x = GEN[gen](b, n, 501)
    x[0, 5, 1] = np.nan  # a NaN coordinate
    flags = want_flags(WANTS[want], len(radii))
    sess = SetAbstractionHost(b, n, m, radii, nsamples, device=dev, want_grouped=flags)
    got = sess.run(x)
    assert_same(got, device_reference(x, m, radii, nsamples, dev), flags, f"{gen} {n}")
    assert sess.h2d_bytes == 12 * b * n
    assert sess.d2h_bytes == d2h_bytes(b, m, nsamples, [flags] * len(radii) if isinstance(flags, bool) else flags)


@pytest.mark.parametrize("gen,b,n,m,radii,nsamples", [DENSE[0], DENSE[3], DENSE[4]])
def test_each_scale_equals_the_single_scale_host_layer(dev, gen, b, n, m, radii, nsamples):
    x = GEN[gen](b, n, 502)
    new_xyz, idx, cnt, grouped = SetAbstractionHost(b, n, m, radii, nsamples, device=dev).run(x)
    for j, (r, s) in enumerate(zip(radii, nsamples)):
        w = SetAbstractionHost(b, n, m, r, s, device=dev).run(x)
        np.testing.assert_array_equal(bits(new_xyz), bits(w[0]), err_msg=f"scale {j}")
        np.testing.assert_array_equal(idx[j], w[1], err_msg=f"scale {j}")
        np.testing.assert_array_equal(cnt[j], w[2], err_msg=f"scale {j}")
        np.testing.assert_array_equal(bits(grouped[j]), bits(w[3]), err_msg=f"scale {j}")


RAGGED = [
    # gen, capacity n, npoint, radii, nsamples, lengths: the stride is max(lengths)
    ("U", 1024, 512, [0.1, 0.2, 0.4], [16, 32, 128], [1024, 600, 1, 513, 1000, 3, 700, 512]),  # cls_msg level 1
    ("U", 4096, 1024, [0.1, 0.2], [16, 32], [1500, 1, 700, 2047, 513, 3, 1024]),                 # stride < 2048
    ("D", 4096, 512, [0.1, 0.3], [32, 64], [4096, 4095, 1, 2, 3000, 511]),                       # full stride
    ("L", 4096, 256, [0.15, 1.5], [16, 64], [2197, 1000, 7, 2048]),                              # lattice ties
    ("S", 16384, 512, [0.1, 0.2], [16, 32], [8192, 5000, 1, 2049, 600]),                         # overlapped at stride 8192
    ("U", 20000, 256, [0.05, 0.2], [32, 16], [16384, 9701, 3, 12000]),                           # sequential layer
]


@pytest.mark.parametrize("gen,n,m,radii,nsamples,lengths", RAGGED)
def test_ragged_equals_the_padded_device_layer(dev, gen, n, m, radii, nsamples, lengths):
    x = GEN[gen](len(lengths), max(lengths), 503)
    x[0, min(5, lengths[0] - 1), 1] = np.nan  # a NaN coordinate inside a real row
    clouds = clouds_of(x, lengths)
    want = device_reference(padded(clouds, n), m, radii, nsamples, dev, lengths=lengths)
    for flags in (True, [False] + [True] * (len(radii) - 1)):
        sess = SetAbstractionHost(len(lengths), n, m, radii, nsamples, device=dev, ragged=True, want_grouped=flags)
        assert_same(sess.run(clouds), want, flags, f"{gen} {flags}")
        assert sess.h2d_bytes == 4 * len(lengths) + 12 * sum(lengths)


@pytest.mark.parametrize("gen,n,m,radii,nsamples,lengths", [RAGGED[0], RAGGED[3], RAGGED[5]])
def test_ragged_equals_the_dense_entry_on_each_cloud_alone(dev, gen, n, m, radii, nsamples, lengths):
    clouds = clouds_of(GEN[gen](len(lengths), max(lengths), 504), lengths)
    got = SetAbstractionHost(len(lengths), n, m, radii, nsamples, device=dev, ragged=True).run(clouds)
    for i, c in enumerate(clouds):
        w = SetAbstractionHost(1, len(c), m, radii, nsamples, device=dev).run(c[None])
        row = (got[0][i:i + 1], [a[i:i + 1] for a in got[1]], [a[i:i + 1] for a in got[2]], [a[i:i + 1] for a in got[3]])
        assert_same(row, w, True, f"cloud {i}")


@pytest.mark.parametrize("gen,n,m,radii,nsamples,lengths", [RAGGED[0], RAGGED[2], RAGGED[4]])
def test_ragged_capacity_does_not_change_a_bit(dev, gen, n, m, radii, nsamples, lengths):
    clouds = clouds_of(GEN[gen](len(lengths), max(lengths), 505), lengths)
    a = SetAbstractionHost(len(lengths), n, m, radii, nsamples, device=dev, ragged=True).run(clouds)
    b = SetAbstractionHost(len(lengths), 4 * n, m, radii, nsamples, device=dev, ragged=True).run(clouds)
    assert_same(a, b, True, "capacity 4n")


@pytest.mark.parametrize("b,n,m", [(32, 1024, 512), (4, 4096, 1024), (2, 16384, 512)])
def test_ragged_full_lengths_equal_the_dense_entry(dev, b, n, m):
    radii, nsamples = [0.1, 0.2, 0.4], [16, 32, 128]
    x = W.cloud_uniform(b, n, 506)
    want = SetAbstractionHost(b, n, m, radii, nsamples, device=dev).run(x)
    got = SetAbstractionHost(b, n, m, radii, nsamples, device=dev, ragged=True).run(list(x))
    assert_same(got, want, True, "dense")


def test_ragged_equals_the_oracle_on_each_truncated_cloud(dev):
    n, m, radii, nsamples, lengths = 1024, 128, [0.1, 0.25], [8, 32], [1024, 300, 1, 77]
    clouds = clouds_of(W.cloud_surface(len(lengths), n, 507), lengths)
    new_xyz, idx, cnt, grouped = SetAbstractionHost(len(lengths), n, m, radii, nsamples, device=dev, ragged=True).run(clouds)
    for i, c in enumerate(clouds):
        c = c[None]
        o_new = O.oracle_gather_point(c, O.oracle_fps(m, c))
        np.testing.assert_array_equal(bits(new_xyz[i:i + 1]), bits(o_new), err_msg=f"cloud {i}")
        for j, (r, s) in enumerate(zip(radii, nsamples)):
            o_idx, o_cnt = O.oracle_query_ball_point(r, s, c, o_new)
            np.testing.assert_array_equal(idx[j][i:i + 1], o_idx, err_msg=f"cloud {i} scale {j}")
            np.testing.assert_array_equal(cnt[j][i:i + 1], o_cnt, err_msg=f"cloud {i} scale {j}")
            np.testing.assert_array_equal(bits(grouped[j][i:i + 1]), bits(O.oracle_group_point(c, o_idx)),
                                          err_msg=f"cloud {i} scale {j}")


def launches(dev, fn):
    torch.cuda.synchronize(dev)
    before = _lib.launch_count()
    out = fn()
    torch.cuda.synchronize(dev)
    return _lib.launch_count() - before, out


@pytest.mark.parametrize("want", list(WANTS))
def test_launch_counts_on_the_overlapped_path(dev, want):
    b, n, m, radii, nsamples = 8, 1024, 512, [0.1, 0.2, 0.4], [16, 32, 128]
    flags = want_flags(WANTS[want], len(radii))
    x = W.cloud_uniform(b, n, 508)
    lengths = [n, 700, 1, 1000, 513, n, 64, 900]
    dense = SetAbstractionHost(b, n, m, radii, nsamples, device=dev, want_grouped=flags)
    ragged = SetAbstractionHost(b, n, m, radii, nsamples, device=dev, want_grouped=flags, ragged=True)
    clouds = clouds_of(x, lengths)
    dense.run(x)  # warm-up: every function attribute is set
    ragged.run(clouds)
    k_dense, _ = launches(dev, lambda: dense.run(x))
    k_ragged, _ = launches(dev, lambda: ragged.run(clouds))
    assert k_dense == 1 + len(radii)  # one sampling launch, one consumer grid per scale
    assert k_ragged == k_dense + 1  # and the unpack kernel


def test_ragged_launches_the_device_layer_and_the_unpack_kernel_on_the_sequential_path(dev):
    n, m, radii, nsamples, lengths = 20000, 256, [0.05, 0.2], [32, 16], [16384, 9701, 3, 12000]
    clouds = clouds_of(W.cloud_uniform(len(lengths), max(lengths), 509), lengths)
    sess = SetAbstractionHost(len(lengths), n, m, radii, nsamples, device=dev, ragged=True, want_grouped=False)
    sess.run(clouds)
    x = padded(clouds, max(lengths))
    k_host, _ = launches(dev, lambda: sess.run(clouds))
    k_dev, _ = launches(dev, lambda: sample_group_msg(m, radii, nsamples, torch.from_numpy(x).to(dev), center=False,
                                                      want_grouped=False, lengths=lengths))
    assert k_host == k_dev + 1


def random_lengths(rng, b, lo, hi):
    return [int(v) for v in rng.integers(lo, hi + 1, b)]


@pytest.mark.parametrize("ragged", [False, True])
@pytest.mark.parametrize("depth", [1, 3])
def test_pipeline_returns_batches_in_order(dev, depth, ragged):
    b, n, m, radii, nsamples = 8, 2048, 512, [0.1, 0.2, 0.4], [16, 32, 64]
    flags = [True, False, True]
    rng = np.random.default_rng(510 + depth)
    batches, wants = [], []
    for k in range(6):
        x = W.DISTRIBUTIONS["USD"[k % 3]](b, n, 600 + k)
        if ragged:
            lens = random_lengths(rng, b, n // 2, n) if k % 2 == 0 else random_lengths(rng, b, 1, n // 3)
            clouds = clouds_of(x, lens)
            batches.append(clouds)
            wants.append(device_reference(padded(clouds, n), m, radii, nsamples, dev, lengths=lens))
        else:
            batches.append(x)
            wants.append(device_reference(x, m, radii, nsamples, dev))
    pipe = SetAbstractionPipeline(b, n, m, radii, nsamples, depth=depth, device=dev, want_grouped=flags, ragged=ragged)
    assert pipe.d2h_bytes == d2h_bytes(b, m, nsamples, flags)
    got = []
    copy = lambda v: [copy(a) for a in v] if isinstance(v, list) else (v.copy() if v is not None else None)  # noqa: E731
    for k, batch in enumerate(batches):
        if pipe.full():
            got.append(copy(list(pipe.collect())))
        if ragged and k % 3 == 2:  # the caller packs into the slot's pinned buffer itself
            buf = pipe.input_buffer()
            assert buf.shape == (b * n, 3)
            buf[:sum(map(len, batch))] = np.concatenate(batch)
            pipe.submit(lengths=[len(c) for c in batch])
        elif not ragged and k % 3 == 2:
            pipe.input_buffer()[...] = batch
            pipe.submit()
        else:
            pipe.submit(batch)
        assert pipe.h2d_bytes == (4 * b + 12 * sum(map(len, batch)) if ragged else 12 * b * n)
    while pipe.pending():
        got.append(copy(list(pipe.collect())))
    assert len(got) == len(batches)
    for k, (g, w) in enumerate(zip(got, wants)):
        assert_same(g, w, flags, f"batch {k}")
    if ragged:
        with pytest.raises(ValueError):
            pipe.submit()  # a ragged submit needs clouds or lengths
        with pytest.raises(ValueError):
            pipe.submit([np.zeros((n + 1, 3), np.float32)] * b)
    else:
        with pytest.raises(ValueError):
            pipe.submit(lengths=[n] * b)  # lengths need ragged=True
    assert not pipe.pending()


def test_scalar_arguments_keep_the_single_scale_layer(dev):
    """radius and nsample scalars: the same entry and the same tuple as before, not lists"""
    b, n, m = 4, 1024, 256
    x = W.cloud_uniform(b, n, 511)
    new_xyz, idx, cnt, grouped = SetAbstractionHost(b, n, m, 0.2, 32, device=dev).run(x)
    assert idx.shape == (b, m, 32) and cnt.shape == (b, m) and grouped.shape == (b, m, 32, 3)
    one = SetAbstractionHost(b, n, m, [0.2], [32], device=dev).run(x)
    assert isinstance(one[1], list) and len(one[1]) == 1
    assert_same(one, (new_xyz, [idx], [cnt], [grouped]), True, "one scale")
