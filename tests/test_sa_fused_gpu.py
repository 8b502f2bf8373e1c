"""GPU tests of the overlapped sampling+grouping layer (csrc/sa_fused.cu): pn2_sa_layer_device and
pn2_ball_group must be BIT-IDENTICAL to the four separate ops (which test_parity_gpu.py pins to
the oracle, the goldens and the rebuilt reference kernels), in every regime of the consumer kernel:
uniform grid, index-ordered scan, dense-ball overflow, NaN data, NaN / out-of-box queries, rows with
no hit, npoint > n, and the sequential fallback for clouds the shared-memory grid cannot hold."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import oracle as O
from pointnet2_b200 import _lib, workloads as W
from pointnet2_b200.host import SetAbstractionHost
from pointnet2_b200.sa_layer import SetAbstractionDevice, ball_group, sample_group, sample_group_msg
from pointnet2_b200.tf_grouping import group_point, query_ball_point
from pointnet2_b200.tf_sampling import farthest_point_sample, farthest_point_sample_and_gather, gather_point

pytestmark = pytest.mark.gpu


def T(a, dev):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


def brute_force_query(radius, nsample, x, q):
    """query_ball_point on the brute-force kernel: in the automatic mode, 2048 <= n <= 9727 with b * m >= 4096 runs
    ball_group_kernel, and the layer and ball_group would be compared with themselves"""
    lib = _lib.load()
    try:
        lib.pn2_set_bq_mode(1)
        return query_ball_point(radius, nsample, x, q)
    finally:
        lib.pn2_set_bq_mode(0)


def sequential(npoint, radius, nsample, x, center):
    fi = farthest_point_sample(npoint, x)
    nx = gather_point(x, fi)
    idx, cnt = brute_force_query(radius, nsample, x, nx)
    g = group_point(x, idx)
    if center:
        g = g - nx.unsqueeze(2)
    return fi, nx, idx, cnt, g


LAYER_CASES = [
    # gen, b, n, npoint, radius, nsample
    ("U", 4, 4096, 1024, 0.1, 32),     # cfg2 shape: sparse balls -> grid
    ("S", 3, 4096, 512, 0.1, 32),      # surface-like: dense cells -> ordered scan
    ("D", 3, 8192, 1024, 0.1, 32),     # cfg4 L1: duplicate-heavy
    ("U", 2, 1024, 512, 0.2, 32),
    ("S", 2, 1024, 512, 0.4, 128),     # cfg3 L1 widest scale
    ("U", 2, 512, 128, 0.8, 128),      # every point in every ball
    ("U", 2, 700, 64, 0.02, 16),       # nearly empty balls
    ("U", 1, 9700, 300, 0.05, 24),     # at the shared-memory limit
    ("S", 2, 4096, 1024, 0.25, 32),    # dense balls in grid mode: the hit buffer is compacted several times
    ("S", 2, 2048, 256, 0.3, 128),     # dense balls, nsample = the compaction limit
    ("S", 2, 2048, 64, 0.3, 200),      # nsample beyond it: a full buffer falls back to the ordered scan
    ("U", 2, 40, 64, 0.3, 8),          # npoint > n
    ("U", 3, 1, 4, 0.5, 3),            # single point
    ("D", 2, 5000, 1, 0.2, 5),         # one centroid
    ("U", 2, 3000, 257, 0.15, 1),      # nsample 1
    ("U", 40, 2048, 256, 0.12, 20),    # more clouds than fit two per SM pair
]


@pytest.mark.parametrize("center", [False, True])
@pytest.mark.parametrize("gen,b,n,m,r,s", LAYER_CASES)
def test_fused_layer_is_bit_identical_to_the_four_ops(dev, gen, b, n, m, r, s, center):
    x = T(W.DISTRIBUTIONS[gen](b, n, 51), dev)
    want = sequential(m, r, s, x, center)
    got = sample_group(m, r, s, x, center=center)
    for name, a, w in zip(("fps_idx", "new_xyz", "idx", "pts_cnt", "grouped_xyz"), got, want):
        assert torch.equal(a, w), f"{name} differs"


def test_fused_layer_matches_oracle_directly(dev):
    xyz = W.cloud_uniform(2, 2048, 52)
    fi, nx, idx, cnt, g = sample_group(256, 0.12, 16, T(xyz, dev), center=True)
    o_fi = O.oracle_fps(256, xyz)
    o_nx = O.oracle_gather_point(xyz, o_fi)
    o_idx, o_cnt = O.oracle_query_ball_point(0.12, 16, xyz, o_nx)
    np.testing.assert_array_equal(fi.cpu().numpy(), o_fi)
    np.testing.assert_array_equal(nx.cpu().numpy(), o_nx)
    np.testing.assert_array_equal(idx.cpu().numpy(), o_idx)
    np.testing.assert_array_equal(cnt.cpu().numpy(), o_cnt)
    np.testing.assert_array_equal(g.cpu().numpy(), O.oracle_group_point(xyz, o_idx) - o_nx[:, :, None, :])


def test_fused_layer_without_grouped_output(dev):
    x = T(W.cloud_uniform(3, 4096, 53), dev)
    fi, nx, idx, cnt, g = sample_group(512, 0.1, 32, x, want_grouped=False)
    assert g is None
    w = sequential(512, 0.1, 32, x, False)
    assert torch.equal(idx, w[2]) and torch.equal(cnt, w[3]) and torch.equal(nx, w[1])


def test_fused_layer_with_nan_and_inf_points(dev):
    """A NaN point is a hit in every ball (fmaxf semantics, tf_grouping_g.cu:24-25): the consumer must
    take the ordered scan for such a cloud.  FPS itself never picks across a NaN in these clouds'
    first picks identically in both paths (same kernel), so only the grouping half is at stake."""
    xyz = W.cloud_uniform(3, 3000, 54)
    xyz[0, 17] = np.nan
    xyz[1, 40, 2] = np.inf
    x = T(xyz, dev)
    want = sequential(200, 0.08, 16, x, False)
    got = sample_group(200, 0.08, 16, x, center=False)
    # new_xyz and grouped rows may hold NaN coordinates (FPS picks the NaN point): compare bit patterns
    for a, w in zip(got, want):
        assert torch.equal(a.view(torch.int32), w.view(torch.int32))


def test_fused_layer_repeated_launches_are_stable(dev):
    """The consumer polls indices the producer is still writing: 60 back-to-back layers (two
    alternating inputs, buffers reused) must all reproduce the sequential result."""
    xs = [T(W.cloud_uniform(8, 4096, 55 + i), dev) for i in range(2)]
    wants = [sequential(1024, 0.1, 32, x, False) for x in xs]
    for it in range(60):
        got = sample_group(1024, 0.1, 32, xs[it & 1], center=False)
        for a, w in zip(got, wants[it & 1]):
            assert torch.equal(a, w), f"iteration {it}"


def test_fused_layer_inside_a_cuda_graph(dev):
    x = T(W.cloud_uniform(8, 4096, 57), dev)
    want = sequential(1024, 0.1, 32, x, False)
    sa = SetAbstractionDevice(8, 4096, 1024, 0.1, 32, depth=1, center=False, device=dev)
    slot = sa.slots[0]
    st = torch.cuda.Stream(dev)
    st.wait_stream(torch.cuda.current_stream(dev))
    with torch.cuda.stream(st):
        sa.enqueue(slot, x, st)  # warm-up outside the capture (function attributes)
    st.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=st):
        sa.enqueue(slot, x, torch.cuda.current_stream(dev))
    for _ in range(5):
        for k in ("fps_idx", "new_xyz", "idx", "pts_cnt", "grouped"):
            slot[k].zero_()
        g.replay()
        torch.cuda.synchronize(dev)
        for k, w in zip(("fps_idx", "new_xyz", "idx", "pts_cnt", "grouped"), want):
            assert torch.equal(slot[k], w), k


def test_several_batches_in_flight(dev):
    xs = [T(W.cloud_uniform(16, 4096, 60 + i), dev) for i in range(5)]
    wants = [sequential(512, 0.1, 32, x, False) for x in xs]
    sa = SetAbstractionDevice(16, 4096, 512, 0.1, 32, depth=3, center=False, device=dev)
    out = []
    for x in xs:
        if sa.full():
            out.append([t.clone() for t in sa.collect(sync=True)])
        sa.submit(x)
    while sa.pending():
        out.append([t.clone() for t in sa.collect(sync=True)])
    assert len(out) == 5
    for got, want in zip(out, wants):
        for a, w in zip(got, want):
            assert torch.equal(a, w)


@pytest.mark.parametrize("gen,b,n,m,radii,nsamples", [("S", 32, 1024, 512, [0.1, 0.2, 0.4], [16, 32, 128]),   # cfg3 layer 1
                                                      ("S", 32, 512, 128, [0.2, 0.4, 0.8], [32, 64, 128]),    # cfg3 layer 2
                                                      ("U", 3, 4096, 300, [0.05, 0.3], [8, 40]),
                                                      ("D", 2, 16384, 256, [0.1, 0.2], [16, 32])])             # sequential fallback
@pytest.mark.parametrize("ctas", [0, 2])
def test_multi_scale_layer_is_bit_identical_to_the_separate_ops(dev, gen, b, n, m, radii, nsamples, ctas):
    x = T(W.DISTRIBUTIONS[gen](b, n, 59), dev)
    lib = _lib.load()
    lib.pn2_set_sa_consumer_ctas(ctas)
    try:
        fi, nx, idxs, cnts, grps = sample_group_msg(m, radii, nsamples, x, center=True)
    finally:
        lib.pn2_set_sa_consumer_ctas(0)
    wfi = farthest_point_sample(m, x)
    wnx = gather_point(x, wfi)
    assert torch.equal(fi, wfi) and torch.equal(nx, wnx)
    for r, s, idx, cnt, g in zip(radii, nsamples, idxs, cnts, grps):
        widx, wcnt = brute_force_query(r, s, x, wnx)
        assert torch.equal(idx, widx) and torch.equal(cnt, wcnt)
        assert torch.equal(g, group_point(x, widx) - wnx.unsqueeze(2))


@pytest.mark.parametrize("n,m", [(16384, 512), (12000, 128)])
def test_layer_falls_back_when_the_overlapped_path_does_not_apply(dev, n, m):
    """Clustered sampling (n > 8192) or a cloud beyond the shared-memory grid: same call, sequential
    kernels, same bits."""
    x = T(W.cloud_uniform(2, n, 58), dev)
    want = sequential(m, 0.05, 16, x, True)
    got = sample_group(m, 0.05, 16, x, center=True)
    for a, w in zip(got, want):
        assert torch.equal(a, w)


# ------------------------------------------------------------------------------------------- ball_group on its own
BG_CASES = [("U", 4, 4096, 1024, 0.1, 32), ("S", 2, 1024, 512, 0.2, 32), ("D", 2, 8192, 256, 0.2, 32), ("U", 32, 1024, 512, 0.1, 16),
            ("U", 1, 600, 1000, 0.3, 64), ("S", 3, 512, 128, 0.4, 64), ("U", 2, 100, 7, 0.2, 130)]


@pytest.mark.parametrize("center", [False, True])
@pytest.mark.parametrize("gen,b,n,m,r,s", BG_CASES)
def test_ball_group_matches_query_plus_group(dev, gen, b, n, m, r, s, center):
    xyz = W.DISTRIBUTIONS[gen](b, n, 61)
    x = T(xyz, dev)
    # queries: a mix of data points and free points, some outside the bounding box
    q = W.cloud_uniform(b, m, 62) * 1.4 - 0.2
    q[:, ::3] = xyz[:, np.arange(0, m, 3) % n]
    qt = T(q.astype(np.float32), dev)
    idx, cnt, g = ball_group(r, s, x, qt, center=center)
    widx, wcnt = brute_force_query(r, s, x, qt)
    wg = group_point(x, widx)
    if center:
        wg = wg - qt.unsqueeze(2)
    assert torch.equal(idx, widx) and torch.equal(cnt, wcnt) and torch.equal(g, wg)


def test_ball_group_nan_query_and_empty_rows(dev):
    xyz = W.cloud_uniform(2, 3000, 63)
    q = W.cloud_uniform(2, 64, 64)
    q[0, 5] = np.nan          # a NaN query hits every point: indices 0..nsample-1
    q[1, 7] = (9.0, 9.0, 9.0)  # far away: empty row -> zeros, pts_cnt 0
    q[1, 9, 0] = np.inf
    x, qt = T(xyz, dev), T(q, dev)
    idx, cnt, g = ball_group(0.07, 12, x, qt, center=False)
    oi, oc = O.oracle_query_ball_point(0.07, 12, xyz, q)
    np.testing.assert_array_equal(idx.cpu().numpy(), oi)
    np.testing.assert_array_equal(cnt.cpu().numpy(), oc)
    assert int(cnt[0, 5]) == 12 and idx[0, 5].tolist() == list(range(12))
    assert int(cnt[1, 7]) == 0 and not idx[1, 7].any()
    assert torch.equal(g, group_point(x, idx))


# ------------------------------------------------------------------------------------------- C-ABI robustness (ADVICE r1)
def test_fps_gather_and_host_layer_beyond_the_cluster_capacity(dev):
    """n > 16 * 512 * 52 = 425 984 takes the global-scratch kernel: pn2_fps_gather and pn2_sa_layer_host must
    serve it (round 1 passed temp = NULL and returned cudaErrorInvalidValue)."""
    lib = _lib.load()
    b, n, m = 2, 425984 + 300, 8
    xyz = W.cloud_uniform(b, n, 65)
    want = O.oracle_fps(m, xyz)
    x = T(xyz, dev)
    tb = int(lib.pn2_fps_scratch_bytes(b, n))
    assert tb == 4 * b * n
    temp = torch.empty(tb, dtype=torch.uint8, device=dev)
    fi = torch.empty((b, m), dtype=torch.int32, device=dev)
    nx = torch.empty((b, m, 3), dtype=torch.float32, device=dev)
    p = lambda t: ctypes.c_void_p(t.data_ptr())  # noqa: E731
    assert lib.pn2_fps_gather(b, n, m, p(x), None, p(fi), p(nx), None) == 1  # no scratch: refused, not a crash
    assert lib.pn2_fps_gather(b, n, m, p(x), p(temp), p(fi), p(nx), None) == 0
    torch.cuda.synchronize()
    np.testing.assert_array_equal(fi.cpu().numpy(), want)
    np.testing.assert_array_equal(nx.cpu().numpy(), O.oracle_gather_point(xyz, want))
    sess = SetAbstractionHost(b, n, m, 0.01, 4, device=dev)
    new_xyz, idx, cnt, grouped = sess.run(xyz)
    np.testing.assert_array_equal(new_xyz, O.oracle_gather_point(xyz, want))
    oi, oc = O.oracle_query_ball_point(0.01, 4, xyz, new_xyz)
    np.testing.assert_array_equal(idx, oi)
    np.testing.assert_array_equal(cnt, oc)


def test_fps_between_262144_and_425984_points_needs_no_scratch(dev):
    """Clouds beyond the 16 x 16 384 points of the all-in-shared-memory clusters are held in registers + shared
    memory (fps_cluster_big_kernel): no scratch, same picks as the CPU restatement."""
    lib = _lib.load()
    b, n, m = 2, 300001, 24
    assert int(lib.pn2_fps_scratch_bytes(b, n)) == 0
    xyz = np.concatenate([W.cloud_uniform(1, n, 67), W.cloud_duplicates(1, n, 68)])
    want = O.oracle_fps(m, xyz)
    fi, fx = farthest_point_sample_and_gather(m, T(xyz, dev))
    np.testing.assert_array_equal(fi.cpu().numpy(), want)
    np.testing.assert_array_equal(fx.cpu().numpy(), O.oracle_gather_point(xyz, want))


def test_host_layer_idx_only_mode(dev):
    xyz = W.cloud_uniform(4, 4096, 66)
    full = SetAbstractionHost(4, 4096, 512, 0.1, 32, device=dev).run(xyz)
    lean = SetAbstractionHost(4, 4096, 512, 0.1, 32, device=dev, want_grouped=False)
    new_xyz, idx, cnt, grouped = lean.run(xyz)
    assert grouped is None and lean.d2h_bytes < full[3].nbytes
    np.testing.assert_array_equal(idx, full[1])
    np.testing.assert_array_equal(new_xyz, full[0])
    np.testing.assert_array_equal(cnt, full[2])
