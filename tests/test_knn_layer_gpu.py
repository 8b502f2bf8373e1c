"""GPU tests of the kNN set-abstraction layer (pn2_sa_knn_layer_device, sa_layer.sample_knn): every output must be
BIT-IDENTICAL to farthest_point_sample_and_gather, knn_point and group_point(xyz) [- new_xyz] run one after the other
(which test_parity_gpu.py pins to the oracle and the reference composite), on the overlapped path — the kNN
consumer grid polling the sampling kernel's picks — and on the sequential one."""
import numpy as np
import pytest
import torch

from oracle import oracle as O
from pointnet2_b200 import _lib, layers, workloads as W
from pointnet2_b200.pointnet_util import pointnet_sa_module, sample_and_group
from pointnet2_b200.sa_layer import sample_knn
from pointnet2_b200.tf_grouping import group_point, knn_point
from pointnet2_b200.tf_sampling import farthest_point_sample_and_gather

pytestmark = pytest.mark.gpu


def T(a, dev):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


def cloud(gen, b, n, seed):
    if gen == "G":  # a coarse lattice: exact ties in almost every distance (the replay path)
        return (np.random.RandomState(seed).randint(0, 6, (b, n, 3)) * 0.125).astype(np.float32)
    return W.DISTRIBUTIONS[gen](b, n, seed)


def sequential(npoint, k, x, center):
    fi, nx = farthest_point_sample_and_gather(npoint, x)
    val, idx = knn_point(k, x, nx)
    g = group_point(x, idx)
    if center:
        g = g - nx.unsqueeze(2)
    return fi, nx, idx, val, g


def assert_same_bits(got, want, want_dist=True, want_grouped=True):
    names = ("fps_idx", "new_xyz", "idx", "dist", "grouped_xyz")
    for name, a, w in zip(names, got, want):
        if (name == "dist" and not want_dist) or (name == "grouped_xyz" and not want_grouped):
            assert a is None, name
            continue
        assert a.shape == w.shape, name
        assert torch.equal(a.view(torch.int32), w.view(torch.int32)), f"{name} differs"


CASES = [
    # gen, b, n, npoint, k
    ("U", 4, 4096, 1024, 32),    # cfg2's shape, fewer clouds
    ("D", 3, 4096, 512, 32),     # duplicate-heavy: ties
    ("G", 2, 2048, 512, 33),     # lattice: the exact replay nearly everywhere
    ("U", 2, 1024, 512, 1),
    ("S", 2, 1024, 256, 8),
    ("S", 2, 1024, 256, 64),
    ("D", 2, 1024, 256, 65),
    ("G", 2, 1024, 256, 128),
    ("U", 2, 128, 300, 128),     # k = n, npoint > n
    ("D", 2, 100, 64, 100),      # k = n
    ("U", 1, 8192, 1024, 32),    # b = 1, the largest single-CTA sampling
    ("U", 32, 1024, 512, 32),    # b = 32
    ("U", 140, 256, 64, 16),     # more clouds than SMs: sequential by the rule
    ("U", 70, 512, 128, 8),      # more than SMs / 2: sequential by the rule
    ("U", 2, 16384, 256, 32),    # clustered sampling: sequential
    ("U", 2, 20000, 128, 8),     # beyond pn2_sa_knn_layer_fits: sequential
    ("U", 16, 1024, 512, 128),   # k > 64: sequential
    ("U", 40, 1024, 256, 32),    # 2 consumer CTAs per cloud: sequential by the cost rule
]
OUTPUTS = [(True, True), (False, False), (True, False)]  # (want_grouped, want_dist)


@pytest.mark.parametrize("want", OUTPUTS)
@pytest.mark.parametrize("center", [False, True])
@pytest.mark.parametrize("gen,b,n,m,k", CASES)
def test_sample_knn_is_bit_identical_to_the_op_sequence(dev, gen, b, n, m, k, center, want):
    want_grouped, want_dist = want
    x = T(cloud(gen, b, n, 71), dev)
    got = sample_knn(m, k, x, center=center, want_grouped=want_grouped, want_dist=want_dist)
    assert_same_bits(got, sequential(m, k, x, center), want_dist, want_grouped)


def test_the_sequential_cases_are_beyond_the_overlapped_layer():
    lib = _lib.load()
    assert lib.pn2_sa_knn_layer_fits(20000, 8) == 0
    assert lib.pn2_sa_knn_layer_fits(4096, 64) == 1
    assert lib.pn2_sa_knn_layer_fits(4096, 128) == 0  # k > 64: sequential


@pytest.mark.parametrize("k", [1, 8, 32, 33, 64, 65, 128])
@pytest.mark.parametrize("gen", ["U", "D", "G"])
def test_every_kc_instance_on_each_cloud_kind(dev, gen, k):
    x = T(cloud(gen, 6, 2048, 72), dev)
    assert_same_bits(sample_knn(700, k, x, want_dist=True), sequential(700, k, x, True))


def test_clouds_with_nan_and_inf_rows(dev):
    xyz = W.cloud_uniform(4, 3000, 73)
    xyz[0, 17] = np.nan
    xyz[1, 40:44, 2] = np.nan
    xyz[2, 5] = np.inf
    xyz[3, 0, 0] = -np.inf
    xyz[3, 2999] = np.nan
    x = T(xyz, dev)
    for k in (8, 40, 128):
        for center in (False, True):
            assert_same_bits(sample_knn(300, k, x, center=center, want_dist=True), sequential(300, k, x, center))


def launches_of(fn):
    before = _lib.launch_count()
    out = fn()
    torch.cuda.synchronize()
    return out, _lib.launch_count() - before


@pytest.fixture
def knn_path():
    """pn2_set_sa_knn_path for one test, reset to the rule afterwards."""
    lib = _lib.load()
    yield lib.pn2_set_sa_knn_path
    lib.pn2_set_sa_knn_path(0)


@pytest.mark.parametrize("gen,b,n,m,k", [("U", 2, 48, 100, 48),    # m > n, k = n: offer() has nothing, B stays empty
                                         ("D", 2, 64, 64, 64),     # k = n
                                         ("G", 3, 33, 70, 33),     # k = n > 32, m > n
                                         ("U", 40, 4096, 1024, 32),  # 2 consumer CTAs per cloud
                                         ("D", 64, 2048, 512, 16),   # 1 consumer CTA per cloud
                                         ("U", 3, 2048, 64, 1)])
@pytest.mark.parametrize("mode,launches", [(1, 2), (2, 3)])  # overlapped: sampling + consumer; sequential: + knn + group
def test_each_path_forced(dev, knn_path, gen, b, n, m, k, mode, launches):
    """Both paths on shapes the rule would not send there, with the path checked by the launches it makes."""
    x = T(cloud(gen, b, n, 90), dev)
    want = sequential(m, k, x, True)
    knn_path(mode)
    got, count = launches_of(lambda: sample_knn(m, k, x, center=True, want_dist=True))
    assert count == launches
    assert_same_bits(got, want)


@pytest.mark.parametrize("gen,b,n,m,k,overlapped", [("U", 32, 4096, 1024, 32, True), ("U", 33, 4096, 1024, 32, True),
                                                    ("U", 34, 4096, 1024, 32, False), ("U", 26, 4096, 1024, 64, True),
                                                    ("U", 27, 4096, 1024, 64, False), ("U", 16, 1024, 512, 32, True),
                                                    ("U", 16, 1024, 512, 64, False), ("U", 44, 4096, 1024, 8, True),
                                                    ("U", 8, 8192, 1024, 32, True), ("U", 16, 1024, 512, 128, False)])
def test_the_rule_picks_the_path(dev, gen, b, n, m, k, overlapped):
    """The cost rule of DESIGN.md §6.2.1 on a 132-SM H100 (other SM counts move its boundary)."""
    if torch.cuda.get_device_properties(dev).multi_processor_count != 132:
        pytest.skip("the boundary below is the one for 132 SMs")
    x = T(cloud(gen, b, n, 91), dev)
    got, count = launches_of(lambda: sample_knn(m, k, x, center=True))
    assert count == (2 if overlapped else 3)
    assert (_lib.load().pn2_sa_knn_layer_workspace_bytes(b, n, m, k) == 0) == overlapped
    assert_same_bits(got, sequential(m, k, x, True), want_dist=False)


@pytest.mark.parametrize("ctas", [1, 1000])  # forced to one, and to every SM the sampling leaves (the override is clamped)
@pytest.mark.parametrize("gen,b,n,m,k", [("U", 32, 4096, 1024, 32), ("D", 16, 1024, 512, 64), ("G", 8, 8192, 1024, 64),
                                         ("U", 3, 2048, 64, 16)])
def test_forced_consumer_ctas(dev, knn_path, gen, b, n, m, k, ctas):
    x = T(cloud(gen, b, n, 74), dev)
    lib = _lib.load()
    knn_path(1)  # with one consumer CTA per cloud the rule would pick the sequential path
    lib.pn2_set_sa_consumer_ctas(ctas)
    try:
        got, count = launches_of(lambda: sample_knn(m, k, x, center=True, want_dist=True))
    finally:
        lib.pn2_set_sa_consumer_ctas(0)
    assert count == 2
    assert_same_bits(got, sequential(m, k, x, True))


def test_repeated_launches_are_stable(dev):
    """The consumer polls indices the producer is still writing: 40 back-to-back layers (two alternating inputs,
    fresh outputs) must all reproduce the sequential result."""
    xs = [T(W.cloud_uniform(16, 4096, 75 + i), dev) for i in range(2)]
    wants = [sequential(1024, 32, x, True) for x in xs]
    for it in range(40):
        assert_same_bits(sample_knn(1024, 32, xs[it & 1], want_dist=True), wants[it & 1])


@pytest.mark.parametrize("k", [16, 100])
def test_matches_the_oracle_directly(dev, k):
    xyz = W.cloud_duplicates(2, 700, 76)
    fi, nx, idx, dist, g = sample_knn(96, k, T(xyz, dev), center=True, want_dist=True)
    o_fi = O.oracle_fps(96, xyz)
    o_nx = O.oracle_gather_point(xyz, o_fi)
    o_val, o_idx = O.oracle_knn_point(k, xyz, o_nx)
    np.testing.assert_array_equal(fi.cpu().numpy(), o_fi)
    np.testing.assert_array_equal(nx.cpu().numpy(), o_nx)
    np.testing.assert_array_equal(idx.cpu().numpy(), o_idx)
    np.testing.assert_array_equal(dist.cpu().numpy(), o_val)
    np.testing.assert_array_equal(g.cpu().numpy(), O.oracle_group_point(xyz, o_idx) - o_nx[:, :, None, :])


def test_cuda_graph_replay_with_new_coordinates(dev):
    b, n, m, k = 8, 4096, 1024, 32
    x = T(W.cloud_uniform(b, n, 77), dev)
    st = torch.cuda.Stream(dev)
    st.wait_stream(torch.cuda.current_stream(dev))
    with torch.cuda.stream(st):
        sample_knn(m, k, x, want_dist=True)  # first call on the device: function attributes, outside the capture
    st.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=st):
        out = sample_knn(m, k, x, want_dist=True)
    for seed in (78, 79, 80):
        x.copy_(T(cloud("G" if seed == 79 else "U", b, n, seed), dev))
        for t in out:
            t.zero_()
        g.replay()
        torch.cuda.synchronize(dev)
        assert_same_bits(out, sequential(m, k, x, True))


# ------------------------------------------------------------------------------------------- the layer glue
@pytest.mark.parametrize("c,use_xyz", [(0, True), (6, True), (6, False)])
def test_sample_and_group_knn_fused_equals_unfused(dev, c, use_xyz):
    x = T(W.cloud_surface(4, 2048, 81), dev)
    p = T(W.features(4, 2048, c, 82), dev) if c else None
    got = sample_and_group(512, 0.2, 32, x, p, knn=True, use_xyz=use_xyz, fused=True)
    want = sample_and_group(512, 0.2, 32, x, p, knn=True, use_xyz=use_xyz, fused=False)
    for a, w in zip(got, want):
        assert torch.equal(a.view(torch.int32), w.view(torch.int32))


def test_sa_module_knn_training_fused_equals_unfused(dev):
    torch.manual_seed(83)
    x = T(W.cloud_uniform(4, 2048, 84), dev)
    p = T(W.features(4, 2048, 9, 85), dev)
    mlp = layers.SharedMLP(12, [32, 64]).to(dev).train()
    outs, grads = [], []
    for fused in (True, False):
        mlp.zero_grad()
        pp = p.clone().requires_grad_(True)
        nx, feats, idx = pointnet_sa_module(x, pp, 256, 0.2, 32, mlp=mlp, knn=True, fused=fused)
        feats.square().sum().backward()
        outs.append((nx, feats.detach(), idx))
        grads.append([q.grad.clone() for q in mlp.parameters()])
    for a, w in zip(*outs):
        assert torch.equal(a, w)
    for a, w in zip(*grads):
        assert torch.equal(a, w)


def test_sa_module_knn_eval_under_no_grad(dev):
    """Eval under no_grad runs the fused inference tail (layers.sa_mlp_max) on the layer's idx: it must see what the
    op sequence gives it."""
    torch.manual_seed(86)
    x = T(W.cloud_uniform(4, 2048, 87), dev)
    p = T(W.features(4, 2048, 9, 88), dev)
    mlp = layers.SharedMLP(12, [32, 64]).to(dev).eval()
    with torch.no_grad():
        nx, feats, idx = pointnet_sa_module(x, p, 256, 0.2, 32, mlp=mlp, knn=True)
        _, wnx = farthest_point_sample_and_gather(256, x)
        _, widx = knn_point(32, x, wnx)
        want = layers.sa_mlp_max(x, wnx, p, widx, mlp, True, True)
        unfused = pointnet_sa_module(x, p, 256, 0.2, 32, mlp=mlp, knn=True, fused=False)
    assert torch.equal(nx, wnx) and torch.equal(idx, widx) and torch.equal(feats, want)
    assert torch.equal(nx, unfused[0]) and torch.equal(idx, unfused[2])
