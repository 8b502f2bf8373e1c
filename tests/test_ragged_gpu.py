"""GPU tests of variable-size clouds (the `lengths` argument of FPS, the ball query and the set-abstraction layers).

Cloud i of a ragged batch must get, bit for bit, what the op computes on the truncated cloud xyz[i:i+1, :lengths[i]]
alone — checked against the C oracle for the raw ops and against the unragged call for the layers — and the padding
rows must be inert: every case runs twice, once with poisoned padding (NaN, +inf and a far point that FPS would pick
at once and every ball query would count) and once with padding that copies real points, and the two runs must agree
bit for bit."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import oracle as O
from pointnet2_b200 import _lib, workloads as W
from pointnet2_b200.nets import PointNet2ClsMSG, PointNet2ClsSSG
from pointnet2_b200.pointnet_util import sample_and_group
from pointnet2_b200.sa_layer import sample_group, sample_group_msg
from pointnet2_b200.tf_grouping import query_ball_point
from pointnet2_b200.tf_sampling import farthest_point_sample, farthest_point_sample_and_gather

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FAR = np.float32(50.0)


def lengths_for(n, npoint):
    """n, n-1, 1, 2, 3, 511, 513, a length that is not a multiple of 4, and one below npoint"""
    ls = [n, n - 1, 1, 2, 3, 511, 513, (n * 5) // 7 | 1, max(1, npoint // 2 - 1)]
    return [min(max(l, 1), n) for l in ls]


def pad(x, lengths, kind):
    """x (b, n, 3) with the rows of cloud i from lengths[i] on overwritten: 'poison' or 'copy'"""
    x = x.copy()
    for i, l in enumerate(lengths):
        rows = np.arange(l, x.shape[1])
        if kind == "poison":
            x[i, rows[0::3]] = np.nan
            x[i, rows[1::3]] = np.inf
            x[i, rows[2::3]] = (FAR, -FAR, FAR)
        else:
            x[i, rows] = x[i, rows % l]
    return x


def T(a, dev):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


def both_paddings(fn, x, lengths, dev):
    """fn(padded batch on the device) for both paddings; the two results must be bit-identical"""
    outs = [fn(T(pad(x, lengths, kind), dev)) for kind in ("poison", "copy")]
    for a, b in zip(outs[0], outs[1]):
        assert torch.equal(a, b) if a.dtype != torch.float32 else torch.equal(a.view(torch.int32), b.view(torch.int32)), \
            "padding changed the result"
    return outs[0]


# ------------------------------------------------------------------------------------------------------------ FPS
FPS_PLANS = [
    # (threads, points per thread, cluster), n, npoint — every kernel family through pn2_set_fps_config
    ((256, 16, -1), 4096, 600),      # one CTA, plain chain
    ((256, 16, -2), 4096, 600),      # one CTA, packed chain
    ((128, 8, -2), 1024, 300),       # one CTA, packed chain, fewer points per thread
    ((256, 4, -1), 1000, 200),       # one CTA, plain chain, n not a multiple of the CTA
    ((128 + 1, 8, 4), 4096, 500),    # cluster, packed
    ((128 + 2, 8, 4), 4096, 500),    # cluster, plain
    ((512 + 1, 32, 2), 20000, 300),  # cluster, register + streamed shared-memory points (PR < P), packed
    ((512 + 2, 32, 2), 20000, 300),  # the same, plain
    ((512 + 1, 44, 3), 60000, 200),  # the register + shared-memory kernel at a non-power-of-two cluster size, packed
    ((512 + 2, 44, 3), 60000, 200),  # the same, plain
    ((1024, 1, 0), 3000, 300),       # global-scratch path
]


@pytest.mark.parametrize("plan,n,npoint", FPS_PLANS)
def test_fps_ragged_equals_each_truncated_cloud(dev, plan, n, npoint):
    lengths = lengths_for(n, npoint)
    x = W.cloud_uniform(len(lengths), n, 7)
    lib = _lib.load()
    try:
        lib.pn2_set_fps_config(*plan)
        idx, nx = both_paddings(lambda t: farthest_point_sample_and_gather(npoint, t, lengths=lengths), x, lengths, dev)
        idx_only = farthest_point_sample(npoint, T(pad(x, lengths, "poison"), dev), lengths=lengths)
    finally:
        lib.pn2_set_fps_config(0, 0, 0)
    assert torch.equal(idx, idx_only)
    idx, nx = idx.cpu().numpy(), nx.cpu().numpy()
    for i, l in enumerate(lengths):
        cloud = x[i:i + 1, :l]
        o = O.oracle_fps(npoint, cloud)
        np.testing.assert_array_equal(idx[i:i + 1], o, err_msg=f"cloud {i}, length {l}")
        np.testing.assert_array_equal(nx[i:i + 1], O.oracle_gather_point(cloud, o), err_msg=f"cloud {i}, length {l}")


def test_fps_ragged_at_full_capacity_with_ties_across_ctas(dev):
    n, npoint = 262144, 160
    lengths = [262144, 262143, 131073, 70001]
    x = W.cloud_duplicates(len(lengths), n, 11)
    idx, nx = both_paddings(lambda t: farthest_point_sample_and_gather(npoint, t, lengths=lengths), x, lengths, dev)
    idx = idx.cpu().numpy()
    for i, l in enumerate(lengths):
        np.testing.assert_array_equal(idx[i:i + 1], O.oracle_fps(npoint, x[i:i + 1, :l]), err_msg=f"length {l}")


# ----------------------------------------------------------------------------------------------------- ball query
BQ_CASES = [
    # n, npoint (queries), radius, nsample, extra lengths (in another path regime than n)
    (1024, 256, 0.15, 32, []),
    (4096, 512, 0.1, 32, [1000]),
    (16384, 512, 0.06, 32, [3000, 1000]),
]


@pytest.mark.parametrize("mode", [0, 1, 2])
@pytest.mark.parametrize("n,m,r,s,extra", BQ_CASES)
def test_ball_query_ragged_equals_each_truncated_cloud(dev, n, m, r, s, extra, mode):
    lengths = lengths_for(n, m) + extra
    b = len(lengths)
    x = W.cloud_uniform(b, n, 21)
    q = W.cloud_uniform(b, m, 22)
    q[:, : m // 2] = x[:, : m // 2]  # half the queries sit on data points (those of short clouds also on padding rows)
    qd = T(q, dev)
    lib = _lib.load()
    try:
        lib.pn2_set_bq_mode(mode)
        idx, cnt = both_paddings(lambda t: query_ball_point(r, s, t, qd, lengths=lengths), x, lengths, dev)
    finally:
        lib.pn2_set_bq_mode(0)
    idx, cnt = idx.cpu().numpy(), cnt.cpu().numpy()
    for i, l in enumerate(lengths):
        o_idx, o_cnt = O.oracle_query_ball_point(r, s, x[i:i + 1, :l], q[i:i + 1])
        np.testing.assert_array_equal(cnt[i:i + 1], o_cnt, err_msg=f"cloud {i}, length {l}")
        np.testing.assert_array_equal(idx[i:i + 1], o_idx, err_msg=f"cloud {i}, length {l}")


# --------------------------------------------------------------------------------------------------------- layers
def dense_per_cloud(fn, x, lengths, dev):
    """fn on each truncated cloud alone, results concatenated over the batch"""
    parts = [fn(T(x[i:i + 1, :l], dev)) for i, l in enumerate(lengths)]
    return [torch.cat([p[k] for p in parts]) for k in range(len(parts[0]))]


LAYER_CASES = [
    # n, npoint: 4096 takes the overlapped path (one sampling CTA per cloud + the consumer grid), 16384 the sequential one
    (4096, 1024),
    (16384, 512),
]


@pytest.mark.parametrize("center", [False, True])
@pytest.mark.parametrize("n,m", LAYER_CASES)
def test_sample_group_ragged_equals_each_truncated_cloud(dev, n, m, center):
    lengths = lengths_for(n, m)
    x = W.cloud_surface(len(lengths), n, 31)
    got = both_paddings(lambda t: sample_group(m, 0.1, 32, t, center=center, lengths=lengths), x, lengths, dev)
    want = dense_per_cloud(lambda t: sample_group(m, 0.1, 32, t, center=center), x, lengths, dev)
    for name, a, w in zip(("fps_idx", "new_xyz", "idx", "pts_cnt", "grouped_xyz"), got, want):
        assert torch.equal(a, w), name


@pytest.mark.parametrize("center", [False, True])
@pytest.mark.parametrize("n,m", LAYER_CASES)
def test_sample_group_msg_ragged_equals_each_truncated_cloud(dev, n, m, center):
    lengths = lengths_for(n, m)
    x = W.cloud_uniform(len(lengths), n, 32)
    radii, nsamples = [0.05, 0.1, 0.2], [16, 32, 64]

    def flat(out):
        fi, nx, idx, cnt, g = out
        return [fi, nx] + list(idx) + list(cnt) + list(g)

    got = both_paddings(lambda t: flat(sample_group_msg(m, radii, nsamples, t, center=center, lengths=lengths)), x, lengths, dev)
    want = dense_per_cloud(lambda t: flat(sample_group_msg(m, radii, nsamples, t, center=center)), x, lengths, dev)
    for k, (a, w) in enumerate(zip(got, want)):
        assert torch.equal(a, w), k


@pytest.mark.parametrize("n,m", [(4096, 1024), (16384, 256)])
def test_sample_and_group_fused_and_unfused_agree(dev, n, m):
    lengths = lengths_for(n, m)
    x = T(pad(W.cloud_uniform(len(lengths), n, 41), lengths, "poison"), dev)
    feats = T(W.features(len(lengths), n, 6, 42), dev)
    for points in (None, feats):
        a = sample_and_group(m, 0.1, 32, x, points, fused=True, lengths=lengths)
        b = sample_and_group(m, 0.1, 32, x, points, fused=False, lengths=lengths)
        for k, (u, v) in enumerate(zip(a, b)):
            assert torch.equal(u, v), k
        assert not torch.isnan(a[1]).any(), "a padding row reached the grouped output"


def test_sample_group_in_a_cuda_graph_follows_rewritten_lengths(dev):
    n, m = 4096, 512
    x = T(pad(W.cloud_uniform(6, n, 51), [n] * 6, "copy"), dev)
    lens = torch.tensor([n, 3000, 513, 1000, 7, 2049], dtype=torch.int32, device=dev)
    st = torch.cuda.Stream(dev)
    st.wait_stream(torch.cuda.current_stream(dev))
    with torch.cuda.stream(st):
        sample_group(m, 0.1, 32, x, lengths=lens)  # warm-up outside the capture
    st.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=st):
        out = sample_group(m, 0.1, 32, x, lengths=lens)
    for new in ([n, 3000, 513, 1000, 7, 2049], [5, 4096, 1111, 2, 4000, 600], [n] * 6):
        lens.copy_(torch.tensor(new, dtype=torch.int32))  # an in-place write; the graph is not re-captured
        g.replay()
        torch.cuda.synchronize(dev)
        want = sample_group(m, 0.1, 32, x, lengths=new)
        for k, (a, w) in enumerate(zip(out, want)):
            assert torch.equal(a, w), (new, k)


# ------------------------------------------------------------------------------------------------ lengths handling
def test_host_lengths_are_validated(dev):
    x = T(W.cloud_uniform(3, 100, 61), dev)
    q = x[:, :10].contiguous()
    for bad in ([0, 5, 5], [5, 101, 5], [5, 5], [[5, 5, 5]], torch.tensor([5, -1, 5]), np.array([5, 5, 5, 5])):
        with pytest.raises(ValueError):
            farthest_point_sample(10, x, lengths=bad)
        with pytest.raises(ValueError):
            query_ball_point(0.2, 8, x, q, lengths=bad)
        with pytest.raises(ValueError):
            sample_group(10, 0.2, 8, x, lengths=bad)
    with pytest.raises(ValueError):
        farthest_point_sample(10, x, lengths=torch.tensor([5, 5], device=dev))  # wrong shape on the device too
    with pytest.raises(TypeError):
        farthest_point_sample(10, x, lengths=[1.5, 2.0, 3.0])


def test_device_lengths_out_of_range_are_clamped(dev):
    n, m = 2048, 256
    x = T(pad(W.cloud_uniform(4, n, 62), [n] * 4, "copy"), dev)
    for dtype in (torch.int32, torch.int64):
        dl = torch.tensor([0, -3, n + 5, 700], dtype=dtype, device=dev)
        got = sample_group(m, 0.1, 16, x, lengths=dl)
        want = sample_group(m, 0.1, 16, x, lengths=[1, 1, n, 700])
        for a, w in zip(got, want):
            assert torch.equal(a, w)
        assert torch.equal(farthest_point_sample(m, x, lengths=dl), farthest_point_sample(m, x, lengths=[1, 1, n, 700]))
        q = x[:, :m].contiguous()
        for a, w in zip(query_ball_point(0.1, 16, x, q, lengths=dl), query_ball_point(0.1, 16, x, q, lengths=[1, 1, n, 700])):
            assert torch.equal(a, w)


@pytest.mark.parametrize("n", [1024, 4096, 16384])
def test_full_lengths_equal_todays_outputs(dev, n):
    b, m = 3, 256
    x = T(W.cloud_uniform(b, n, 63), dev)
    q = x[:, :m].contiguous()
    for lengths in (None, [n] * b, torch.full((b,), n, dtype=torch.int32, device=dev)):
        for a, w in zip(sample_group(m, 0.1, 32, x, lengths=lengths), sample_group(m, 0.1, 32, x)):
            assert torch.equal(a, w)
        assert torch.equal(farthest_point_sample(m, x, lengths=lengths), farthest_point_sample(m, x))
        for a, w in zip(query_ball_point(0.1, 32, x, q, lengths=lengths), query_ball_point(0.1, 32, x, q)):
            assert torch.equal(a, w)


# ------------------------------------------------------------------------------------------------------------- nets
@pytest.mark.parametrize("net_cls", [PointNet2ClsSSG, PointNet2ClsMSG])
def test_net_logits_of_a_ragged_batch_match_each_cloud_alone(dev, net_cls):
    n = 1024
    lengths = [1024, 700, 513, 1000, 300]
    torch.manual_seed(0)
    net = net_cls(num_class=10).to(dev).eval()
    x = W.cloud_surface(len(lengths), n, 71)
    with torch.no_grad():
        got, _ = net(T(pad(x, lengths, "poison"), dev), lengths=lengths)
        for i, l in enumerate(lengths):
            alone, _ = net(T(x[i:i + 1, :l], dev))
            torch.testing.assert_close(got[i:i + 1], alone)  # the linear layers run at another batch size


def _train_child(name):
    """one training step on a ragged batch with each padding, in a fresh process with deterministic gradients;
    prints whether logits and parameter gradients agree bit for bit and are finite"""
    code = f"""
import sys, numpy as np, torch
sys.path.insert(0, {ROOT!r})
sys.path.insert(0, {os.path.join(ROOT, 'tests')!r})
from pointnet2_b200 import nets, workloads as W
from test_ragged_gpu import pad
torch.use_deterministic_algorithms(True)
dev = torch.device("cuda:0")
torch.manual_seed(0)
net = {{"cls_ssg": nets.PointNet2ClsSSG, "cls_msg": nets.PointNet2ClsMSG}}[{name!r}](num_class=10).to(dev).train()
lengths = [1024, 700, 513, 1000]
x = W.cloud_surface(len(lengths), 1024, 81)
res = []
for kind in ("poison", "copy"):
    net.zero_grad()
    torch.manual_seed(1)  # the same dropout masks for both paddings
    pred, _ = net(torch.from_numpy(pad(x, lengths, kind)).to(dev), lengths=torch.tensor(lengths, device=dev))
    pred.square().mean().backward()
    res.append([pred.detach().clone()] + [p.grad.detach().clone() for p in net.parameters()])
same = all(torch.equal(a, b) for a, b in zip(*res))
finite = all(bool(torch.isfinite(t).all()) for t in res[0])
print("same", same, "finite", finite)
"""
    env = dict(os.environ, CUBLAS_WORKSPACE_CONFIG=":4096:8")
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, env=env, cwd=ROOT, timeout=900)
    assert r.returncode == 0, r.stderr[-3000:]
    return r.stdout.strip().splitlines()[-1]


@pytest.mark.parametrize("name", ["cls_ssg", "cls_msg"])
def test_training_step_is_independent_of_the_padding(name):
    assert _train_child(name) == "same True finite True"
