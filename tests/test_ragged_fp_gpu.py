"""GPU tests of variable-size clouds in feature propagation (the `lengths` of the unknown side of three_nn, the FP front
end and three_interpolate with its gradients) and in the segmentation net.

Every real row must be bit for bit what the op computes without lengths (checked against the C oracle on the truncated
clouds where the op has one), padding rows must hold the documented filler, and the padding must be inert: every case
runs once with poisoned padding (NaN, +inf, a far point) and once with padding that copies real rows, and the two runs
must agree bit for bit."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import numerics as NUM
from oracle import oracle as O
from pointnet2_b200 import _lib, tf_interpolate, workloads as W
from pointnet2_b200.layers import SharedMLP, row_mask
from pointnet2_b200.nets import PointNet2SemSeg, sem_seg_loss
from pointnet2_b200.pointnet_util import pointnet_fp_module
from pointnet2_b200.tf_interpolate import fp_interpolate_concat, three_interpolate, three_nn, three_nn_interpolate

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FAR = np.float32(50.0)
FMT = {torch.float32: "f32", torch.bfloat16: "bf16", torch.float16: "f16"}


def pad(x, lengths, kind):
    """x (b, n, c) with the rows of cloud i from lengths[i] on overwritten: 'poison' or 'copy'"""
    x = x.copy()
    for i, l in enumerate(lengths):
        rows = np.arange(l, x.shape[1])
        if kind == "poison":
            x[i, rows[0::3]] = np.nan
            x[i, rows[1::3]] = np.inf
            x[i, rows[2::3]] = FAR
        else:
            x[i, rows] = x[i, rows % l]
    return x


def T(a, dev):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


def bits(t):
    return t.view(torch.int16) if t.element_size() == 2 else t.view(torch.int32) if t.is_floating_point() else t


def both_paddings(fn, arrays, lengths, dev):
    """fn(*padded arrays on the device) for both paddings; the two results must be bit-identical"""
    outs = []
    for kind in ("poison", "copy"):
        outs.append(fn(*[T(pad(a, lengths, kind), dev) for a in arrays]))
    for a, b in zip(outs[0], outs[1]):
        assert torch.equal(bits(a), bits(b)), "padding changed the result"
    return outs[0]


def real(lengths, n, dev):
    return row_mask(torch.tensor(lengths, dtype=torch.int32, device=dev), n)


def assert_filler(t, mask, value):
    pad_rows = t[~mask]
    assert torch.equal(pad_rows, torch.full_like(pad_rows, value)), "padding rows must hold the filler"


# -------------------------------------------------------------------------------------------------------- three_nn
def test_three_nn_real_rows_equal_the_oracle_on_each_truncated_cloud(dev):
    n, m = 8192, 1024
    lengths = [n, n - 1, 1, 127, 129, 255, 257, 4095, 4097, 3001]
    x1 = W.cloud_uniform(len(lengths), n, 1)
    x2 = W.cloud_uniform(len(lengths), m, 2)
    x2d = T(x2, dev)
    dist, idx = both_paddings(lambda a: three_nn(a, x2d, lengths=lengths), [x1], lengths, dev)
    mask = real(lengths, n, dev)
    assert_filler(dist, mask, float("inf"))
    assert_filler(idx, mask, 0)
    dist, idx = dist.cpu().numpy(), idx.cpu().numpy()
    for i, l in enumerate(lengths):
        od, oi = O.oracle_three_nn(x1[i:i + 1, :l], x2[i:i + 1])
        np.testing.assert_array_equal(idx[i:i + 1, :l], oi, err_msg=f"length {l}")
        np.testing.assert_array_equal(dist[i:i + 1, :l].view(np.int32), od.view(np.int32), err_msg=f"length {l}")


def test_three_nn_with_fewer_than_three_known_points(dev):
    n, m, lengths = 300, 2, [300, 5, 129]
    x1, x2 = W.cloud_uniform(3, n, 3), W.cloud_uniform(3, m, 4)
    dist, idx = both_paddings(lambda a: three_nn(a, T(x2, dev), lengths=lengths), [x1], lengths, dev)
    want_d, want_i = three_nn(T(pad(x1, lengths, "copy"), dev), T(x2, dev))
    mask = real(lengths, n, dev)
    assert torch.equal(bits(dist[mask]), bits(want_d[mask])) and torch.equal(idx[mask], want_i[mask])
    assert_filler(dist, mask, float("inf"))


# ---------------------------------------------------------------------------------------------- fused front end
# (n, m) with b = 9 clouds: lanes per point G = 1 from b*n alone (n 8192); G = 2, 4, 8, 16, 32 from small batches whose
# known set caps G (2G <= (m+1)/2: m = 3, 7, 15, 31, 63), and 32 again from m = 127
FRONT_SHAPES = [(8192, 1024), (2000, 3), (200, 7), (200, 15), (200, 31), (200, 63), (200, 127)]


def front_lengths(n):
    ls = [n, n - 1, 1, 2, 33, 65, 127, 129, (n * 5) // 7 | 1]
    return [min(max(l, 1), n) for l in ls]


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.float16])
@pytest.mark.parametrize("n,m", FRONT_SHAPES)
def test_fp_front_end_real_rows_equal_the_dense_call(dev, n, m, dtype):
    lengths = front_lengths(n)
    b = len(lengths)
    x1, x2 = W.cloud_surface(b, n, 11), W.cloud_uniform(b, m, 12)
    x2d = T(x2, dev)
    mask = real(lengths, n, dev)
    for c2, c1 in ((16, 8), (5, 3)):  # vector and scalar phase 2
        p2 = T(W.features(b, m, c2, 13), dev).to(dtype)
        p1 = W.features(b, n, c1, 14)
        # dense reference: the call without lengths on the copied padding (every row computed from its own point)
        x1c, p1c = T(pad(x1, lengths, "copy"), dev), T(pad(p1, lengths, "copy"), dev).to(dtype)
        want_cat = fp_interpolate_concat(x1c, x2d, p1c, p2)
        want_out, want_d, want_i, want_w = three_nn_interpolate(x1c, x2d, p2, return_aux=True)

        got_cat = both_paddings(lambda a, q: [fp_interpolate_concat(a, x2d, q.to(dtype), p2, lengths=lengths)], [x1, p1], lengths, dev)[0]
        assert torch.equal(bits(got_cat[mask]), bits(want_cat[mask])), (c2, c1)
        assert_filler(got_cat, mask, 0)
        got_nop1 = both_paddings(lambda a: [fp_interpolate_concat(a, x2d, None, p2, lengths=lengths)], [x1], lengths, dev)[0]
        assert torch.equal(bits(got_nop1[mask]), bits(want_cat[..., :c2][mask]))
        assert_filler(got_nop1, mask, 0)
        out, d, i, w = both_paddings(lambda a: three_nn_interpolate(a, x2d, p2, return_aux=True, lengths=lengths), [x1], lengths, dev)
        for g, wnt in ((out, want_out), (d, want_d), (i, want_i), (w, want_w)):
            assert torch.equal(bits(g[mask]), bits(wnt[mask]))
        assert_filler(out, mask, 0)
        assert_filler(d, mask, float("inf"))
        assert_filler(i, mask, 0)
        assert_filler(w, mask, 0)


# ------------------------------------------------------------------------------------------------ three_interpolate
def interp_inputs(b, n, m, lengths, seed, dev):
    """idx / weight of the unknown rows as the FP layer makes them (copied padding), on the device and as numpy"""
    x1, x2 = W.cloud_uniform(b, n, seed), W.cloud_uniform(b, m, seed + 1)
    _, d, i, w = three_nn_interpolate(T(pad(x1, lengths, "copy"), dev), T(x2, dev), T(np.zeros((b, m, 4), np.float32), dev),
                                      return_aux=True)
    return i.cpu().numpy(), w.cpu().numpy()


def poison_rows(idx, weight, lengths, kind, m):
    """padding rows of idx / weight: 'poison' (in-range index m - 1, NaN weights) or 'copy'"""
    idx, weight = idx.copy(), weight.copy()
    for k, l in enumerate(lengths):
        if kind == "poison":
            idx[k, l:] = m - 1
            weight[k, l:] = np.nan
        else:
            idx[k, l:] = idx[k, np.arange(l, idx.shape[1]) % l]
            weight[k, l:] = weight[k, np.arange(l, idx.shape[1]) % l]
    return idx, weight


# (b, n, m, c, lengths): short lists; lists > 256 entries (m = 4: inv_long_kernel); m > 16000 (count / scan / fill)
GRAD_CASES = [
    (4, 8192, 1024, 128, [8192, 4097, 1, 6000]),
    (3, 2000, 4, 12, [2000, 1999, 700]),
    (3, 4096, 20000, 8, [4096, 129, 3000]),
    (3, 1000, 256, 5, [1000, 1, 777]),
]


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.float16])
@pytest.mark.parametrize("b,n,m,c,lengths", GRAD_CASES)
def test_three_interpolate_and_its_deterministic_gradient(dev, b, n, m, c, lengths, dtype):
    idx, weight = interp_inputs(b, n, m, lengths, 21, dev)
    pts = W.features(b, m, c, 22)
    gout = W.features(b, n, c, 23)
    mask = real(lengths, n, dev)
    res = []
    for kind in ("poison", "copy"):
        ii, ww = poison_rows(idx, weight, lengths, kind, m)
        p = T(pts, dev).to(dtype).requires_grad_(True)
        out = three_interpolate(p, T(ii, dev), T(ww, dev), lengths=lengths)
        out.backward(T(pad(gout, lengths, kind), dev).to(dtype))
        res.append((out.detach(), p.grad))
    for a, g in zip(*res):
        assert torch.equal(bits(a), bits(g)), "padding changed the result"
    out, grad = res[0]
    want = three_interpolate(T(pts, dev).to(dtype), T(idx, dev), T(weight, dev))
    assert torch.equal(bits(out[mask]), bits(want[mask]))
    assert_filler(out, mask, 0)
    # the gradient of the call on each truncated cloud, and the oracle's ordered sum of the upcast gradient, rounded
    # once: bit for bit on lists of up to 256 entries, within the float64 bound on longer ones (summed in 8 pieces)
    fmt = FMT[dtype]
    gq = NUM.quantize(gout, fmt)
    for k, l in enumerate(lengths):
        p = T(pts[k:k + 1], dev).to(dtype).requires_grad_(True)
        three_interpolate(p, T(idx[k:k + 1, :l], dev), T(weight[k:k + 1, :l], dev)).backward(T(gout[k:k + 1, :l], dev).to(dtype))
        assert torch.equal(bits(grad[k:k + 1]), bits(p.grad)), f"length {l}"
        o = O.oracle_three_interpolate_grad((1, m, c), idx[k:k + 1, :l], weight[k:k + 1, :l], gq[k:k + 1, :l])[0]
        terms = weight[k, :l].astype(np.float64).reshape(-1, 1) * np.repeat(gq[k, :l].astype(np.float64), 3, axis=0)
        ref, mass, count = NUM.scatter64(m, idx[k, :l], terms)
        got = grad[k].float().cpu().numpy()
        short = count <= 256
        assert (m < 16) == (not short.all()), "the cases with m < 16 are the ones with lists longer than 256 entries"
        want = NUM.quantize(o, fmt)
        np.testing.assert_array_equal(got[short].view(np.int32), want[short].view(np.int32), err_msg=f"length {l}")
        assert NUM.within_bound(got, ref, mass, np.maximum(count, 1)[:, None], fmt).all(), f"length {l}"


@pytest.mark.parametrize("b,n,m,c,lengths", [GRAD_CASES[0], GRAD_CASES[3]])
def test_three_interpolate_atomic_gradient(dev, monkeypatch, b, n, m, c, lengths):
    monkeypatch.setattr(tf_interpolate, "DETERMINISTIC_GRAD", False)
    idx, weight = interp_inputs(b, n, m, lengths, 31, dev)
    pts, gout = W.features(b, m, c, 32), W.features(b, n, c, 33)
    ii, ww = poison_rows(idx, weight, lengths, "poison", m)
    p = T(pts, dev).requires_grad_(True)
    three_interpolate(p, T(ii, dev), T(ww, dev), lengths=lengths).backward(T(pad(gout, lengths, "poison"), dev))
    got = p.grad.cpu().numpy()
    for k, l in enumerate(lengths):  # float atomics: any order of the float32 sum, within the float64 bound
        terms = weight[k, :l].astype(np.float64).reshape(-1, 1) * np.repeat(gout[k, :l].astype(np.float64), 3, axis=0)
        ref, mass, count = NUM.scatter64(m, idx[k, :l], terms)
        assert NUM.within_bound(got[k], ref, mass, np.maximum(count, 1)[:, None], "f32").all(), f"length {l}"


def test_deterministic_gradient_of_full_lengths_equals_todays(dev):
    b, n, m, c = 3, 4096, 1024, 64
    lengths = [n] * b
    idx, weight = interp_inputs(b, n, m, lengths, 41, dev)
    pts, gout = T(W.features(b, m, c, 42), dev), T(W.features(b, n, c, 43), dev)
    grads = []
    for lg in (None, lengths):
        p = pts.clone().requires_grad_(True)
        out = three_interpolate(p, T(idx, dev), T(weight, dev), lengths=lg)
        out.backward(gout)
        grads += [out.detach(), p.grad]
    assert torch.equal(grads[0], grads[2]) and torch.equal(grads[1], grads[3])


# ------------------------------------------------------------------------------------------------ FP module routes
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_the_three_fp_module_routes_agree_on_every_real_row(dev, dtype):
    b, n, m, c2, c1 = 4, 4096, 1024, 32, 16
    lengths = [4096, 2049, 1, 3000]
    x1, x2 = W.cloud_surface(b, n, 51), T(W.cloud_uniform(b, m, 52), dev)
    p2 = T(W.features(b, m, c2, 53), dev).to(dtype)
    p1 = W.features(b, n, c1, 54)
    mask = real(lengths, n, dev)
    outs = []
    for route in ("fused", "three_nn_interpolate", "unfused"):
        def fn(a, q):
            q = q.to(dtype)
            if route == "three_nn_interpolate":
                q.requires_grad_(True)  # points1 needs a gradient: the fused concat is skipped
            return [pointnet_fp_module(a, x2, q, p2 if route != "unfused" else p2.detach().requires_grad_(True), None,
                                       fused=route != "unfused", lengths=lengths).detach()]
        outs.append(both_paddings(fn, [x1, p1], lengths, dev)[0])
    for o in outs:
        assert_filler(o, mask, 0)
    # the two kernel routes agree bit for bit
    assert torch.equal(bits(outs[1][mask]), bits(outs[0][mask]))
    # The unfused route computes the weights in torch, whose 3-term sum may take another order than the kernel's
    # (r1 + r2) + r3 (so it differs from the fused kernel in the last bits with or without lengths, as
    # test_fp_and_concat_gpu.py allows): its real rows equal the unfused call without lengths bit for bit, and the
    # kernels' within 1e-5 in float32, within one rounding of the output in bfloat16
    x1c, p1c = T(pad(x1, lengths, "copy"), dev), T(pad(p1, lengths, "copy"), dev).to(dtype)
    dense = pointnet_fp_module(x1c, x2, p1c, p2.detach().requires_grad_(True), None, fused=False).detach()
    assert torch.equal(bits(outs[2][mask]), bits(dense[mask]))
    tol = 1e-5 if dtype == torch.float32 else 2 ** -7
    torch.testing.assert_close(outs[2][mask].float(), outs[0][mask].float(), rtol=tol, atol=tol)
    # with a SharedMLP in training mode: the masked batch norm sees the same rows on both kernel routes
    torch.manual_seed(0)
    mlp = SharedMLP(c2 + c1, [32, 16]).to(dev)
    state = {k: v.clone() for k, v in mlp.state_dict().items()}
    res = []
    for route in ("fused", "three_nn_interpolate"):
        mlp.load_state_dict(state)
        q = T(pad(p1, lengths, "poison"), dev).to(dtype).requires_grad_(route != "fused")
        with torch.autocast("cuda", dtype=torch.bfloat16, enabled=dtype != torch.float32):
            res.append(pointnet_fp_module(T(pad(x1, lengths, "poison"), dev), x2, q, p2, mlp, lengths=lengths).detach())
    assert torch.equal(bits(res[0]), bits(res[1]))
    assert_filler(res[0], mask, 0)


# ------------------------------------------------------------------------------------------------------------- net
def test_sem_seg_eval_logits_match_each_cloud_alone(dev):
    n = 2048
    lengths = [2048, 1500, 1100, 700]
    torch.manual_seed(0)
    net = PointNet2SemSeg(num_class=13).to(dev).eval()
    x = W.cloud_surface(len(lengths), n, 61)
    mask = real(lengths, n, dev)
    with torch.no_grad():
        got = both_paddings(lambda a: [net(a, lengths=lengths)[0]], [x], lengths, dev)[0]
        assert_filler(got, mask, 0)
        for i, l in enumerate(lengths):
            alone, _ = net(T(x[i:i + 1, :l], dev))
            # The geometry underneath is bit-exact (the raw-op tests above); the linear layers run cuBLAS at another row
            # count (b*N rows against l), which may pick another kernel and round differently in the last bits, and
            # eleven layers carry that on.  Hence a float32 tolerance a few hundred ulps wide, not bit equality.
            torch.testing.assert_close(got[i:i + 1, :l], alone, rtol=1e-4, atol=1e-4)


def test_sem_seg_ragged_forward_in_a_cuda_graph_follows_rewritten_lengths(dev):
    n = 2048
    torch.manual_seed(0)
    net = PointNet2SemSeg(num_class=13).to(dev).eval()
    x = T(pad(W.cloud_surface(4, n, 62), [n] * 4, "copy"), dev)
    lens = torch.tensor([n, 1500, 700, 1100], dtype=torch.int32, device=dev)
    st = torch.cuda.Stream(dev)
    st.wait_stream(torch.cuda.current_stream(dev))
    with torch.no_grad():
        with torch.cuda.stream(st):
            net(x, lengths=lens)  # warm-up outside the capture
        st.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=st):
            out, _ = net(x, lengths=lens)
        for new in ([n, 1500, 700, 1100], [5, 2048, 1111, 2000], [n] * 4):
            lens.copy_(torch.tensor(new, dtype=torch.int32))  # an in-place write; the graph is not re-captured
            g.replay()
            torch.cuda.synchronize(dev)
            want, _ = net(x, lengths=new)
            torch.testing.assert_close(out, want, rtol=1e-5, atol=1e-5)
            assert_filler(out, real(new, n, dev), 0)


def _train_child():
    """ragged training steps of the sem-seg net in a fresh process with deterministic algorithms, in float32 and under
    bf16 autocast: poisoned against copied padding, and the poisoned step twice"""
    code = f"""
import sys, numpy as np, torch
sys.path.insert(0, {ROOT!r})
sys.path.insert(0, {os.path.join(ROOT, 'tests')!r})
from pointnet2_b200 import nets, workloads as W
from test_ragged_fp_gpu import pad
torch.use_deterministic_algorithms(True)
dev = torch.device("cuda:0")
lengths = [4096, 2500, 1025, 3000]
x = W.cloud_surface(len(lengths), 4096, 71)
rs = np.random.RandomState(72)
label = torch.from_numpy(rs.randint(0, 13, (4, 4096))).to(dev)
smpw = torch.from_numpy(rs.rand(4, 4096).astype(np.float32) + 0.5).to(dev)
out = []
for amp in (False, True):
    res = []
    for kind in ("poison", "copy", "poison"):
        torch.manual_seed(0)
        net = nets.PointNet2SemSeg(num_class=13).to(dev).train()
        torch.manual_seed(1)  # the same dropout masks in every run
        with torch.autocast("cuda", dtype=torch.bfloat16, enabled=amp):
            pred, _ = net(torch.from_numpy(pad(x, lengths, kind)).to(dev), lengths=torch.tensor(lengths, device=dev))
            loss = nets.sem_seg_loss(pred.float(), label, smpw, lengths=lengths)
        loss.backward()
        stats = [b for m in net.modules() if isinstance(m, torch.nn.BatchNorm1d) for b in (m.running_mean, m.running_var)]
        res.append([loss.detach(), pred.detach()] + [p.grad.detach().clone() for p in net.parameters()] + stats)
    same = all(torch.equal(a, b) for a, b in zip(res[0], res[1]))
    again = all(torch.equal(a, b) for a, b in zip(res[0], res[2]))
    finite = all(bool(torch.isfinite(t).all()) for t in res[0])
    out.append(f"amp={{amp}} same {{same}} again {{again}} finite {{finite}}")
print("; ".join(out))
"""
    env = dict(os.environ, CUBLAS_WORKSPACE_CONFIG=":4096:8")
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, env=env, cwd=ROOT, timeout=900)
    assert r.returncode == 0, r.stderr[-3000:]
    return r.stdout.strip().splitlines()[-1]


def test_sem_seg_training_step_is_independent_of_the_padding_and_deterministic():
    assert _train_child() == ("amp=False same True again True finite True; amp=True same True again True finite True")


def test_sem_seg_without_lengths_is_unchanged(dev):
    torch.manual_seed(0)
    net = PointNet2SemSeg(num_class=13).to(dev).eval()
    x = T(W.cloud_surface(2, 2048, 81), dev)
    with torch.no_grad():
        a, _ = net(x)
        b, _ = net(x, lengths=[2048, 2048])
    torch.testing.assert_close(a, b, rtol=0, atol=0)
    label = torch.zeros(2, 2048, dtype=torch.long, device=dev)
    w = torch.ones(2, 2048, device=dev)
    assert torch.equal(sem_seg_loss(a, label, w), sem_seg_loss(a, label, w, lengths=[2048, 2048]))
