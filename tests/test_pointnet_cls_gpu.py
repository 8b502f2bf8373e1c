"""PointNet v1 on the GPU: layers.masked_bn_relu_max (csrc/masked_bn.cu) bit for bit against masked_batch_norm_relu + a
masked max, and its backward against float64; sa_mlp_max's whole-cloud entry with lengths (csrc/sa_mlp.cu) bit for bit
against the one-CTA walk and each cloud alone at 1, a few and many CTAs per cloud, and under a CUDA graph with rewritten
lengths; nets.PointNetClsBasic against the float64 restatement (tests/pointnet_cls_oracle.py), inside
batch_invariant(), and under bf16 autocast."""
import copy

import numpy as np
import pytest
import torch
from torch import nn

import numerics as NUM
import pointnet_cls_oracle as PO
from pointnet2_b200 import _lib, layers, nets, shapes as SH, workloads as W
from pointnet2_b200._tensor import DTYPE_CODES, ptr, stream_ptr
from pointnet2_b200.layers import SharedMLP, batch_invariant, masked_batch_norm_relu, masked_bn_relu_max, sa_mlp_max

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
DTYPES = [torch.float32, torch.bfloat16, torch.float16]


@pytest.fixture(autouse=True)
def no_tf32():
    old = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = old


def _bits(t):
    return t.contiguous().view(torch.int16 if t.element_size() == 2 else torch.int32)


def _bn(c, seed=0):
    g = torch.Generator().manual_seed(seed)
    bn = nn.BatchNorm1d(c, eps=layers.BN_EPS, momentum=0.1)
    with torch.no_grad():
        bn.weight.copy_(torch.rand(c, generator=g) * 2 - 0.5)  # some negative gammas
        bn.bias.copy_(torch.randn(c, generator=g) * 0.3)
        bn.running_mean.copy_(torch.randn(c, generator=g))
        bn.running_var.copy_(torch.rand(c, generator=g) + 0.5)
    return bn.to(DEV).train()


def _first_rows(y, mask):
    """(B, C) first row of each (cloud, column) maximum of y (B, N, C) over the rows where mask (B, N)"""
    y = torch.where(mask.unsqueeze(-1), y.float(), float("-inf"))
    m = y.amax(1, keepdim=True)
    rows = torch.arange(y.shape[1], device=y.device).view(1, -1, 1)
    return torch.where(y == m, rows, y.shape[1]).amin(1).int(), m.squeeze(1)


# ------------------------------------------------------------------------------------------------ masked_bn_relu_max
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("c", [1024, 37])
@pytest.mark.parametrize("lens", ["full", "ragged"])
def test_forward_is_the_fused_pair_followed_by_a_masked_max(dtype, c, lens):
    b, n = 6, 300
    torch.manual_seed(1)
    x = (torch.randn(b, n, c, device=DEV) * 2 + 0.5).to(dtype)
    x[:, 7] = x[:, 3]  # tied rows: the first must win
    lengths = [n] * b if lens == "full" else [n, 1, 150, 7, n, 299]
    lt = torch.tensor(lengths, device=DEV)
    mask = layers.row_mask(lt, n)
    bn_a, bn_b = _bn(c), None
    bn_b = copy.deepcopy(bn_a)
    y = masked_batch_norm_relu(bn_a, x.reshape(-1, c), mask.reshape(-1)).reshape(b, n, c)
    want_arg, want = _first_rows(y, mask)
    poisoned = x.clone()
    for i, l in enumerate(lengths):
        poisoned[i, l:] = float("nan")
    got, arg = masked_bn_relu_max(bn_b, poisoned, lt, with_indices=True)
    assert got.dtype == dtype and tuple(got.shape) == (b, c)
    assert torch.equal(_bits(got), _bits(want.to(dtype)))
    assert torch.equal(arg, want_arg)
    for name in ("running_mean", "running_var", "num_batches_tracked"):
        assert torch.equal(getattr(bn_a, name), getattr(bn_b, name)), name
    zeroed = torch.where(mask.unsqueeze(-1), x, 0)
    bn_c = copy.deepcopy(bn_a)
    assert torch.equal(_bits(masked_bn_relu_max(bn_c, zeroed, lt)), _bits(got))  # NaN and zero padding: the same bits
    if lens == "full":
        assert torch.equal(_bits(masked_bn_relu_max(copy.deepcopy(bn_a), x)), _bits(got))  # lengths=None: every row


def _tie_free(lengths, n, c, seed):
    """x (b, n, c) in [0, 1) plus 3 at one real row per (cloud, column): that row's maximum leads by far more than
    rounding, in every dtype"""
    g = torch.Generator(device=DEV).manual_seed(seed)
    b = len(lengths)
    x = torch.rand(b, n, c, device=DEV, generator=g)
    lt = torch.tensor(lengths, device=DEV).view(b, 1, 1)
    win = (torch.rand(b, 1, c, device=DEV, generator=g) * lt).long().clamp(max=n - 1)
    return x.scatter_add(1, win, torch.full((b, 1, c), 3.0, device=DEV))


def _composition64(bn, x, lengths, dout):
    """float64 masked batch norm + ReLU + first-row max: its gradients (dx, dgamma, dbeta), xhat and invstd"""
    b, n, c = x.shape
    mask = layers.row_mask(torch.tensor(lengths, device=DEV), n)
    x64 = x.double().requires_grad_(True)
    w = bn.weight.detach().double().requires_grad_(True)
    bias = bn.bias.detach().double().requires_grad_(True)
    keep = mask.reshape(-1, 1)
    rows = x64.reshape(-1, c)
    cnt = keep.sum()
    mean = torch.where(keep, rows, 0).sum(0) / cnt
    var = (torch.where(keep, rows - mean, 0) ** 2).sum(0) / cnt
    invstd = 1.0 / torch.sqrt(var + bn.eps)
    y = torch.relu((rows - mean) * invstd * w + bias).reshape(b, n, c)
    out = layers._first_max(torch.where(mask.unsqueeze(-1), y, float("-inf")))
    out.backward(dout.double())
    xh = torch.where(keep, (rows - mean) * invstd, 0).detach().reshape(b, n, c)
    return x64.grad, w.grad, bias.grad, xh, invstd.detach(), mask


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("c", [256, 37])
def test_backward_within_the_float64_bound_and_repeatable(dtype, c):
    b, n = 5, 200
    lengths = [200, 1, 120, 64, 199]
    x = _tie_free(lengths, n, c, 4).to(dtype)
    dout = torch.randn(b, c, device=DEV).to(dtype)

    def bn_pos():  # positive gammas: the largest x is the largest y, and it is > 0
        bn = _bn(c)
        with torch.no_grad():
            bn.weight.abs_().add_(0.1)
        return bn

    ref_dx, ref_dg, ref_db, xh, invstd, mask = _composition64(bn_pos(), x, lengths, dout)
    results = []
    for det in (False, True, False):
        bn = bn_pos()
        xr = x.clone().requires_grad_(True)
        prev = torch.are_deterministic_algorithms_enabled()
        torch.use_deterministic_algorithms(det)
        try:
            out = masked_bn_relu_max(bn, xr, torch.tensor(lengths, device=DEV))
            out.backward(dout)
        finally:
            torch.use_deterministic_algorithms(prev)
        assert bool((out.float() > 0).all())
        results.append((xr.grad.clone(), bn.weight.grad.clone(), bn.bias.grad.clone()))
    for r in results[1:]:
        for got, first in zip(r, results[0]):
            assert torch.equal(_bits(got), _bits(first))
    dx, dg, db = results[0]
    fmt = {torch.float32: "f32", torch.bfloat16: "bf16", torch.float16: "f16"}[dtype]
    rows = b * n
    np64 = lambda t: t.double().cpu().numpy()
    gabs = np.abs(np64(dout))                 # every output is > 0: g is dout at the maximum rows
    xhmax = np64(xh.abs().amax((0, 1)))
    # dbeta: a float32 sum of b exact terms.  dgamma and dx also carry the float32 statistics' rounding (sums over every
    # real row, hence L = rows), taken as a relative error of xhat and invstd, so their mass adds (1 + |xhat|) factors.
    mass_db = gabs.sum(0)
    mass_dg = mass_db * (xhmax + 1.0)
    assert NUM.within_bound(np64(db), np64(ref_db), mass_db, b, "f32").all()
    assert NUM.within_bound(np64(dg), np64(ref_dg), mass_dg, rows, "f32").all()
    cnt = float(mask.sum())
    scale = np64(bn.weight.detach().abs() * invstd.float())
    mass_dx = scale * (gabs.max(0) + (mass_db + xhmax * mass_dg) / cnt) * (1.0 + xhmax)
    ok = NUM.within_bound(np64(dx), np64(ref_dx), np.broadcast_to(mass_dx, dx.shape), rows, fmt)
    assert ok.all(), float((dx.double() - ref_dx).abs().max())
    assert torch.equal(dx[~mask], torch.zeros_like(dx[~mask]))


# ------------------------------------------------------------------------------------------- whole-cloud sa_mlp_max
def _old_entry(xyz, points, mlp, dtype):
    """the one-CTA walk of pn2_sa_mlp_max_typed (idx NULL)"""
    stack = layers._mlp_stack(mlp)
    b, n = xyz.shape[:2]
    c = 0 if points is None else points.shape[2]
    out = torch.empty((b, 1, mlp.out_channels), dtype=dtype, device=DEV)
    rc = _lib.load().pn2_sa_mlp_max_typed(DTYPE_CODES[dtype], b, n, c, 1, n, ptr(xyz), ptr(None), ptr(points), ptr(None),
                                          1, 1, *layers._layer_args(stack), ptr(out), out.stride(1), stream_ptr(DEV))
    _lib.check(rc, "pn2_sa_mlp_max_typed")
    return out


def _eval_mlp(cin, widths, seed):
    torch.manual_seed(seed)
    mlp = SharedMLP(cin, widths).to(DEV)
    with torch.no_grad():
        for m in mlp.modules():
            if isinstance(m, nn.BatchNorm1d):
                m.running_mean.normal_(0, 0.3)
                m.running_var.uniform_(0.5, 2.0)
                m.weight.uniform_(-0.5, 1.5)
                m.bias.normal_(0, 0.2)
    return mlp.eval()


# (b, n, c, widths): one CTA per cloud (many clouds), a few per cloud, many per cloud, and clouds packed into one tile
SPLITS = {"one": (600, 128, 13, [64, 128]), "few": (32, 1024, 256, [256, 512, 1024]),
          "many": (2, 4096, 61, [64, 256]), "packed": (7, 20, 5, [32, 48])}


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("shape", list(SPLITS))
def test_whole_cloud_entry_matches_the_one_cta_walk_and_each_cloud_alone(dtype, shape):
    b, n, c, widths = SPLITS[shape]
    mlp = _eval_mlp(c + 3, widths, 5)
    g = torch.Generator(device=DEV).manual_seed(6)
    xyz = torch.rand(b, n, 3, device=DEV, generator=g)
    points = torch.randn(b, n, c, device=DEV, generator=g).to(dtype)
    with torch.no_grad():
        got = sa_mlp_max(xyz, None, points, None, mlp)
        assert torch.equal(_bits(got), _bits(_old_entry(xyz, points, mlp, dtype)))
        rs = np.random.RandomState(7)
        lengths = rs.randint(1, n + 1, b)
        lengths[0], lengths[-1] = 1, n
        lt = torch.from_numpy(lengths).to(DEV)
        px, pp = xyz.clone(), points.clone()
        for i, l in enumerate(lengths):
            px[i, l:] = float("nan")
            pp[i, l:] = float("nan")
        ragged = sa_mlp_max(px, None, pp, None, mlp, lengths=lt)
        assert not torch.isnan(ragged.float()).any()
        for i in sorted({0, b - 1, b // 2, 1 % b}):
            l = int(lengths[i])
            alone = _old_entry(xyz[i:i + 1, :l].contiguous(), points[i:i + 1, :l].contiguous(), mlp, dtype)
            assert torch.equal(_bits(ragged[i:i + 1]), _bits(alone)), i


def test_cuda_graph_replays_rewritten_lengths():
    b, n, c, widths = 4, 2048, 29, [64, 128, 256]
    mlp = _eval_mlp(c, widths, 8)
    points = torch.randn(b, n, c, device=DEV)
    lt = torch.tensor([2048, 100, 1, 1500], device=DEV, dtype=torch.int32)
    with torch.no_grad():
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            sa_mlp_max(None, None, points, None, mlp, True, False, lengths=lt)  # warm-up outside the capture
        torch.cuda.current_stream().wait_stream(s)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            out = sa_mlp_max(None, None, points, None, mlp, True, False, lengths=lt)
        for new in ([2048, 100, 1, 1500], [5, 2048, 999, 64]):
            lt.copy_(torch.tensor(new, device=DEV))
            graph.replay()
            torch.cuda.synchronize()
            want = sa_mlp_max(None, None, points, None, mlp, True, False, lengths=torch.tensor(new, device=DEV))
            assert torch.equal(_bits(out), _bits(want))


# ----------------------------------------------------------------------------------------------- PointNetClsBasic
def _net(num_class=40):
    torch.manual_seed(0)
    net = nets.PointNetClsBasic(num_class).to(DEV)
    net.dp1.p = 0.0
    return net


CASE = dict(b=4, n=1024, lengths=[1024, 700, 300, 1])


def _rel(got, ref, floor=0.0):
    got, ref = got.double().reshape(-1).cpu(), ref.double().reshape(-1).cpu()
    return float((got - ref).norm()) / max(float(ref.norm()), floor, 1e-300)


@pytest.mark.parametrize("layout", ["dense", "ragged"])
def test_training_step_matches_the_float64_restatement(layout):
    b, n = CASE["b"], CASE["n"]
    pts = W.DISTRIBUTIONS["S"](b, n, 21)
    lengths = CASE["lengths"] if layout == "ragged" else None
    label = np.array([1, 5, 39, 0])
    net = _net().train()
    state = copy.deepcopy(net.state_dict())
    x = torch.from_numpy(NUM.pad_rows(pts, lengths, "poison") if lengths else pts).to(DEV)
    lens = None if lengths is None else torch.tensor(lengths, device=DEV)
    logits, _ = net(x, lens)
    loss = nets.cls_loss(logits, torch.from_numpy(label).to(DEV))
    loss.backward()
    ref = PO.run(state, pts, lengths=lengths, label=label, training=True, device=DEV)
    assert _rel(logits, ref.logits) <= 3e-4 and _rel(loss, ref.loss) <= 3e-4
    for prefix in ("feat", "conv5", "fc1", "fc2", "fc3"):
        keys = [k for k, _ in net.named_parameters() if k.startswith(prefix + ".")]
        got = torch.cat([dict(net.named_parameters())[k].grad.reshape(-1) for k in keys])
        want = torch.cat([ref.grads[k].reshape(-1) for k in keys])
        assert _rel(got, want) <= 5e-2, prefix
    sd = net.state_dict()
    for k, v in ref.stats.items():
        if k.endswith("num_batches_tracked"):
            assert int(sd[k]) == int(v)
        else:
            assert _rel(sd[k], v, floor=1e-3) <= 1e-4, k
    # eval forward with the updated statistics, in the default mode and inside batch_invariant()
    net.eval()
    ev = PO.run(dict(state, **ref.stats), pts, lengths=lengths, training=False, device=DEV)
    with torch.no_grad():
        assert _rel(net(x, lens)[0], ev.logits) <= 3e-4
        with batch_invariant():
            assert _rel(net(x, lens)[0], ev.logits) <= 3e-4


def test_batch_invariant_logits_do_not_depend_on_the_batch():
    b, n = 6, 1024
    pts = torch.from_numpy(W.DISTRIBUTIONS["S"](b, n, 31)).to(DEV)
    lengths = [1024, 333, 1, 800, 1024, 77]
    net = _net(10).eval()
    with torch.no_grad():  # a few steps' worth of running statistics
        for m in net.modules():
            if isinstance(m, nn.BatchNorm1d):
                m.running_mean.normal_(0, 0.2)
                m.running_var.uniform_(0.5, 2.0)
    lt = torch.tensor(lengths, device=DEV)
    with torch.no_grad(), batch_invariant():
        full = net(pts, lt)[0]
        assert tuple(full.shape) == (b, 10)
        perm = torch.tensor([4, 2, 0, 5, 1, 3], device=DEV)
        permuted = net(pts[perm], lt[perm])[0]
        assert torch.equal(_bits(permuted), _bits(full[perm]))
        for i, l in enumerate(lengths):
            alone = net(pts[i:i + 1, :l].contiguous())[0]
            assert torch.equal(_bits(alone), _bits(full[i:i + 1])), i
        rs = np.random.RandomState(3)
        ss = SH.ShapeSet([rs.standard_normal((s, 3)).astype(np.float32) for s in (1024, 3000, 700)], rs.randint(0, 10, 3),
                         num_class=10, normalize=False, device=DEV)
        idx = torch.tensor([0, 1, 2, 1], device=DEV)
        a = SH.classify_votes(net, ss, idx, 4, 7, chunk=1)
        c = SH.classify_votes(net, ss, idx, 4, 7, chunk=3)
        assert torch.equal(_bits(a), _bits(c))


def test_bf16_autocast_training_step_is_finite():
    b, n = 8, 1024
    pts = torch.from_numpy(W.DISTRIBUTIONS["S"](b, n, 41)).to(DEV)
    lt = torch.tensor([1024, 900, 10, 512, 1024, 1, 640, 333], device=DEV)
    net = _net().train()
    with torch.autocast("cuda", dtype=torch.bfloat16):
        logits, _ = net(pts, lt)
    loss = nets.cls_loss(logits.float(), torch.arange(b, device=DEV))
    loss.backward()
    assert torch.isfinite(loss)
    for k, p in net.named_parameters():
        assert p.grad is not None and bool(torch.isfinite(p.grad).all()), k
    assert float(net.conv5.body[0].weight.grad.abs().sum()) > 0
