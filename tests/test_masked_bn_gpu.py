"""The fused masked batch norm + ReLU (csrc/masked_bn.cu, layers.masked_batch_norm_relu) on the GPU: against float64
truth and the torch path, its gradient, inert padding, determinism, accuracy far from zero mean, the routing in
SharedMLP, CUDA-graph capture without host synchronisation, the segmentation nets, and a tensor beyond 2^31 elements."""
import copy
import json
import os
import subprocess
import sys

import pytest
import torch

from pointnet2_b200 import _lib, layers
from pointnet2_b200.layers import SharedMLP, masked_batch_norm, masked_batch_norm_relu, row_mask

sys.path.insert(0, os.path.dirname(__file__))
from numerics import ulp  # noqa: E402

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DTYPES = [torch.float32, torch.bfloat16, torch.float16]
FMT = {torch.float32: "f32", torch.bfloat16: "bf16", torch.float16: "f16"}


def _keep(kind, r, dev, seed=0):
    if kind == "one":
        k = torch.zeros(r, dtype=torch.bool)
        k[r // 2] = True
    elif kind == "all":
        k = torch.ones(r, dtype=torch.bool)
    else:  # random, about 60 % real rows
        k = torch.rand(r, generator=torch.Generator().manual_seed(seed)) < 0.6
        k[0] = True
    return k.to(dev)


def _poison(x, keep, kind="nan"):
    """x with its padding rows overwritten: NaN / +inf / -inf cycling, or copies of the first real row"""
    x = x.clone()
    pad = (~keep).nonzero().squeeze(1)
    if kind == "nan":
        vals = torch.tensor([float("nan"), float("inf"), float("-inf")], device=x.device, dtype=x.dtype)
        x[pad] = vals[torch.arange(pad.numel(), device=x.device) % 3].unsqueeze(1).expand(-1, x.shape[1])
    else:
        first = keep.nonzero()[0, 0]
        x[pad] = x[first].clone()
    return x


def _bn(c, dev, affine=True, track=True, momentum=0.1, seed=0):
    torch.manual_seed(seed)
    bn = torch.nn.BatchNorm1d(c, affine=affine, track_running_stats=track, momentum=momentum).to(dev).train()
    if affine:
        with torch.no_grad():
            bn.weight.uniform_(0.5, 1.5)
            bn.bias.uniform_(-0.5, 0.5)
    if track:
        with torch.no_grad():
            bn.running_mean.uniform_(-1, 1)
            bn.running_var.uniform_(0.5, 2)
    return bn


def _truth(x, keep, bn):
    """float64: y of the masked formula + ReLU, padding rows 0, and the batch mean / biased variance"""
    xr = x[keep].double()
    mean, var = xr.mean(0), xr.var(0, unbiased=False)
    y = (x.double() - mean) / torch.sqrt(var + bn.eps)
    if bn.affine:
        y = y * bn.weight.double() + bn.bias.double()
    y = torch.where(keep.unsqueeze(1), y.clamp_min(0), 0)
    return y, mean, var


def _assert_close_fmt(got, ref64, dtype, rtol=1e-5, atol=1e-5):
    """float32: rtol / atol; 16-bit: within the float32 tolerance plus 1/2 ulp of the format (one rounding)"""
    got, ref64 = got.detach().double(), ref64.detach()
    tol = atol + rtol * ref64.abs()
    if dtype != torch.float32:
        tol = tol + 0.5 * torch.from_numpy(ulp((ref64.abs() + tol).cpu().numpy(), FMT[dtype])).to(ref64.device)
    err = (got - ref64).abs()
    assert bool((err <= tol).all()), f"max err {float(err.max()):.3g}, at tol {float(tol[err.argmax() // err.shape[1]].max()):.3g}"


@pytest.mark.parametrize("dtype", DTYPES, ids=["f32", "bf16", "f16"])
@pytest.mark.parametrize("c", [1, 3, 16, 128, 130, 512])
@pytest.mark.parametrize("kind,r", [("one", 77), ("all", 4096), ("random", 10007)])
def test_forward_matches_float64(dev, dtype, c, kind, r):
    keep = _keep(kind, r, dev, seed=c)
    bn = _bn(c, dev, seed=c)
    x = (torch.randn(r, c, device=dev) * 2 + 0.5).to(dtype)
    want, _, _ = _truth(x, keep, bn)
    y = masked_batch_norm_relu(bn, _poison(x, keep), keep)
    assert y.dtype == dtype
    _assert_close_fmt(y, want, dtype)
    assert bool((y[~keep] == 0).all())


@pytest.mark.parametrize("dtype", DTYPES, ids=["f32", "bf16", "f16"])
@pytest.mark.parametrize("affine", [True, False])
@pytest.mark.parametrize("track,momentum", [(True, 0.1), (True, 0.5), (True, None), (False, 0.1)])
def test_variants_and_running_statistics(dev, dtype, affine, track, momentum):
    r, c = 3001, 130
    bn = _bn(c, dev, affine=affine, track=track, momentum=momentum)
    rm0 = bn.running_mean.clone() if track else None
    rv0 = bn.running_var.clone() if track else None
    rm, rv, nbt = (rm0.double(), rv0.double(), 0) if track else (None, None, 0)
    for step in range(2):  # the statistics and num_batches_tracked accumulate
        keep = _keep("random", r, dev, seed=step)
        x = (torch.randn(r, c, device=dev) + step).to(dtype)
        want, mean, var = _truth(x, keep, bn)
        y = masked_batch_norm_relu(bn, _poison(x, keep), keep)
        _assert_close_fmt(y, want, dtype)
        if track:
            nbt += 1
            f = 1.0 / nbt if momentum is None else momentum
            cnt = int(keep.sum())
            rm = rm * (1 - f) + mean * f
            rv = rv * (1 - f) + var * cnt / max(cnt - 1, 1) * f
            assert int(bn.num_batches_tracked) == nbt
            torch.testing.assert_close(bn.running_mean.double(), rm, rtol=1e-5, atol=1e-5)
            torch.testing.assert_close(bn.running_var.double(), rv, rtol=1e-5, atol=1e-5)
        else:
            assert bn.running_mean is None


@pytest.mark.parametrize("dtype", DTYPES, ids=["f32", "bf16", "f16"])
@pytest.mark.parametrize("c", [1, 16, 128, 130])
def test_matches_the_torch_path(dev, dtype, c):
    r = 20000
    keep = _keep("random", r, dev, seed=3)
    x = (torch.randn(r, c, device=dev) * 3 - 1).to(dtype)
    a, b = _bn(c, dev), _bn(c, dev)
    got = masked_batch_norm_relu(a, _poison(x, keep), keep)
    k1 = keep.unsqueeze(1)
    want = torch.where(k1, torch.relu(masked_batch_norm(b, torch.where(k1, x, 0), k1)), 0)
    if dtype == torch.float32:
        torch.testing.assert_close(got, want, rtol=1e-5, atol=1e-5)
    else:  # one rounding of the format apart at most, on top of float32 noise
        tol = 1e-5 + torch.from_numpy(ulp(want.detach().float().abs().cpu().numpy(), FMT[dtype])).to(dev)
        assert bool(((got.detach().double() - want.detach().double()).abs() <= tol).all())
    torch.testing.assert_close(a.running_mean, b.running_mean, rtol=1e-5, atol=1e-6)
    torch.testing.assert_close(a.running_var, b.running_var, rtol=1e-5, atol=1e-6)
    assert torch.equal(a.num_batches_tracked, b.num_batches_tracked)


def _grads(bn, x, keep, dy):
    xx = x.clone().requires_grad_(True)
    for p in bn.parameters():
        p.grad = None
    y = masked_batch_norm_relu(bn, xx, keep)
    y.backward(dy)
    return y.detach(), xx.grad, (bn.weight.grad if bn.affine else None), (bn.bias.grad if bn.affine else None)


@pytest.mark.parametrize("dtype", DTYPES, ids=["f32", "bf16", "f16"])
@pytest.mark.parametrize("affine", [True, False])
@pytest.mark.parametrize("c,r", [(1, 999), (3, 5000), (128, 10007), (130, 4096), (512, 2049)])
def test_backward_matches_float64_autograd(dev, dtype, affine, c, r):
    keep = _keep("random", r, dev, seed=r)
    bn = _bn(c, dev, affine=affine)
    x = (torch.randn(r, c, device=dev) * 2 + 1).to(dtype)
    dy = torch.randn(r, c, device=dev).to(dtype)
    y, dx, dg, db = _grads(bn, _poison(x, keep), keep, _poison(dy, keep))
    # float64 autograd of the masked formula, with the ReLU's gate taken from the kernel's own y (an element within
    # rounding of 0 may fall either side)
    x64 = x.double().requires_grad_(True)
    g64 = bn.weight.detach().double().requires_grad_(True) if affine else None
    b64 = bn.bias.detach().double().requires_grad_(True) if affine else None
    k1 = keep.unsqueeze(1)
    xr = torch.where(k1, x64, 0)
    cnt = keep.sum()
    mean = xr.sum(0) / cnt
    var = (torch.where(k1, x64 - mean, 0) ** 2).sum(0) / cnt
    t = (x64 - mean) / torch.sqrt(var + bn.eps)
    if affine:
        t = t * g64 + b64
    out = torch.where(k1 & (y > 0), t, 0)
    out.backward(torch.where(k1, dy.double(), 0))
    k = keep
    _assert_close_fmt(dx[k], x64.grad[k], dtype, rtol=1e-4, atol=1e-5)
    assert bool((dx[~k] == 0).all()), "dx is exactly 0 on padding rows"
    if affine:
        torch.testing.assert_close(dg.double(), g64.grad, rtol=1e-4, atol=1e-5)
        torch.testing.assert_close(db.double(), b64.grad, rtol=1e-4, atol=1e-5)


def _run_all(x, dy, keep, c, dev):
    bn = _bn(c, dev, momentum=None)
    outs = []
    for _ in range(2):
        y, dx, dg, db = _grads(bn, x, keep, dy)
        outs += [y, dx, dg.clone(), db.clone(), bn.running_mean.clone(), bn.running_var.clone()]
    return outs


@pytest.mark.parametrize("dtype", DTYPES, ids=["f32", "bf16", "f16"])
@pytest.mark.parametrize("c", [3, 128])
def test_padding_and_determinism_are_bit_exact(dev, dtype, c):
    r = 30011
    keep = _keep("random", r, dev, seed=5)
    x = torch.randn(r, c, device=dev).to(dtype)
    dy = torch.randn(r, c, device=dev).to(dtype)
    ref = _run_all(_poison(x, keep), _poison(dy, keep), keep, c, dev)
    copied = _run_all(_poison(x, keep, "copy"), _poison(dy, keep, "copy"), keep, c, dev)
    again = _run_all(_poison(x, keep), _poison(dy, keep), keep, c, dev)
    was = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        det = _run_all(_poison(x, keep), _poison(dy, keep), keep, c, dev)
    finally:
        torch.use_deterministic_algorithms(was)
    for other in (copied, again, det):
        for a, b in zip(ref, other):
            assert torch.equal(a, b)


@pytest.mark.parametrize("offset", [10.0, 1000.0, 3000.0])
@pytest.mark.parametrize("c", [4, 128])
def test_statistics_hold_far_from_zero_mean(dev, offset, c):
    """the bound of test_masked_batch_norm_statistics_hold_far_from_zero_mean: 4x BatchNorm1d's own float32 error"""
    r = 65536
    g = torch.Generator().manual_seed(8)
    x = torch.randn(r, c, generator=g) + offset
    keep = torch.arange(r) % 4 != 0  # 75 % real rows
    bn, ref = torch.nn.BatchNorm1d(c, affine=False).to(dev), torch.nn.BatchNorm1d(c, affine=False)
    real = x[keep]
    got = masked_batch_norm_relu(bn, x.to(dev), keep.to(dev))[keep.to(dev)].cpu().double()
    want = ref(real).detach()
    x64 = real.double()
    truth = ((x64 - x64.mean(0)) / torch.sqrt(x64.var(0, unbiased=False) + ref.eps)).clamp_min(0)
    own = float((want.double().clamp_min(0) - truth).abs().max())
    assert float((got - truth).abs().max()) <= 4 * own + 1e-5, (offset, own)
    torch.testing.assert_close(bn.running_mean.cpu(), ref.running_mean, rtol=1e-5, atol=1e-5)
    torch.testing.assert_close(bn.running_var.cpu(), ref.running_var, rtol=1e-2, atol=1e-4)


def _mlp(dev, seed=0, cin=6, widths=(32, 64, 16)):
    torch.manual_seed(seed)
    m = SharedMLP(cin, list(widths))
    with torch.no_grad():
        for mod in m.body:
            if isinstance(mod, torch.nn.BatchNorm1d):
                mod.weight.uniform_(0.5, 1.5)
                mod.bias.uniform_(-0.2, 0.2)
    return m.to(dev)


def test_shared_mlp_routes_training_through_the_kernels(dev):
    b, n, lengths = 4, 1000, [1000, 3, 640, 999]
    mask = row_mask(torch.tensor(lengths), n)
    t = torch.randn(b, n, 6)
    t[~mask] = float("nan")
    gpu = _mlp(dev).train()
    cpu = copy.deepcopy(gpu).cpu()
    tg = t.to(dev).requires_grad_(True)
    before = _lib.launch_count()
    out = gpu(tg, mask.to(dev))
    assert _lib.launch_count() - before == 3 * 3  # three batch norms, three kernels each
    out.square().sum().backward()
    assert _lib.launch_count() - before == 6 * 3
    tc = t.clone().requires_grad_(True)
    want = cpu(tc, mask)
    want.square().sum().backward()
    torch.testing.assert_close(out.cpu(), want, rtol=1e-4, atol=1e-5)
    torch.testing.assert_close(tg.grad.cpu(), tc.grad, rtol=1e-3, atol=1e-4)
    for p, q in zip(gpu.parameters(), cpu.parameters()):
        torch.testing.assert_close(p.grad.cpu(), q.grad, rtol=1e-3, atol=1e-3)
    for p, q in zip(gpu.buffers(), cpu.buffers()):
        torch.testing.assert_close(p.cpu(), q, rtol=1e-4, atol=1e-5)
    assert torch.equal(out[~mask.to(dev)], torch.zeros_like(out[~mask.to(dev)]))


def _composition(m, t, mask):
    """SharedMLP(t, mask) as the torch modules compute it without the fused op: the input's padding rows zeroed, then
    per module Linear -> where, BatchNorm1d -> where(masked_batch_norm) (bn(x) in eval mode), ReLU"""
    keep = mask.reshape(-1, 1)
    x = torch.where(keep, t.reshape(-1, t.shape[-1]), 0)
    for mod in m.body:
        if isinstance(mod, torch.nn.BatchNorm1d):
            x = torch.where(keep, masked_batch_norm(mod, x, keep), 0)
        elif isinstance(mod, torch.nn.Linear):
            x = torch.where(keep, mod(x), 0)
        else:
            x = mod(x)
    return x.reshape(*t.shape[:-1], -1)


def test_shared_mlp_eval_and_dense_paths_are_the_torch_modules(dev):
    b, n, lengths = 2, 300, [300, 111]
    mask = row_mask(torch.tensor(lengths), n).to(dev)
    t = torch.randn(b, n, 6, device=dev)
    m = _mlp(dev).train()
    m(t, mask)  # non-trivial running statistics
    ref = copy.deepcopy(m).eval()
    before = _lib.launch_count()
    got_eval = m.eval()(t, mask)
    got_dense = m.train()(t)
    assert _lib.launch_count() == before
    # eval: bn(x) with the running statistics, written out independently of SharedMLP.forward
    keep = mask.reshape(-1, 1)
    x = torch.where(keep, t.reshape(-1, 6), 0)
    for mod in ref.body:
        x = torch.where(keep, mod(x), 0) if not isinstance(mod, torch.nn.ReLU) else mod(x)
    assert torch.equal(got_eval, x.reshape(b, n, -1))
    assert torch.equal(got_dense, ref.body.train()(t.reshape(-1, 6)).reshape(b, n, -1))


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
def test_16bit_converted_shared_mlp_keeps_the_torch_path(dev, dtype):
    """a module converted with .half() / .to(bfloat16) has 16-bit batch-norm parameters and buffers, which the kernels
    do not take: it trains through masked_batch_norm exactly as before, with no launch of the library"""
    b, n, lengths = 3, 500, [500, 77, 260]
    mask = row_mask(torch.tensor(lengths), n).to(dev)
    t = torch.randn(b, n, 6, device=dev)
    t[~mask] = float("nan")
    t = t.to(dtype)
    m = _mlp(dev).to(dtype).train()
    ref = copy.deepcopy(m)
    tg, tr = t.clone().requires_grad_(True), t.clone().requires_grad_(True)
    before = _lib.launch_count()
    out = m(tg, mask)
    out.float().square().sum().backward()
    assert _lib.launch_count() == before
    want = _composition(ref, tr, mask)
    want.float().square().sum().backward()
    assert torch.equal(out, want)
    assert torch.equal(tg.grad, tr.grad)
    for p, q in zip(m.parameters(), ref.parameters()):
        assert torch.equal(p.grad, q.grad)
    for p, q in zip(m.buffers(), ref.buffers()):
        assert torch.equal(p, q)


def test_op_argument_errors(dev):
    x = torch.randn(64, 8, device=dev)
    keep = torch.ones(64, dtype=torch.bool, device=dev)
    before = _lib.launch_count()
    with pytest.raises(RuntimeError, match="device"):
        masked_batch_norm_relu(_bn(8, dev), x, keep.cpu())  # a host mask next to a CUDA x
    with pytest.raises(ValueError):
        masked_batch_norm_relu(_bn(8, dev), x, keep.to(torch.uint8))
    with pytest.raises(ValueError, match="eval"):
        masked_batch_norm_relu(_bn(8, dev).eval(), x, keep)  # eval with running statistics is bn(x)
    for dtype in (torch.float16, torch.bfloat16):
        with pytest.raises(TypeError, match="float32"):
            masked_batch_norm_relu(_bn(8, dev).to(dtype), x.to(dtype), keep)
    with pytest.raises(RuntimeError, match="device"):
        masked_batch_norm_relu(_bn(8, "cpu"), x, keep)  # the module left on the host
    assert _lib.launch_count() == before


@pytest.mark.parametrize("dtype", DTYPES, ids=["f32", "bf16", "f16"])
@pytest.mark.parametrize("c", [16, 128])
def test_misaligned_tensors_give_the_same_bits(dev, dtype, c):
    """c % 4 == 0 with tensors one element off a 4-element boundary: scalar loads in the same thread geometry, so the
    same sums in the same order and the same bits as the aligned call"""
    r = 10007
    keep = _keep("random", r, dev, seed=11)
    x = torch.randn(r, c, device=dev).to(dtype)
    dy = torch.randn(r, c, device=dev).to(dtype)

    def offset(t):
        buf = torch.empty(t.numel() + 1, dtype=t.dtype, device=dev)
        v = buf[1:].view(t.shape)
        v.copy_(t)
        assert v.is_contiguous() and v.data_ptr() % (4 * t.element_size()) != 0
        return v

    res = []
    for xx, gg in ((x, dy), (offset(x), offset(dy))):
        bn = _bn(c, dev)
        xx = xx.detach().requires_grad_(True)
        y = masked_batch_norm_relu(bn, xx, keep)
        y.backward(gg)
        res.append([y.detach(), xx.grad, bn.weight.grad, bn.bias.grad, bn.running_mean, bn.running_var])
    for a, b in zip(*res):
        assert torch.equal(a, b)


def test_no_host_sync_and_cuda_graph_capture(dev):
    b, n = 4, 2048
    t = torch.randn(b, n, 6, device=dev)
    lengths = torch.tensor([2048, 1000, 7, 1500], device=dev)
    m_graph = _mlp(dev, seed=3).train()
    m_eager = copy.deepcopy(m_graph)
    torch.cuda.set_sync_debug_mode("error")
    try:
        x = t.clone().requires_grad_(True)
        m_eager(x, row_mask(lengths, n)).sum().backward()  # forward and backward: no synchronisation
    finally:
        torch.cuda.set_sync_debug_mode("default")
    with torch.no_grad():
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            m_graph(t, row_mask(lengths, n))  # warm-up, as m_eager had
        torch.cuda.current_stream().wait_stream(s)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            out = m_graph(t, row_mask(lengths, n))
        lengths.copy_(torch.tensor([100, 2048, 1, 2000], device=dev))
        graph.replay()
        want = m_eager(t, row_mask(lengths, n))
    torch.cuda.synchronize()
    assert torch.equal(out, want)
    for p, q in zip(m_graph.buffers(), m_eager.buffers()):
        assert torch.equal(p, q)


def _nets_child():
    """In a fresh process with deterministic algorithms: ragged training steps of PointNet2SemSeg and PointNet2PartSeg in
    float32 and under bf16 autocast.  Prints, per case, whether the step is finite and bit-identical with poisoned and
    copied padding, its distance to the same step on the torch path (loss, and the largest relative gradient error per
    parameter), and the losses of four Adam steps."""
    code = f"""
import sys, json, numpy as np, torch
sys.path.insert(0, {ROOT!r})
sys.path.insert(0, {os.path.join(ROOT, 'tests')!r})
from pointnet2_b200 import nets, layers, workloads as W
from pointnet2_b200.layers import row_mask
from test_ragged_fp_gpu import pad
torch.use_deterministic_algorithms(True)
dev = torch.device("cuda:0")
fused = layers.fused_bn_applies

def setup(name):
    if name == "semseg":
        lengths, n = [2048, 1500, 700, 1999], 2048
        x = W.cloud_surface(len(lengths), n, 71)
        rs = np.random.RandomState(72)
        label = torch.from_numpy(rs.randint(0, 13, (4, n))).to(dev)
        smpw = torch.from_numpy(rs.rand(4, n).astype(np.float32) + 0.5).to(dev)
        make = lambda: nets.PointNet2SemSeg(num_class=13)
        loss = lambda pred, lens: nets.sem_seg_loss(pred.float(), label, smpw, lengths=lens)
    else:
        lengths, n = [2048, 1200, 2047, 600], 2048
        x, cls, lab = W.part_shapes(len(lengths), n, 2, nets.PART_OFFSETS)
        label = torch.from_numpy(lab).to(dev)
        make = lambda: nets.PointNet2PartSeg()
        loss = lambda pred, lens: nets.part_seg_loss(pred, label, lengths=lens)
    return x, lengths, make, loss

def step(net, x, lens, loss, amp):
    torch.manual_seed(1)  # the same dropout masks in every run
    with torch.autocast("cuda", dtype=torch.bfloat16, enabled=amp):
        pred, _ = net(x, lengths=lens)
        l = loss(pred, lens)
    l.backward()
    return l

out = {{}}
for name in ("semseg", "partseg"):
    pts, lengths, make, loss = setup(name)
    lens = torch.tensor(lengths, device=dev)
    for amp in (False, True):
        res = []
        for kind, path in (("poison", "fused"), ("copy", "fused"), ("poison", "torch")):
            layers.fused_bn_applies = fused if path == "fused" else (lambda bn, x: False)
            torch.manual_seed(0)
            net = make().to(dev).train()
            x = torch.from_numpy(pad(pts, lengths, kind)).to(dev)
            l = step(net, x, lens, loss, amp)
            stats = [b for m in net.modules() if isinstance(m, torch.nn.BatchNorm1d) for b in (m.running_mean, m.running_var)]
            res.append([l.detach()] + [p.grad.detach().clone() for p in net.parameters()] + stats)
        layers.fused_bn_applies = fused
        same = all(torch.equal(a, b) for a, b in zip(res[0], res[1]))
        finite = all(bool(torch.isfinite(t).all()) for t in res[0])
        loss_rel = abs(float(res[0][0]) - float(res[2][0])) / abs(float(res[2][0]))
        # over all gradients together: a Linear bias feeding a batch norm has an analytically zero gradient, whose
        # rounding noise differs between the paths by 100 % of itself
        ga = torch.cat([g.flatten().double() for g in res[0][1:]])
        gb = torch.cat([g.flatten().double() for g in res[2][1:]])
        grad_rel = float((ga - gb).norm() / gb.norm())
        torch.manual_seed(0)
        net = make().to(dev).train()
        opt = torch.optim.Adam(net.parameters(), lr=1e-3)
        x = torch.from_numpy(pad(pts, lengths, "poison")).to(dev)
        losses = []
        for _ in range(4):
            opt.zero_grad()
            losses.append(float(step(net, x, lens, loss, amp)))
            opt.step()
        out[f"{{name}} amp={{amp}}"] = dict(same=same, finite=finite, loss_rel=loss_rel, grad_rel=grad_rel, losses=losses)
print(json.dumps(out))
"""
    env = dict(os.environ, CUBLAS_WORKSPACE_CONFIG=":4096:8")
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, env=env, cwd=ROOT, timeout=900)
    assert r.returncode == 0, r.stderr[-3000:]
    return json.loads(r.stdout.strip().splitlines()[-1])


def test_segmentation_nets_train_on_the_fused_path():
    res = _nets_child()
    print(json.dumps(res, indent=1))
    assert len(res) == 4
    for case, v in res.items():
        amp = case.endswith("True")
        assert v["finite"] and v["same"], case
        assert v["loss_rel"] <= (1e-2 if amp else 1e-4), (case, v)
        assert v["grad_rel"] <= (5e-2 if amp else 1e-3), (case, v)
        assert v["losses"][-1] < v["losses"][0], (case, v)


def test_beyond_2_to_31_elements(dev):
    """bf16, 2^31 + 2^21 elements: the running statistics (momentum 1, so the batch's own) against float64 sums over the
    real rows, and y, dx on sampled rows, the last ones included, against the formula"""
    free, _ = torch.cuda.mem_get_info(dev)
    if free < 24 * (1 << 30):
        pytest.skip("needs 24 GiB of free device memory")
    c = 128
    r = (1 << 31) // c + (1 << 14)
    keep = torch.arange(r, device=dev) % 3 != 1
    x = torch.empty(r, c, dtype=torch.bfloat16, device=dev)
    gen = torch.Generator(device=dev).manual_seed(4)
    step = 1 << 20
    for s in range(0, r, step):
        x[s:s + step] = (torch.randn(min(step, r - s), c, device=dev, generator=gen) * 2 + 5).to(torch.bfloat16)
    x[(~keep).nonzero().squeeze(1)[-1000:]] = float("nan")  # never read
    bn = torch.nn.BatchNorm1d(c, momentum=1.0).to(dev)
    xr = x.requires_grad_(True)
    y = masked_batch_norm_relu(bn, xr, keep)
    dy = torch.ones_like(y)
    y.backward(dy)
    dx = xr.grad
    x = x.detach()
    # float64 two-pass over the real rows, in slices
    tot = torch.zeros(c, dtype=torch.float64, device=dev)
    for s in range(0, r, step):
        tot += torch.where(keep[s:s + step, None], x[s:s + step].double(), 0).sum(0)
    cnt = int(keep.sum())
    mean = tot / cnt
    m2 = torch.zeros_like(mean)
    for s in range(0, r, step):
        m2 += torch.where(keep[s:s + step, None], x[s:s + step].double() - mean, 0).square().sum(0)
    var = m2 / cnt
    torch.testing.assert_close(bn.running_mean.double(), mean, rtol=1e-5, atol=1e-5)
    torch.testing.assert_close(bn.running_var.double(), var * cnt / (cnt - 1), rtol=1e-4, atol=1e-5)
    invstd = 1 / torch.sqrt(var + bn.eps)
    rows = torch.cat([torch.randint(0, r, (100000,), device=dev, generator=gen), torch.arange(r - 1000, r, device=dev)])
    k = keep[rows]
    xh = (x[rows].double() - mean) * invstd
    want = torch.where(k[:, None], xh.clamp_min(0), 0)
    _assert_close_fmt(y[rows], want, torch.bfloat16, rtol=1e-4, atol=1e-4)
    assert bool((dx[rows][~k] == 0).all()) and bool((y[rows][~k] == 0).all())
    # with dy = 1: g = [y > 0]; the column sums of g and g * xhat in float64, in slices
    sg = torch.zeros_like(mean)
    sgx = torch.zeros_like(mean)
    for s in range(0, r, step):
        gg = torch.where(keep[s:s + step, None], y[s:s + step].detach(), 0) > 0
        sg += gg.double().sum(0)
        sgx += torch.where(gg, (x[s:s + step].detach().double() - mean) * invstd, 0).sum(0)
    torch.testing.assert_close(bn.bias.grad.double(), sg, rtol=1e-5, atol=1e-3)
    torch.testing.assert_close(bn.weight.grad.double(), sgx, rtol=1e-4, atol=1.0)
    g = (y[rows].detach() > 0).double()
    want_dx = torch.where(k[:, None], invstd * (g - sg / cnt - xh * sgx / cnt), 0)
    _assert_close_fmt(dx[rows], want_dx, torch.bfloat16, rtol=1e-4, atol=1e-5)
