"""CPU tests of variable-size clouds in feature propagation and the segmentation net: the masked batch norm of SharedMLP
against BatchNorm1d on the packed real rows, the padding's independence, sem_seg_loss with lengths, the validation of
lengths, and which C entry each interpolation op calls (the library mocked)."""
import copy
import inspect
from unittest import mock

import pytest
import torch

from pointnet2_b200 import _lib, layers, nets, pointnet_util, tf_interpolate
from pointnet2_b200.layers import SharedMLP, row_mask


def _padded(b, n, c, lengths, seed, padding):
    g = torch.Generator().manual_seed(seed)
    t = torch.randn(b, n, c, generator=g)
    for i, l in enumerate(lengths):
        if padding == "nan":
            t[i, l:] = float("nan")
            t[i, l + 1::3] = float("inf")
        elif padding == "copy":
            t[i, l:] = t[i, torch.arange(l, n) % l]
    return t


def _mlp(seed, cin=6, widths=(16, 8)):
    torch.manual_seed(seed)
    m = SharedMLP(cin, list(widths))
    with torch.no_grad():  # non-trivial affine parameters
        for mod in m.body:
            if isinstance(mod, torch.nn.BatchNorm1d):
                mod.weight.uniform_(0.5, 1.5)
                mod.bias.uniform_(-0.5, 0.5)
    return m


def _bns(m):
    return [mod for mod in m.body if isinstance(mod, torch.nn.BatchNorm1d)]


@pytest.mark.parametrize("momentum", [0.1, 0.5, None])
def test_masked_shared_mlp_matches_batch_norm_on_the_packed_rows(momentum):
    b, n, lengths = 3, 40, [40, 17, 2]
    t = _padded(b, n, 6, lengths, 0, "nan")
    mask = row_mask(torch.tensor(lengths), n)
    masked, packed = _mlp(1), _mlp(1)
    for m in (masked, packed):
        for bn in _bns(m):
            bn.momentum = momentum
    g = torch.randn(b, n, 8, generator=torch.Generator().manual_seed(2))
    for step in range(2):  # twice: the running statistics and num_batches_tracked accumulate
        masked.zero_grad()
        packed.zero_grad()
        out = masked(t, mask)
        want = packed(t[mask])
        torch.testing.assert_close(out[mask], want, rtol=1e-5, atol=1e-5)
        assert torch.equal(out[~mask], torch.zeros_like(out[~mask])), "padding rows must be 0"
        (out[mask] * g[mask]).sum().backward()
        (want * g[mask]).sum().backward()
        for p, q in zip(masked.parameters(), packed.parameters()):
            torch.testing.assert_close(p.grad, q.grad, rtol=1e-4, atol=1e-5)
        for u, v in zip(_bns(masked), _bns(packed)):
            torch.testing.assert_close(u.running_mean, v.running_mean, rtol=1e-5, atol=1e-6)
            torch.testing.assert_close(u.running_var, v.running_var, rtol=1e-5, atol=1e-6)
            assert int(u.num_batches_tracked) == int(v.num_batches_tracked) == step + 1
    # eval mode: the running statistics, row by row as without a mask
    masked.eval()
    packed.eval()
    with torch.no_grad():
        torch.testing.assert_close(masked(t, mask)[mask], packed(t[mask]), rtol=1e-5, atol=1e-5)


@pytest.mark.parametrize("offset", [10.0, 1000.0, 3000.0])
def test_masked_batch_norm_statistics_hold_far_from_zero_mean(offset):
    """inputs with |mean| far above their standard deviation: a one-pass E[x^2] - mean^2 variance cancels there"""
    r, c = 65536, 4
    g = torch.Generator().manual_seed(8)
    x = torch.randn(r, c, generator=g) + offset
    keep = (torch.arange(r) % 4 != 0).unsqueeze(1)  # 75 % real rows
    bn, ref = torch.nn.BatchNorm1d(c), torch.nn.BatchNorm1d(c)
    real_rows = x[keep.squeeze(1)]
    got = layers.masked_batch_norm(bn, torch.where(keep, x, 0), keep)[keep.squeeze(1)]
    want = ref(real_rows).detach()
    # float64 truth; float32 inputs this far from 0 are themselves quantised (ulp 2.4e-4 at 3000), so the bound is
    # BatchNorm1d's own float32 error, not a fixed tolerance
    x64 = real_rows.double()
    truth = (x64 - x64.mean(0)) / torch.sqrt(x64.var(0, unbiased=False) + ref.eps)
    own = float((want.double() - truth).abs().max())
    assert float((got.double() - truth).abs().max()) <= 4 * own + 1e-5, (offset, own)
    torch.testing.assert_close(bn.running_mean, ref.running_mean, rtol=1e-5, atol=1e-5)
    torch.testing.assert_close(bn.running_var, ref.running_var, rtol=1e-2, atol=1e-4)


def test_masked_shared_mlp_is_independent_of_the_padding():
    b, n, lengths = 4, 33, [33, 1, 20, 32]
    mask = row_mask(torch.tensor(lengths), n)
    res = []
    for padding in ("nan", "copy"):
        m = _mlp(3)
        t = _padded(b, n, 6, lengths, 4, padding).requires_grad_(True)
        out = m(t, mask)
        out.square().sum().backward()
        res.append([out.detach(), t.grad] + [p.grad for p in m.parameters()] + [x for bn in _bns(m) for x in (bn.running_mean, bn.running_var)])
    for a, c in zip(*res):
        assert torch.equal(a, c)
    assert torch.equal(res[0][0][~mask], torch.zeros_like(res[0][0][~mask]))
    assert torch.equal(res[0][1][~mask], torch.zeros_like(res[0][1][~mask])), "no gradient reaches the padding"


def test_shared_mlp_without_mask_is_the_plain_stack():
    t = torch.randn(2, 9, 1, 6)
    m = _mlp(5)
    ref = copy.deepcopy(m)
    got = m(t)
    want = ref.body(t.reshape(-1, 6)).reshape(2, 9, 1, 8)
    assert torch.equal(got, want)
    for u, v in zip(_bns(m), _bns(ref)):
        assert torch.equal(u.running_mean, v.running_mean) and torch.equal(u.running_var, v.running_var)


def test_row_mask_clamps_like_the_kernels():
    got = row_mask(torch.tensor([0, 3, 9, -2], dtype=torch.int32), 5)
    want = torch.tensor([[1, 0, 0, 0, 0], [1, 1, 1, 0, 0], [1, 1, 1, 1, 1], [1, 0, 0, 0, 0]], dtype=torch.bool)
    assert torch.equal(got, want)


def test_sem_seg_loss_ignores_the_padding_rows():
    b, n, k, lengths = 3, 10, 5, [10, 4, 7]
    g = torch.Generator().manual_seed(6)
    pred = torch.randn(b, n, k, generator=g)
    label = torch.randint(0, k, (b, n), generator=g)
    smpw = torch.rand(b, n, generator=g) + 0.1
    mask = row_mask(torch.tensor(lengths), n)
    want = nets.sem_seg_loss(pred[mask].unsqueeze(0), label[mask].unsqueeze(0), smpw[mask].unsqueeze(0))
    pred2, label2, smpw2 = pred.clone(), label.clone(), smpw.clone()
    pred2[~mask] = float("nan")
    label2[~mask] = 999  # not a class: must not be looked up
    smpw2[~mask] = 5.0
    for lengths_arg in (lengths, torch.tensor(lengths)):
        got = nets.sem_seg_loss(pred2, label2, smpw2, lengths=lengths_arg)
        torch.testing.assert_close(got, want, rtol=1e-6, atol=1e-7)
    assert torch.equal(nets.sem_seg_loss(pred, label, smpw, lengths=[n] * b), nets.sem_seg_loss(pred, label, smpw))
    # the gradient too: zero on the padding rows, finite everywhere, equal to the packed loss's on the real rows
    p2 = pred2.clone().requires_grad_(True)
    nets.sem_seg_loss(p2, label2, smpw2, lengths=lengths).backward()
    p = pred.clone().requires_grad_(True)
    nets.sem_seg_loss(p[mask].unsqueeze(0), label[mask].unsqueeze(0), smpw[mask].unsqueeze(0)).backward()
    assert bool(torch.isfinite(p2.grad).all())
    assert torch.equal(p2.grad[~mask], torch.zeros_like(p2.grad[~mask]))
    torch.testing.assert_close(p2.grad[mask], p.grad[mask], rtol=1e-6, atol=1e-7)


def test_lengths_are_validated():
    pred, label, smpw = torch.zeros(3, 10, 4), torch.zeros(3, 10, dtype=torch.long), torch.ones(3, 10)
    for bad in ([0, 5, 5], [5, 11, 5], [5, 5], [[5, 5, 5]], torch.tensor([5, -1, 5])):
        with pytest.raises(ValueError):
            nets.sem_seg_loss(pred, label, smpw, lengths=bad)
    with pytest.raises(TypeError):
        nets.sem_seg_loss(pred, label, smpw, lengths=[1.5, 2.0, 3.0])
    # a callable mlp cannot take the row mask: refused before any kernel runs
    x = torch.zeros(2, 16, 3)
    with pytest.raises(ValueError, match="SharedMLP"):
        pointnet_util.pointnet_fp_module(x, x[:, :4], None, torch.zeros(2, 4, 5), mlp=lambda t: t, lengths=[16, 8])


def test_lengths_is_a_keyword_of_the_new_surface():
    for fn in (tf_interpolate.three_nn, tf_interpolate.three_interpolate, tf_interpolate.three_nn_interpolate,
               tf_interpolate.fp_interpolate_concat):
        p = inspect.signature(fn).parameters["lengths"]
        assert p.kind == inspect.Parameter.KEYWORD_ONLY and p.default is None, fn.__name__
    for fn in (pointnet_util.pointnet_fp_module, nets.FeaturePropagation.forward, nets.PointNet2SemSeg.forward, nets.sem_seg_loss):
        assert inspect.signature(fn).parameters["lengths"].default is None, fn.__qualname__
    assert inspect.signature(SharedMLP.forward).parameters["mask"].default is None


RAGGED = ["pn2_three_nn_ragged", "pn2_three_nn_interpolate_ragged_typed", "pn2_fp_interpolate_concat_ragged_typed",
          "pn2_three_interpolate_ragged_typed", "pn2_three_interpolate_grad_ragged", "pn2_three_interpolate_grad_det_ragged_typed"]


def test_ragged_entries_are_declared_and_loaded():
    lib = _lib.load()
    for name in RAGGED:
        assert name in _lib.EXPORTED_SYMBOLS and hasattr(lib, name)


def test_ragged_entry_argument_errors_return_invalid_value_without_a_launch():
    import ctypes
    lib = _lib.load()
    fake, null = ctypes.c_void_p(256), ctypes.c_void_p(0)
    ws = lib.pn2_three_interpolate_grad_det_workspace_bytes(1, 8, 4)
    before = _lib.launch_count()
    calls = [
        lib.pn2_three_nn_ragged(1, 8, 4, null, fake, fake, fake, fake, None),
        lib.pn2_three_nn_ragged(-1, 8, 4, fake, fake, fake, fake, fake, None),
        lib.pn2_three_nn_ragged(65536, 8, 4, fake, fake, fake, fake, fake, None),
        lib.pn2_three_nn_interpolate_ragged_typed(3, 1, 8, 4, 2, fake, fake, fake, fake, fake, null, null, null, None),
        lib.pn2_three_nn_interpolate_ragged_typed(0, 1, 8, 0, 2, fake, fake, fake, fake, fake, null, null, null, None),
        lib.pn2_fp_interpolate_concat_ragged_typed(1, 1, 8, 4, 2, 3, fake, fake, fake, null, fake, fake, None),
        lib.pn2_fp_interpolate_concat_ragged_typed(0, 1, 8, 4, 0, 3, fake, fake, fake, fake, fake, fake, None),
        lib.pn2_three_interpolate_ragged_typed(7, 1, 4, 2, 8, fake, fake, fake, fake, fake, None),
        lib.pn2_three_interpolate_ragged_typed(0, 1, 0, 2, 8, fake, fake, fake, fake, fake, None),
        lib.pn2_three_interpolate_ragged_typed(2, 1, 4, 2, 8, fake, null, fake, fake, fake, None),
        lib.pn2_three_interpolate_grad_ragged(1, 8, 2, 4, fake, fake, null, fake, fake, None),
        lib.pn2_three_interpolate_grad_ragged(1, 8, 2, 0, fake, fake, fake, fake, fake, None),
        lib.pn2_three_interpolate_grad_det_ragged_typed(0, 1, 8, 2, 4, fake, fake, fake, fake, fake, fake, ws - 1, None),
        lib.pn2_three_interpolate_grad_det_ragged_typed(1, 1, 8, 2, 4, fake, fake, fake, fake, fake, null, ws, None),
        lib.pn2_three_interpolate_grad_det_ragged_typed(5, 1, 8, 2, 4, fake, fake, fake, fake, fake, fake, ws, None),
    ]
    assert calls == [1] * len(calls)
    assert _lib.launch_count() == before


class _Recorder:
    """stands in for the library: records the entry points called, returns 0 (success) from each"""

    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        def fn(*args):
            self.calls.append(name)
            return 64 if name.endswith("workspace_bytes") else 0
        return fn


@pytest.fixture
def recorder(monkeypatch):
    rec = _Recorder()
    monkeypatch.setattr(_lib, "load", lambda: rec)
    monkeypatch.setattr(tf_interpolate, "on_device", lambda t: mock.MagicMock())
    monkeypatch.setattr(tf_interpolate, "stream_ptr", lambda d: None)
    monkeypatch.setattr(tf_interpolate, "require_cuda", lambda t, name, dtype: t.contiguous())  # CPU tensors stand in
    yield rec
    torch.use_deterministic_algorithms(False)


@pytest.mark.parametrize("with_lengths", [False, True])
def test_each_op_calls_the_ragged_entry_exactly_when_given_lengths(recorder, monkeypatch, with_lengths):
    b, n, m, c = 2, 16, 4, 8
    lengths = [16, 5] if with_lengths else None
    xyz1, xyz2 = torch.zeros(b, n, 3), torch.zeros(b, m, 3)
    for dtype in (torch.float32, torch.bfloat16):
        p2, p1 = torch.zeros(b, m, c, dtype=dtype), torch.zeros(b, n, 3, dtype=dtype)
        recorder.calls.clear()
        tf_interpolate.three_nn(xyz1, xyz2, lengths=lengths)
        tf_interpolate.three_nn_interpolate(xyz1, xyz2, p2, lengths=lengths)
        tf_interpolate.fp_interpolate_concat(xyz1, xyz2, p1, p2, lengths=lengths)
        tf_interpolate.three_interpolate(p2, torch.zeros(b, n, 3, dtype=torch.int32), torch.zeros(b, n, 3), lengths=lengths)
        f32 = dtype == torch.float32
        if with_lengths:
            want = RAGGED[:4]
        else:
            want = ["pn2_three_nn", "pn2_three_nn_interpolate" if f32 else "pn2_three_nn_interpolate_typed",
                    "pn2_fp_interpolate_concat" if f32 else "pn2_fp_interpolate_concat_typed",
                    "pn2_three_interpolate" if f32 else "pn2_three_interpolate_typed"]
        assert recorder.calls == want, dtype
    # the backward routes, with the lengths saved next to idx and weight
    saved = (torch.zeros(b, n, 3, dtype=torch.int32), torch.zeros(b, n, 3))
    if with_lengths:
        saved = saved + (torch.tensor([16, 5], dtype=torch.int32),)
    for det, dtype, want in ((False, torch.float32, "pn2_three_interpolate_grad"), (True, torch.float32, "pn2_three_interpolate_grad_det"),
                             (False, torch.float16, "pn2_three_interpolate_grad_det_typed")):
        monkeypatch.setattr(tf_interpolate, "DETERMINISTIC_GRAD", det)
        ctx = mock.MagicMock(saved_tensors=saved, shape=(b, m, c), dtype=dtype)
        recorder.calls.clear()
        grads = tf_interpolate._ThreeInterpolate.backward(ctx, torch.zeros(b, n, c))
        assert len(grads) == 4 and grads[1:] == (None, None, None)
        if with_lengths:
            want = "pn2_three_interpolate_grad_ragged" if want == "pn2_three_interpolate_grad" else "pn2_three_interpolate_grad_det_ragged_typed"
        assert recorder.calls[-1] == want


def test_sem_seg_forward_passes_lengths_to_sa1_and_fp4_and_the_mask_to_the_head(monkeypatch):
    """the net's plumbing, with the geometry layers replaced by recorders on the CPU"""
    net = nets.PointNet2SemSeg(num_class=4).eval()
    b, n = 2, 12
    seen = {}

    def sa(self, xyz, points, lengths=None):
        seen.setdefault("sa", []).append(lengths)
        m = self.npoint
        return xyz[:, :m].contiguous(), torch.zeros(xyz.shape[0], m, self.mlp.out_channels), None

    def fp(self, xyz1, xyz2, points1, points2, lengths=None):
        seen.setdefault("fp", []).append(lengths)
        return torch.ones(xyz1.shape[0], xyz1.shape[1], self.out_channels)

    monkeypatch.setattr(nets.SetAbstraction, "forward", sa)
    monkeypatch.setattr(nets.FeaturePropagation, "forward", fp)
    for mod in (net.sa1, net.sa2, net.sa3, net.sa4):
        mod.npoint = 2
    x = torch.zeros(b, n, 3)
    logits, _ = net(x, lengths=[12, 5])
    assert seen["sa"][0].tolist() == [12, 5] and all(l is None for l in seen["sa"][1:])
    assert seen["fp"][-1].tolist() == [12, 5] and all(l is None for l in seen["fp"][:-1])
    assert torch.equal(logits[1, 5:], torch.zeros(n - 5, 4)) and logits[1, :5].abs().sum() > 0
