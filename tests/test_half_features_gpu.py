"""bfloat16 / float16 features in the grouping and interpolation ops, held bit for bit to the numerical contract
(DESIGN.md, "16-bit features"): gathered features are copies, everything computed is the float32 result rounded
once to the feature dtype, coordinates / weights / indices stay float32 / int32."""
import numpy as np
import pytest
import torch

from pointnet2_b200 import _lib, workloads as W
from pointnet2_b200.pointnet_util import group_and_concat, pointnet_fp_module, pointnet_sa_module_msg, sample_and_group
from pointnet2_b200.tf_grouping import group_point
from pointnet2_b200.tf_interpolate import fp_interpolate_concat, three_interpolate, three_nn, three_nn_interpolate

pytestmark = pytest.mark.gpu

DTYPES = [torch.bfloat16, torch.float16]
WIDTHS = [1, 3, 4, 8, 16, 64, 67, 128, 131, 259]


def T(a, dev):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


def bits(t):
    return t.contiguous().view(torch.int16)


def assert_bits_equal(got, want):
    assert got.dtype == want.dtype and got.shape == want.shape
    assert torch.equal(bits(got), bits(want))


def one_ulp_mask(got, want):
    gi, wi = bits(got).int(), bits(want).int()
    same_sign = (gi < 0) == (wi < 0)
    return (got.float() == want.float()) | (same_sign & ((gi - wi).abs() <= 1))


def assert_within_one_ulp(got, want):
    """got and want of the same 16-bit dtype differ by at most one unit in the last place."""
    assert got.dtype == want.dtype and got.shape == want.shape
    ok = one_ulp_mask(got, want)
    assert bool(ok.all()), f"{int((~ok).sum())} elements differ by more than one ulp"


def same(x, y):
    return x.dtype == y.dtype and torch.equal(bits(x) if x.dtype in DTYPES else x, bits(y) if y.dtype in DTYPES else y)


def features(b, n, c, dt, dev, seed, offset=0):
    """(b, n, c) features in dtype dt; offset=1 starts the tensor one element past an aligned base."""
    g = torch.Generator(device=dev).manual_seed(seed)
    flat = torch.randn(b * n * c + offset, device=dev, generator=g).to(dt)
    return flat[offset:].view(b, n, c)


@pytest.mark.parametrize("dt", DTYPES)
@pytest.mark.parametrize("c", WIDTHS)
@pytest.mark.parametrize("offset", [0, 1])
def test_group_point_copies_16bit_features(dev, dt, c, offset):
    b, n, m, s = 2, 300, 40, 24
    pts = features(b, n, c, dt, dev, 1, offset)
    if offset:
        assert pts.data_ptr() % 16 != 0
    idx = torch.randint(0, n, (b, m, s), device=dev, dtype=torch.int32, generator=torch.Generator(device=dev).manual_seed(2))
    out = group_point(pts, idx)
    want = pts[torch.arange(b, device=dev).view(b, 1, 1), idx.long()]
    assert_bits_equal(out, want)


def _ball_setup(dev, b=2, n=400, m=50, s=16, seed=3):
    xyz = T(W.cloud_uniform(b, n, seed), dev)
    new_xyz = xyz[:, :m].contiguous() + 0.01
    idx = torch.randint(0, n, (b, m, s), device=dev, dtype=torch.int32, generator=torch.Generator(device=dev).manual_seed(seed))
    return xyz, new_xyz, idx


@pytest.mark.parametrize("dt", DTYPES)
@pytest.mark.parametrize("c", WIDTHS)
@pytest.mark.parametrize("xyz_first", [True, False])
@pytest.mark.parametrize("offset", [0, 1])
def test_group_and_concat_16bit(dev, dt, c, xyz_first, offset):
    xyz, new_xyz, idx = _ball_setup(dev)
    pts = features(xyz.shape[0], xyz.shape[1], c, dt, dev, 4, offset)
    out, gxyz = group_and_concat(xyz, new_xyz, pts, idx, xyz_first=xyz_first)
    _, gxyz32 = group_and_concat(xyz, new_xyz, None, idx)
    assert gxyz.dtype == torch.float32 and torch.equal(gxyz, gxyz32)
    feats = group_point(pts, idx).float()
    want = torch.cat([gxyz32, feats] if xyz_first else [feats, gxyz32], -1).to(dt)
    assert_bits_equal(out, want)


def test_group_and_concat_without_points_stays_float32(dev):
    xyz, new_xyz, idx = _ball_setup(dev)
    for xyz_first in (True, False):
        out, gxyz = group_and_concat(xyz, new_xyz, None, idx, xyz_first=xyz_first)
        assert out.dtype == torch.float32
        want = xyz[torch.arange(2, device=dev).view(2, 1, 1), idx.long()] - new_xyz.unsqueeze(2)
        assert torch.equal(out, want) and torch.equal(gxyz, want)


def _interp_setup(dev, b=2, n=300, m=70, seed=5):
    x1, x2 = T(W.cloud_uniform(b, n, seed), dev), T(W.cloud_uniform(b, m, seed + 1), dev)
    d, i = three_nn(x1, x2)
    r = 1.0 / torch.clamp(d, min=1e-10)
    return x1, x2, i, r / r.sum(2, keepdim=True)


@pytest.mark.parametrize("dt", DTYPES)
@pytest.mark.parametrize("c", WIDTHS)
@pytest.mark.parametrize("offset", [0, 1])
def test_three_interpolate_16bit(dev, dt, c, offset):
    x1, x2, idx, w = _interp_setup(dev)
    pts = features(2, x2.shape[1], c, dt, dev, 6, offset)
    out = three_interpolate(pts, idx, w)
    assert_bits_equal(out, three_interpolate(pts.float(), idx, w).to(dt))


@pytest.mark.parametrize("dt", DTYPES)
@pytest.mark.parametrize("c", WIDTHS)
@pytest.mark.parametrize("offset", [0, 1])
def test_fp_front_end_16bit(dev, dt, c, offset):
    x1, x2, _, _ = _interp_setup(dev)
    p2 = features(2, x2.shape[1], c, dt, dev, 7, offset)
    p1 = features(2, x1.shape[1], c, dt, dev, 8, offset)
    out, d, i, w = three_nn_interpolate(x1, x2, p2, return_aux=True)
    out32, d32, i32, w32 = three_nn_interpolate(x1, x2, p2.float(), return_aux=True)
    assert_bits_equal(out, out32.to(dt))
    assert torch.equal(d, d32) and torch.equal(i, i32) and torch.equal(w, w32)
    cat = fp_interpolate_concat(x1, x2, p1, p2)
    assert_bits_equal(cat[..., :c], fp_interpolate_concat(x1, x2, None, p2.float()).to(dt))
    assert_bits_equal(cat[..., c:], p1)
    assert_bits_equal(fp_interpolate_concat(x1, x2, None, p2), out)


@pytest.mark.parametrize("dt", DTYPES)
@pytest.mark.parametrize("c", [3, 64, 131])
def test_three_interpolate_backward_is_the_rounded_float32_gradient(dev, dt, c):
    x1, x2, idx, w = _interp_setup(dev)
    pts = features(2, x2.shape[1], c, dt, dev, 9).requires_grad_(True)
    g = features(2, x1.shape[1], c, dt, dev, 10)
    three_interpolate(pts, idx, w).backward(g)
    p32 = pts.detach().float().requires_grad_(True)
    three_interpolate(p32, idx, w).backward(g.float())  # the deterministic float32 gradient
    assert pts.grad.dtype == dt
    assert_bits_equal(pts.grad, p32.grad.to(dt))


# Known points referenced by more than 256 (j, t) entries go to the long-list kernel (8 ordered partial sums): layers
# with fewer than 3 known points, and clouds of coincident points like cfg4's duplicates.  Each shape in a width that
# takes the 4-channel vector path and one that takes the scalar path.
LONG_LIST_CASES = [(3, 500, 1, 8, "U"), (3, 500, 1, 7, "U"), (2, 500, 2, 33, "U"), (2, 500, 2, 32, "U"),
                   (1, 20000, 5, 16, "U"), (1, 20000, 5, 15, "U"), (4, 8192, 1024, 128, "D"), (4, 8192, 1024, 129, "D")]


@pytest.mark.parametrize("dt", DTYPES)
@pytest.mark.parametrize("b,n,m,c,dist", LONG_LIST_CASES)
def test_three_interpolate_backward_long_lists(dev, dt, b, n, m, c, dist):
    x1 = T(W.DISTRIBUTIONS[dist](b, n, 31), dev)
    x2 = x1[:, :m].contiguous() if dist == "D" else T(W.cloud_uniform(b, m, 32), dev)
    d, idx = three_nn(x1, x2)
    r = 1.0 / torch.clamp(d, min=1e-10)
    w = r / r.sum(2, keepdim=True)
    counts = torch.stack([torch.bincount(idx[i].reshape(-1).long(), minlength=m) for i in range(b)])
    assert int(counts.max()) > 256  # the long-list kernel runs
    g = features(b, n, c, dt, dev, 33)
    # through the C entry, twice (run-to-run deterministic), against the float32 deterministic gradient rounded once
    lib = _lib.load()
    wsb = int(lib.pn2_three_interpolate_grad_det_workspace_bytes(b, n, m))
    ws = torch.empty(wsb, dtype=torch.uint8, device=dev)
    g32 = g.float()
    want32 = torch.empty((b, m, c), device=dev)
    assert lib.pn2_three_interpolate_grad_det(b, n, c, m, g32.data_ptr(), idx.data_ptr(), w.data_ptr(), want32.data_ptr(),
                                              ws.data_ptr(), wsb, None) == 0
    code = 1 if dt == torch.bfloat16 else 2
    runs = []
    for _ in range(2):
        got = torch.full((b, m, c), 7.0, dtype=dt, device=dev)
        assert lib.pn2_three_interpolate_grad_det_typed(code, b, n, c, m, g.data_ptr(), idx.data_ptr(), w.data_ptr(), got.data_ptr(),
                                                        ws.data_ptr(), wsb, None) == 0
        runs.append(got)
    assert_bits_equal(runs[0], runs[1])
    assert_bits_equal(runs[0], want32.to(dt))
    # and through autograd
    pts = features(b, m, c, dt, dev, 34).requires_grad_(True)
    three_interpolate(pts, idx, w).backward(g)
    assert_bits_equal(pts.grad, want32.to(dt))


def _group_grad_ref(g, idx, n):
    """float64 scatter-add of g (b, m, s, c) into (b, n, c), the sum of |g| and the number of terms per row."""
    b, m, s, c = g.shape
    flat = (torch.arange(b, device=g.device).view(b, 1, 1) * n + idx.long()).view(-1)

    def scatter(v):
        return torch.zeros((b * n, c), dtype=torch.float64, device=g.device).index_add_(0, flat, v.view(-1, c)).view(b, n, c)
    g64 = g.double()
    return scatter(g64), scatter(g64.abs()), scatter(torch.ones_like(g64))


def assert_rounded_sum(got, ref, absum, cnt):
    """got (16-bit) is within one ulp of the exact sum rounded — except where the terms cancel so far that the float32
    accumulation's own error (at most (cnt - 1) * 2^-24 * sum |g|) exceeds an ulp of the result."""
    ok = one_ulp_mask(got, ref.to(got.dtype))
    ok |= (got.double() - ref).abs() <= cnt * 2.0 ** -24 * absum + (ref.to(got.dtype).double() - ref).abs()
    assert bool(ok.all()), f"{int((~ok).sum())} elements off"


@pytest.mark.parametrize("dt", DTYPES)
@pytest.mark.parametrize("c", [3, 8, 67, 128])
def test_group_point_backward(dev, dt, c):
    b, n, m, s = 2, 120, 40, 16
    idx = torch.randint(0, n, (b, m, s), device=dev, dtype=torch.int32, generator=torch.Generator(device=dev).manual_seed(11))
    pts = features(b, n, c, dt, dev, 12).requires_grad_(True)
    # integer-valued gradients: every float32 sum is exact, so the result is exact
    gi = torch.randint(-8, 9, (b, m, s, c), device=dev, generator=torch.Generator(device=dev).manual_seed(13)).to(dt)
    group_point(pts, idx).backward(gi)
    assert pts.grad.dtype == dt
    assert_bits_equal(pts.grad, _group_grad_ref(gi, idx, n)[0].to(dt))
    p32 = pts.detach().float().requires_grad_(True)
    group_point(p32, idx).backward(gi.float())
    assert_bits_equal(pts.grad, p32.grad.to(dt))
    # general gradients: the exact sum rounded, up to one ulp and the float32 accumulation error
    pts.grad = None
    g = features(b, m * s, c, dt, dev, 14).view(b, m, s, c)
    group_point(pts, idx).backward(g)
    ref, absum, cnt = _group_grad_ref(g, idx, n)
    assert_rounded_sum(pts.grad, ref, absum, cnt)
    p32.grad = None
    group_point(p32, idx).backward(g.float())  # the float32 backward, rounded, meets the same bound
    assert_rounded_sum(p32.grad.to(dt), ref, absum, cnt)


@pytest.mark.parametrize("dt", DTYPES)
@pytest.mark.parametrize("xyz_first", [True, False])
def test_group_and_concat_backward(dev, dt, xyz_first):
    xyz, new_xyz, idx = _ball_setup(dev)
    c = 19
    grads = []
    for fdt in (dt, torch.float32):
        x = xyz.clone().requires_grad_(True)
        nx = new_xyz.clone().requires_grad_(True)
        p = features(2, xyz.shape[1], c, dt, dev, 15).to(fdt).requires_grad_(True)
        out, gxyz = group_and_concat(x, nx, p, idx, xyz_first=xyz_first)
        gi = torch.randint(-4, 5, out.shape, device=dev, generator=torch.Generator(device=dev).manual_seed(16)).to(out.dtype)
        (out.float() * gi.float()).sum().backward()
        grads.append((x.grad, nx.grad, p.grad))
    (gx, gnx, gp), (gx32, gnx32, gp32) = grads
    assert gx.dtype == gnx.dtype == torch.float32 and gp.dtype == dt
    assert torch.equal(gx, gx32) and torch.equal(gnx, gnx32)  # integer-valued: exact in every order
    assert_bits_equal(gp, gp32.to(dt))


@pytest.mark.parametrize("dt", DTYPES)
def test_sample_and_group_fused_equals_unfused(dev, dt):
    xyz = T(W.cloud_surface(2, 900, 17), dev)
    pts = features(2, 900, 13, dt, dev, 18)
    a = sample_and_group(100, 0.25, 24, xyz, pts, fused=True)
    u = sample_and_group(100, 0.25, 24, xyz, pts, fused=False)
    assert a[1].dtype == u[1].dtype == dt
    for x, y in zip(a, u):
        assert same(x, y)


@pytest.mark.parametrize("dt", DTYPES)
def test_msg_module_fused_equals_unfused(dev, dt):
    xyz = T(W.cloud_surface(2, 512, 19), dev)
    pts = features(2, 512, 9, dt, dev, 20)
    _, f = pointnet_sa_module_msg(xyz, pts, 64, [0.2, 0.4], [16, 32])
    _, u = pointnet_sa_module_msg(xyz, pts, 64, [0.2, 0.4], [16, 32], fused=False)
    assert f.dtype == dt
    assert_bits_equal(f, u)


@pytest.mark.parametrize("dt", DTYPES)
def test_fp_module_fused_equals_unfused(dev, dt):
    x1, x2 = T(W.cloud_uniform(2, 256, 21), dev), T(W.cloud_uniform(2, 64, 22), dev)
    p1, p2 = features(2, 256, 6, dt, dev, 23), features(2, 64, 32, dt, dev, 24)
    f = pointnet_fp_module(x1, x2, p1, p2)
    u = pointnet_fp_module(x1, x2, p1, p2, fused=False)
    assert f.dtype == u.dtype == dt
    assert_bits_equal(f[..., 32:], u[..., 32:])
    # the float32 weights of the fused kernel and of the unfused torch expression agree to ~1e-7 (the float32 test
    # holds them to 1e-5), so after rounding to 16 bits the interpolated channels agree to the last place
    assert_within_one_ulp(f[..., :32], u[..., :32])
    # mixed dtypes are not fused: the concatenation promotes
    assert pointnet_fp_module(x1, x2, p1.float(), p2).dtype == torch.float32


# ---- beyond 2^31 elements: the 64-bit indexing paths with 2-byte elements -----------------------------------
def _need(dev, gib):
    free, _ = torch.cuda.mem_get_info(dev)
    if free < gib * (1 << 30):
        pytest.skip(f"needs {gib} GiB of free device memory")


def _sample_rows(total_rows, dev, k=200000):
    g = torch.Generator(device=dev).manual_seed(7)
    return torch.cat([torch.randint(0, total_rows, (k,), device=dev, generator=g),
                      torch.arange(0, 1000, device=dev), torch.arange(total_rows - 1000, total_rows, device=dev)])


@pytest.mark.parametrize("c", [520, 515])  # 16-byte vector path and the odd-width row kernel
def test_group_point_bf16_beyond_2_to_31_elements(dev, c):
    _need(dev, 24)
    b, n, m, s = 4, 1536, 16384, 128
    g = torch.Generator(device=dev).manual_seed(1)
    points = torch.randn((b, n, c), device=dev, generator=g).to(torch.bfloat16)
    idx = torch.randint(0, n, (b, m, s), device=dev, generator=g, dtype=torch.int32)
    out = group_point(points, idx)
    assert out.numel() > (1 << 32)
    rows = _sample_rows(b * m * s, dev)
    assert torch.equal(bits(out.view(-1, c)[rows]), bits(points[rows // (m * s), idx.view(-1)[rows].long()]))
    del out


# The gradient's 64-bit instances: the 4-channel vector kernel needs 2^31 vectors (c = 520, S = 256: 8.7e9 elements,
# 17 GB of bf16), the scalar kernel 2^31 elements (c = 515, S = 128).  A gradient of ones makes the float32 sums exact
# counts, checked everywhere without a second 17 GB reference.
@pytest.mark.parametrize("c,s", [(520, 256), (515, 128)])
def test_group_point_grad_bf16_beyond_2_to_31(dev, c, s):
    _need(dev, 24)
    b, n, m = 4, 1536, 16384
    lanes = 4 if c % 4 == 0 else 1
    assert b * m * s * c // lanes >= (1 << 31)
    idx = torch.randint(0, n, (b, m, s), device=dev, generator=torch.Generator(device=dev).manual_seed(4), dtype=torch.int32)
    grad_out = torch.ones((b, m, s, c), dtype=torch.bfloat16, device=dev)
    accum = torch.zeros((b, n, c), dtype=torch.float32, device=dev)
    gp = torch.empty((b, n, c), dtype=torch.bfloat16, device=dev)
    rc = _lib.load().pn2_group_point_grad_typed(1, b, n, c, m, s, grad_out.data_ptr(), idx.data_ptr(), gp.data_ptr(), accum.data_ptr(), None)
    assert rc == 0
    del grad_out
    counts = torch.bincount((torch.arange(b, device=dev).view(b, 1, 1) * n + idx.long()).view(-1), minlength=b * n)
    assert torch.equal(accum.view(b * n, c), counts.float().view(-1, 1).expand(-1, c))
    assert torch.equal(gp, accum.to(torch.bfloat16))


def test_group_concat_bf16_beyond_2_to_31_elements(dev):
    _need(dev, 24)
    b, n, c, m, s = 4, 1536, 512, 16384, 128
    g = torch.Generator(device=dev).manual_seed(2)
    xyz = torch.rand((b, n, 3), device=dev, generator=g)
    new_xyz = torch.rand((b, m, 3), device=dev, generator=g)
    points = torch.randn((b, n, c), device=dev, generator=g).to(torch.bfloat16)
    idx = torch.randint(0, n, (b, m, s), device=dev, generator=g, dtype=torch.int32)
    out, gxyz = group_and_concat(xyz, new_xyz, points, idx, xyz_first=False)
    assert out.numel() > (1 << 32)
    rows = _sample_rows(b * m * s, dev)
    cloud, src = rows // (m * s), idx.view(-1)[rows].long()
    want_xyz = xyz[cloud, src] - new_xyz.view(-1, 3)[rows // s]
    got = out.view(-1, c + 3)[rows]
    assert torch.equal(bits(got[:, :c]), bits(points[cloud, src]))
    assert torch.equal(bits(got[:, c:]), bits(want_xyz.to(torch.bfloat16)))
    assert torch.equal(gxyz.view(-1, 3)[rows], want_xyz)


@pytest.mark.parametrize("c", [1032, 1031])  # 4-channel vectors and the scalar kernel
def test_three_interpolate_bf16_beyond_2_to_31_elements(dev, c):
    _need(dev, 24)
    b, n, m = 2, 1 << 21, 512
    g = torch.Generator(device=dev).manual_seed(3)
    points = torch.randn((b, m, c), device=dev, generator=g).to(torch.bfloat16)
    idx = torch.randint(0, m, (b, n, 3), device=dev, generator=g, dtype=torch.int32)
    w = torch.rand((b, n, 3), device=dev, generator=g)
    w = w / w.sum(dim=2, keepdim=True)
    out = three_interpolate(points, idx, w)
    assert out.numel() > (1 << 32)
    rows = _sample_rows(b * n, dev)
    cloud = rows // n
    ii, ww = idx.view(-1, 3)[rows].long(), w.view(-1, 3)[rows]
    p = points.float()
    want = (p[cloud, ii[:, 0]] * ww[:, 0:1] + p[cloud, ii[:, 1]] * ww[:, 1:2]) + p[cloud, ii[:, 2]] * ww[:, 2:3]
    assert torch.equal(bits(out.view(-1, c)[rows]), bits(want.to(torch.bfloat16)))
