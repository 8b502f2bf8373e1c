"""layers.sa_mlp_max (csrc/sa_mlp.cu), the inference tail of a set-abstraction level in one kernel, on the GPU: against
the torch layers evaluated in float64 on the same indices, for every level shape of the five networks; against the
composition the modules ran before (fused=False); bit-for-bit invariance to the batch; odd shapes; NaN and inf; and the
routing of pointnet_sa_module / pointnet_sa_module_msg."""
import copy

import pytest
import torch

from pointnet2_b200 import nets, scene
from pointnet2_b200 import workloads as W
from pointnet2_b200.layers import SharedMLP, sa_mlp_max
from pointnet2_b200.pointnet_util import pointnet_sa_module, pointnet_sa_module_msg

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")


@pytest.fixture(autouse=True)
def _no_tf32():
    """float32 products stay float32 in the torch layers the kernel is compared with"""
    old = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = old


def _mlp(cin, widths, seed, **kw):
    """an eval-mode SharedMLP with non-trivial biases, running statistics and affine parameters"""
    g = torch.Generator().manual_seed(seed)
    m = SharedMLP(cin, widths, **kw)
    with torch.no_grad():
        for mod in m.body:
            if isinstance(mod, torch.nn.Linear):
                mod.bias.copy_(torch.randn(mod.bias.shape, generator=g) * 0.1)
            elif isinstance(mod, torch.nn.BatchNorm1d):
                mod.running_mean.copy_(torch.randn(mod.num_features, generator=g) * 0.1)
                mod.running_var.copy_(torch.rand(mod.num_features, generator=g) + 0.5)
                mod.weight.copy_(torch.rand(mod.num_features, generator=g) + 0.5)
                mod.bias.copy_(torch.randn(mod.num_features, generator=g) * 0.1)
    return m.to(DEV).eval()


def _inputs(b, n, s, k, c, seed, dtype=torch.float32):
    xyz = torch.from_numpy(W.cloud_uniform(b, n, seed)).to(DEV)
    points = None if c == 0 else torch.from_numpy(W.features(b, n, c, seed + 1)).to(DEV).to(dtype)
    g = torch.Generator().manual_seed(seed + 2)
    idx = torch.randint(0, n, (b, s, k), generator=g, dtype=torch.int32).to(DEV)
    return xyz, xyz[:, :s].contiguous(), points, idx


def _rows(xyz, new_xyz, points, idx, xyz_first, use_xyz):
    """the grouped rows as the composition builds them: float32 differences, features in their own dtype"""
    b = xyz.shape[0]
    if idx is None:
        gx, gp = xyz.unsqueeze(1), None if points is None else points.unsqueeze(1)
    else:
        bi = torch.arange(b, device=xyz.device).view(b, 1, 1)
        gx = xyz[bi, idx.long()] - new_xyz.unsqueeze(2)
        gp = None if points is None else points[bi, idx.long()]
    if gp is None:
        return gx
    if not use_xyz:
        return gp
    return torch.cat([gx.to(gp.dtype), gp] if xyz_first else [gp, gx.to(gp.dtype)], dim=-1)


def _float64(mlp, rows):
    with torch.no_grad():
        return copy.deepcopy(mlp).double()(rows.double()).max(dim=2).values


def _scaled_err(got, want):
    return ((got.double() - want).abs().max() / want.abs().max().clamp_min(1e-30)).item()


# (name, n, s, k, c, widths, xyz_first, use_xyz, group_all): the set-abstraction levels of nets.py
LEVELS = [
    ("sem_seg.sa1", 2048, 256, 32, 0, [32, 32, 64], True, True, False),
    ("sem_seg.sa2", 1024, 128, 32, 64, [64, 64, 128], True, True, False),
    ("sem_seg.sa3", 256, 64, 32, 128, [128, 128, 256], True, True, False),
    ("sem_seg.sa4", 64, 16, 32, 256, [256, 256, 512], True, True, False),
    ("cls_ssg.sa1", 1024, 128, 32, 0, [64, 64, 128], True, True, False),
    ("cls_ssg.sa2", 512, 64, 64, 128, [128, 128, 256], True, True, False),
    ("cls_ssg.sa3", 128, 1, 128, 256, [256, 512, 1024], True, True, True),
    ("cls_msg.sa1a", 1024, 128, 16, 0, [32, 32, 64], False, True, False),
    ("cls_msg.sa1c", 1024, 64, 128, 0, [64, 96, 128], False, True, False),
    ("cls_msg.sa2c", 512, 32, 128, 320, [128, 128, 256], False, True, False),
    ("cls_msg.sa3", 128, 1, 128, 640, [256, 512, 1024], True, True, True),
    ("part_seg.sa1", 1024, 128, 64, 3, [64, 64, 128], True, True, False),
    ("part_seg_msg.sa1b", 1024, 64, 64, 3, [64, 64, 128], False, True, False),
    ("part_seg_msg.sa2b", 512, 32, 128, 320, [128, 196, 256], False, True, False),
    ("part_seg_msg.sa3", 128, 1, 128, 512, [256, 512, 1024], True, True, True),
    ("features_only", 512, 64, 32, 64, [64, 64, 128], True, False, False),
]

# Largest |kernel - float64| over a level's outputs, relative to the largest |output| of the level.  float32: the sums
# are float32 fused multiply-adds (observed at most 6.5e-7).  16 bits: one rounding to 8 (bfloat16) or 11 (float16) bits of
# mantissa per layer plus the rounded weights (observed at most 7.3e-3 in bfloat16).
F64_BOUNDS = {torch.float32: 5e-6, torch.bfloat16: 3e-2, torch.float16: 4e-3}


@pytest.mark.parametrize("level", LEVELS, ids=[l[0] for l in LEVELS])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.float16], ids=["f32", "bf16", "f16"])
def test_against_float64(level, dtype):
    name, n, s, k, c, widths, xyz_first, use_xyz, group_all = level
    xyz, new_xyz, points, idx = _inputs(2, n, s, k, c, 11 + len(name), dtype)
    if group_all:
        new_xyz = idx = None
    cin = c + 3 if (use_xyz or c == 0) else c
    mlp = _mlp(cin, widths, 5 + len(name))
    # without features the arithmetic type comes from autocast
    with torch.no_grad(), torch.autocast("cuda", dtype=dtype, enabled=c == 0 and dtype != torch.float32):
        got = sa_mlp_max(xyz, new_xyz, points, idx, mlp, xyz_first, use_xyz)
    assert got.dtype == dtype and got.shape == (2, 1 if group_all else s, widths[-1])
    rows = _rows(xyz, new_xyz, points, idx, xyz_first, use_xyz)
    want = _float64(mlp, rows)
    err = _scaled_err(got, want)
    print(f"{name} {dtype}: scaled error {err:.3g}")
    assert err <= F64_BOUNDS[dtype], (name, err)
    if dtype != torch.float32:
        # no further from float64 than the torch layers under autocast (which round after the Linear and after the
        # batch norm): compared on the mean error, with 10 % for the scatter of one draw
        with torch.no_grad(), torch.autocast("cuda", dtype=dtype):
            auto = mlp(rows).max(dim=2).values
        assert auto.dtype == dtype
        mine, theirs = (got.double() - want).abs().mean().item(), (auto.double() - want).abs().mean().item()
        assert mine <= 1.1 * theirs, (name, mine, theirs)


def test_module_against_composition():
    xyz, _, points, _ = _inputs(4, 2048, 1, 1, 64, 3)
    mlp = _mlp(67, [64, 64, 128], 8)
    with torch.no_grad():
        a = pointnet_sa_module(xyz, points, 256, 0.2, 32, mlp, fused=True)
        b = pointnet_sa_module(xyz, points, 256, 0.2, 32, mlp, fused=False)
    assert torch.equal(a[0], b[0]) and torch.equal(a[2], b[2])
    torch.testing.assert_close(a[1], b[1], rtol=1e-5, atol=1e-5)
    msg = [_mlp(67, w, 9 + i) for i, w in enumerate([[32, 32, 64], [64, 96, 128]])]
    with torch.no_grad():
        a = pointnet_sa_module_msg(xyz, points, 128, [0.1, 0.2], [16, 32], msg, fused=True)
        b = pointnet_sa_module_msg(xyz, points, 128, [0.1, 0.2], [16, 32], msg, fused=False)
    assert torch.equal(a[0], b[0])
    torch.testing.assert_close(a[1], b[1], rtol=1e-5, atol=1e-5)
    # group_all, and mlp2 on the pooled tensor
    mlp3, post = _mlp(67, [64, 128], 12), _mlp(128, [32], 13)
    x, p = xyz[:, :128].contiguous(), points[:, :128].contiguous()
    with torch.no_grad():
        a = pointnet_sa_module(x, p, None, None, None, mlp3, post, group_all=True, fused=True)
        b = pointnet_sa_module(x, p, None, None, None, mlp3, post, group_all=True, fused=False)
    assert torch.equal(a[0], b[0]) and torch.equal(a[2], b[2]) and a[1].shape == (4, 1, 32)
    torch.testing.assert_close(a[1], b[1], rtol=1e-5, atol=1e-5)


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16], ids=["f32", "bf16"])
def test_bits_do_not_depend_on_the_batch(dtype):
    xyz, new_xyz, points, idx = _inputs(16, 1024, 128, 32, 64, 21, dtype)
    mlp = _mlp(67, [64, 64, 128], 22)
    with torch.no_grad():
        full = sa_mlp_max(xyz, new_xyz, points, idx, mlp)
        assert torch.equal(full, sa_mlp_max(xyz, new_xyz, points, idx, mlp))
        for i in (0, 7, 15):
            alone = sa_mlp_max(xyz[i:i + 1], new_xyz[i:i + 1], points[i:i + 1], idx[i:i + 1], mlp)
            assert torch.equal(alone[0], full[i]), i


def test_ragged_batch_with_nan_padding_equals_each_cloud_alone():
    lengths = [1024, 700, 333, 901]
    xyz, _, points, _ = _inputs(4, 1024, 1, 1, 32, 31)
    for i, l in enumerate(lengths):
        xyz[i, l:] = float("nan")
        points[i, l:] = float("nan")
    mlp = _mlp(35, [32, 48], 32)
    with torch.no_grad():
        _, full, _ = pointnet_sa_module(xyz, points, 128, 0.2, 32, mlp, lengths=torch.tensor(lengths, device=DEV))
        assert torch.isfinite(full).all()
        for i, l in enumerate(lengths):
            _, alone, _ = pointnet_sa_module(xyz[i:i + 1, :l].contiguous(), points[i:i + 1, :l].contiguous(), 128, 0.2, 32, mlp)
            assert torch.equal(alone[0], full[i]), i


def test_msg_slices_equal_separate_scales():
    xyz, new_xyz, points, _ = _inputs(3, 512, 64, 1, 16, 41)
    ks, mlps = [16, 32, 128], [_mlp(19, w, 42 + i) for i, w in enumerate([[32, 64], [64, 128], [64, 96, 100]])]
    g = torch.Generator().manual_seed(43)
    idxs = [torch.randint(0, 512, (3, 64, k), generator=g, dtype=torch.int32).to(DEV) for k in ks]
    out = torch.full((3, 64, 64 + 128 + 100), float("nan"), device=DEV)
    with torch.no_grad():
        lo, parts = 0, []
        for idx, m in zip(idxs, mlps):
            sa_mlp_max(xyz, new_xyz, points, idx, m, False, True, out=out[..., lo:lo + m.out_channels])
            parts.append(sa_mlp_max(xyz, new_xyz, points, idx, m, False, True))
            lo += m.out_channels
    assert torch.equal(out, torch.cat(parts, dim=-1))


ODD = [  # (k, s, c, widths, kwargs)
    (1, 7, 4, [7, 13], {}),
    (5, 1, 0, [7, 13], {}),
    (33, 9, 1, [16], {}),
    (200, 3, 5, [8, 9, 10, 11], {}),
    (20, 6, 1, [12, 5], {"bn": False}),
    (2, 5, 9, [12, 6], {"last_activation": False}),
]


@pytest.mark.parametrize("case", ODD, ids=[f"k{c[0]}_s{c[1]}_c{c[2]}_l{len(c[3])}" for c in ODD])
@pytest.mark.parametrize("dtype", [torch.float32, torch.float16], ids=["f32", "f16"])
def test_odd_shapes(case, dtype):
    k, s, c, widths, kw = case
    xyz, new_xyz, points, idx = _inputs(3, 256, s, k, c, 51 + k, dtype)
    use_xyz = c != 1  # c == 1: the features alone, a one-channel input
    mlp = _mlp(c + 3 if use_xyz or c == 0 else c, widths, 52 + k, **kw)
    with torch.no_grad(), torch.autocast("cuda", dtype=dtype, enabled=c == 0 and dtype != torch.float32):
        got = sa_mlp_max(xyz, new_xyz, points, idx, mlp, True, use_xyz)
    assert got.dtype == dtype
    want = _float64(mlp, _rows(xyz, new_xyz, points, idx, True, use_xyz))
    assert _scaled_err(got, want) <= F64_BOUNDS[dtype]
    if kw.get("last_activation") is False:
        assert (got < 0).any()  # no ReLU on the last layer: negative maxima survive


def test_empty_batch_launches_nothing():
    from pointnet2_b200 import _lib
    mlp = _mlp(3, [8], 61)
    xyz = torch.zeros(0, 16, 3, device=DEV)
    before = _lib.launch_count()
    with torch.no_grad():
        a = sa_mlp_max(xyz, torch.zeros(0, 4, 3, device=DEV), None, torch.zeros(0, 4, 2, dtype=torch.int32, device=DEV), mlp)
        x1 = torch.zeros(2, 16, 3, device=DEV)
        b = sa_mlp_max(x1, torch.zeros(2, 0, 3, device=DEV), None, torch.zeros(2, 0, 2, dtype=torch.int32, device=DEV), mlp)
    assert a.shape == (0, 4, 8) and b.shape == (2, 0, 8) and _lib.launch_count() == before


def test_nan_and_inf():
    xyz, new_xyz, points, _ = _inputs(2, 256, 8, 1, 16, 71)
    # disjoint groups, so that one poisoned point sits in exactly one of them
    idx = torch.arange(2 * 8 * 32, dtype=torch.int32, device=DEV).view(2, 8, 32) % 256
    mlp = _mlp(19, [32, 32], 72)
    with torch.no_grad():
        clean = sa_mlp_max(xyz, new_xyz, points, idx, mlp)
        bad = points.clone()
        bad[1, idx[1, 3, 5].item(), 2] = float("nan")
        got = sa_mlp_max(xyz, new_xyz, bad, idx, mlp)
        assert torch.isnan(got[1, 3]).all()
        keep = torch.ones(2, 8, dtype=torch.bool, device=DEV)
        keep[1, 3] = False
        assert torch.equal(got[keep], clean[keep])
        # one layer, so that no inf - inf arises: +inf reaches the channels whose weight on that input is positive
        one = _mlp(19, [32], 73)
        inf = points.clone()
        inf[0, idx[0, 2, 9].item(), 4] = float("inf")
        got = sa_mlp_max(xyz, new_xyz, inf, idx, one)
        want = one(_rows(xyz, new_xyz, inf, idx, True, True)).max(dim=2).values
    assert torch.isinf(got[0, 2]).any() and not torch.isnan(got).any()
    assert torch.equal(torch.isinf(got), torch.isinf(want))
    finite = ~torch.isinf(want)
    torch.testing.assert_close(got[finite], want[finite], rtol=1e-5, atol=1e-5)


def test_routing_keeps_the_torch_layers_elsewhere():
    xyz, _, points, _ = _inputs(2, 512, 1, 1, 8, 81)
    mlp = _mlp(11, [16, 24], 82)
    fired = []
    h = mlp.body[0].register_forward_hook(lambda m, i, o: fired.append(1))

    def both(**kw):
        fired.clear()
        a = pointnet_sa_module(xyz, points, 64, 0.3, 16, mlp, fused=True, **kw)
        n = len(fired)
        b = pointnet_sa_module(xyz, points, 64, 0.3, 16, mlp, fused=False, **kw)
        return a[1], b[1], n

    try:
        with torch.no_grad():
            a, b, n = both()
            assert n == 0  # the kernel, not the Linear
            a, b, n = both(pooling="avg")
            assert n == 1 and torch.equal(a, b)
        a, b, n = both()  # grad mode on
        assert n == 1 and torch.equal(a, b) and a.requires_grad
        mlp.train()
        with torch.no_grad():
            state = copy.deepcopy(mlp.state_dict())
            a, _, n = both()
            mlp.load_state_dict(state)
            fired.clear()
            b = pointnet_sa_module(xyz, points, 64, 0.3, 16, mlp, fused=False)[1]
            assert n == 1 and torch.equal(a, b)
    finally:
        h.remove()


def test_predict_scene_sa_outputs_do_not_depend_on_batch_size():
    torch.manual_seed(5)
    net = nets.PointNet2SemSeg(21).to(DEV)
    with torch.no_grad():
        for _ in range(2):
            net(torch.rand(4, 2048, 3, device=DEV) * 1.5)  # running statistics away from their initial values
    net.eval()
    xyz = torch.from_numpy(W.scene_room(40000, 9)[0]).to(DEV)
    levels = ("sa1", "sa2", "sa3", "sa4")
    seen = {k: [] for k in levels}
    hooks = [getattr(net, k).register_forward_hook(lambda m, i, o, k=k: seen[k].append(o[1].clone())) for k in levels]
    try:
        scene.predict_scene(net, xyz, batch_size=16, max_points=2048)
        big = {k: torch.cat(v) for k, v in seen.items()}
        for v in seen.values():
            v.clear()
        scene.predict_scene(net, xyz, batch_size=1, max_points=2048)
        one = {k: torch.cat(v) for k, v in seen.items()}
    finally:
        for h in hooks:
            h.remove()
    assert big["sa1"].shape[0] > 16
    for k in levels:
        assert torch.equal(big[k], one[k]), k
