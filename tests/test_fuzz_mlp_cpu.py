"""Without a GPU: the tile planners of the fused inference MLP kernels restated (tests/mlp_oracle.py) and searched for
the plans legal shapes reach; the fixed-seed slice of tests/fuzz_mlp_gpu.py reaches every reachable planner branch;
the float32 C restatement (oracle_mlp_rows_f32) on hand cases and against float64; and the 16-bit bound, sound on a
CPU model of the 16-bit kernel and tight enough to reject the defects it is meant to catch."""
import collections
import itertools

import numpy as np
import pytest
import torch

import fuzz_mlp_gpu as F
import mlp_oracle as MO
import numerics as NUM
from oracle import oracle as O


# ----------------------------------------------------------------------------------------------------- planners
def test_planner_hand_values():
    # the set-abstraction levels DESIGN.md §6.13 names: [256, 512, 1024] on 643 inputs plans TM 32 in float32, 64 in
    # 16 bits; [512, 1024] on 1027 inputs at K 64 misses TM 32 by 128 bytes in float32
    assert MO.sa_plan(4, 643, [256, 512, 1024], 128)["tm"] == 32
    assert MO.sa_plan(2, 643, [256, 512, 1024], 128)["tm"] == 64
    assert MO.sa_smem(4, 1027, [512, 1024], 32, 1) == MO.SMEM_LIMIT + 128
    p = MO.sa_plan(4, 1027, [512, 1024], 64, groups=5)
    assert (p["tm"], p["slots"], p["pieces"], p["grid"]) == (16, 1, 4, 5)
    # K = 1 with a 1024-wide last layer: 64 slots do not fit, the loop trims them
    p = MO.sa_plan(4, 3, [1024], 1, groups=100)
    assert p["tm"] == 64 and p["trimmed"] and p["slots"] == 45 and p["grid"] == 3
    p = MO.sa_plan(2, 3, [1024], 1, groups=100)
    assert p["tm"] == 64 and p["trimmed"] and p["slots"] == 47
    # K = 5 on a 64-row tile: 12 groups, 4 rows unused
    assert MO.sa_plan(4, 67, [64, 64, 128], 5)["slots"] == 12
    # PointNet2PartSegMSG.fp1 (1536 inputs): TM 16 in float32, 32 in 16 bits
    p = MO.row_plan(4, 1536, [256, 256], rows=4096)
    assert p["tm"] == 16 and p["grid"] == 256 and p["smem"] == 135744
    assert MO.row_plan(2, 1536, [256, 256])["tm"] == 32


def _stacks(pool):
    for nl in range(1, MO.MAX_LAYERS + 1):
        yield from (list(w) for w in itertools.product(pool, repeat=nl))


@pytest.fixture(scope="module")
def reachable():
    """(kind, element size) -> the TMs legal shapes plan, over every stack of 1-4 layers from widths around the
    strides' and passes' steps and first-layer widths up to each kernel's limit.  The tile depends on the widths
    alone (slots are trimmed after it is chosen), and the shared memory grows with every width, so the largest
    legal shape bounds the search from above."""
    pool = [1, 32, 33, 64, 65, 512, 513, 1023, 1024]
    seen = collections.defaultdict(set)
    for esize in (4, 2):
        for widths in _stacks(pool):
            for cin in (1, 33, 259, 513, 1024, MO.SA_MAX_IN):
                seen["sa", esize].add(MO.sa_plan(esize, cin, widths, 1)["tm"])
            for cin in (1, 33, 513, 1024, 1027, 1280, MO.ROW_MAX_IN):
                seen["rows", esize].add(MO.row_plan(esize, cin, widths)["tm"])
    return seen


def test_every_legal_shape_plans_a_tile_and_16_bit_tm16_is_dead(reachable):
    assert reachable["sa", 4] == {64, 32, 16} and reachable["rows", 4] == {64, 32, 16}
    # bfloat16 / float16 stacks always fit TM = 32: the TM = 16 instantiations of both kernels are never launched
    assert reachable["sa", 2] == {64, 32} and reachable["rows", 2] == {64, 32}
    for esize in (4, 2):
        top = [MO.MAX_WIDTH] * MO.MAX_LAYERS
        assert MO.sa_plan(esize, MO.SA_MAX_IN, top, 1) is not None  # 1027 -> [1024] x 4 at K = 1
        assert MO.row_plan(esize, MO.ROW_MAX_IN, top) is not None   # 1536 -> [1024] x 4
        # monotone: the widest legal shape at TM 32 bounds every other one
        worst_tm32 = MO.sa_smem(esize, MO.SA_MAX_IN, top, 32, 1), MO.row_smem(esize, MO.ROW_MAX_IN, top, 32)
        assert all(s <= MO.SMEM_LIMIT for s in worst_tm32) == (esize == 2)
    assert MO.sa_plan(2, MO.SA_MAX_IN, [MO.MAX_WIDTH] * 4, 1)["trimmed"]  # 16-bit slot trimming at the extreme


# ------------------------------------------------------------------------------------------------- fuzz slice
@pytest.fixture(scope="module")
def slice_params():
    return {seed: F.draws(seed, F.SLICE_ITERATIONS) for seed in F.SLICE_SEEDS}


REQUIRED_BRANCHES = {
    "sa_e4_tm64", "sa_e4_tm32", "sa_e4_tm16", "sa_e2_tm64", "sa_e2_tm32",
    "sa_pieces_tm64", "sa_pieces_tm32", "sa_pieces_tm16", "sa_partial_piece",
    "sa_groups_tm64", "sa_groups_tm32", "sa_k_ndiv_tm", "sa_trimmed_e4", "sa_trimmed_e2",
    "sa_partial_pass", "sa_cin_off_slab", "sa_four_layers",
    "rows_e4_tm64", "rows_e4_tm32", "rows_e4_tm16", "rows_e2_tm64", "rows_e2_tm32",
    "rows_partial_pass", "rows_cin_off_slab", "rows_four_layers", "rows_partial_tile",
}


def features(p):
    """the non-planner regimes one case reaches"""
    tags = {f"{p['case']}_{p['fmt']}"}
    if p["autocast"]:
        tags.add(f"{p['case']}_autocast")
    if p.get("slice"):
        tags.add(f"{p['case']}_out_slice")
    if p.get("nonfinite"):
        tags.add(f"{p['case']}_nonfinite")
    bns = set(p["bn"])
    tags |= {f"bn_{b}" for b in bns}
    if not p["relu"][-1]:
        tags.add("last_no_relu")
    for L in p["layers"]:
        if "gamma" in L and (L["gamma"] < 0).any():
            tags.add("negative_gamma")
        if "var" in L and L["var"].min() < 1e-3:
            tags.add("small_var")
        if "var" in L and L["var"].max() > 5:
            tags.add("large_var")
        if L.get("eps") == 1e-5:
            tags.add("eps_1e-5")
    if p["case"] == "sa":
        if p["group_all"]:
            tags.add("sa_group_all")
        if p["autocast"] and p["c"] == 0:
            tags.add("sa_autocast_no_features")
        tags.add(f"sa_xyz_first_{p['xyz_first']}")
        if not p["use_xyz"]:
            tags.add("sa_features_only")
        if p["c"] in (0, 1):
            tags.add(f"sa_c{p['c']}")
    if p["case"] == "fp":
        tags.add("fp_ragged" if p["lengths"] else "fp_dense")
        if p["c1"] == 0:
            tags.add("fp_c1_0")
    if p["case"] == "rows" and p["mask"] is not None:
        tags.add("rows_mask")
    return tags


REQUIRED_FEATURES = {
    "sa_f32", "sa_bf16", "sa_f16", "fp_f32", "fp_bf16", "fp_f16", "rows_f32", "rows_bf16", "rows_f16",
    "sa_autocast", "fp_autocast", "rows_autocast", "sa_autocast_no_features",
    "sa_out_slice", "fp_out_slice", "rows_out_slice", "sa_nonfinite", "rows_nonfinite",
    "bn_affine", "bn_plain", "bn_none", "last_no_relu", "negative_gamma", "small_var", "large_var", "eps_1e-5",
    "sa_group_all", "sa_xyz_first_True", "sa_xyz_first_False", "sa_features_only", "sa_c0", "sa_c1",
    "fp_ragged", "fp_dense", "fp_c1_0", "rows_mask",
}


def test_slice_reaches_every_branch_several_times_per_seed(slice_params):
    for seed, ps in slice_params.items():
        count = collections.Counter(t for p in ps for t in p["tags"])
        thin = {t: count[t] for t in REQUIRED_BRANCHES if count[t] < 2}
        assert not thin, (seed, thin)
        assert not {t for t in count if "_e2_tm16" in t}, seed  # unreachable, see above
    seen = set().union(*(features(p) for ps in slice_params.values() for p in ps))
    assert REQUIRED_FEATURES <= seen, sorted(REQUIRED_FEATURES - seen)


def test_targets_are_branches_and_cases_are_complete():
    assert {t for target in F.SA_TARGETS + F.ROW_TARGETS for t in target.split("+")} <= REQUIRED_BRANCHES
    assert set(F.CASES) == set(F.DRAW) == set(F.RUN)
    assert F.SLICE_ITERATIONS % len(F.CASES) == 0


def test_draws_are_reproducible_and_bounded(slice_params):
    a = F.draws(F.SLICE_SEEDS[0], 12)
    for p, q in zip(a, slice_params[F.SLICE_SEEDS[0]]):
        assert F.public(p) == F.public(q)
        for L, M in zip(p["layers"], q["layers"]):
            assert np.array_equal(L["w"], M["w"])
    for ps in slice_params.values():
        for p in ps:
            widths = p["widths"]
            rows = p["b"] * p["s"] * p["k"] if p["case"] == "sa" else p["b"] * p["n"] if p["case"] == "fp" else p["rows"]
            assert rows * F._macs(p["cin"], widths) <= F.MAC_CAP
            assert 1 <= len(widths) <= MO.MAX_LAYERS and max(widths) <= MO.MAX_WIDTH
            assert p["cin"] <= (MO.SA_MAX_IN if p["case"] == "sa" else MO.ROW_MAX_IN)
            if p["case"] == "fp" and p["lengths"]:
                assert all(1 <= l <= p["n"] for l in p["lengths"])


# ----------------------------------------------------------------------------------------------- the C oracle
def _one(w, **kw):
    return dict(w=np.asarray(w, np.float32), **kw)


def test_oracle_uses_fmaf_and_ascending_k():
    # fmaf(1 + 2^-12, 1 + 2^-12, -(1 + 2^-11)) = 2^-24 exactly; a rounded product then a subtraction gives 0
    x = np.array([[-1.0, 1 + 2 ** -12]], np.float32)
    got = O.oracle_mlp_rows_f32(x, [_one([[1 + 2 ** -11, 1 + 2 ** -12]])])
    assert got[0, 0] == 2.0 ** -24
    prod = np.float32(np.float32(1 + 2 ** -12) * np.float32(1 + 2 ** -12))
    assert np.float32(prod - np.float32(1 + 2 ** -11)) == 0
    # the epilogue is one fmaf too: acc·scale + shift with scale = 1 / sqrt(var + eps) ...
    # ascending k: 1 + 2^-24 rounds to 1 (a tie to even), twice; descending, 2^-24 + 2^-24 = 2^-23 survives
    x = np.array([[1.0, 2 ** -24, 2 ** -24]], np.float32)
    assert O.oracle_mlp_rows_f32(x, [_one(np.ones((1, 3)))])[0, 0] == 1.0
    assert O.oracle_mlp_rows_f32(x[:, ::-1], [_one(np.ones((1, 3)))])[0, 0] == np.float32(1 + 2 ** -23)


def test_oracle_affine_and_eps_in_float32():
    L = _one(np.ones((3, 1)), b=[0.5, -2.0, 1.0], mean=[0.25, 1.0, 0.0], var=[0.0, 4.0, 1e-4], eps=1e-3,
             gamma=[2.0, -1.0, 0.5], beta=[0.0, 1.0, -0.125])
    scale, shift = O.oracle_mlp_affine_f32(L)
    f = np.float32
    eps = f(1e-3)  # the kernels take eps as a float32: 1e-3 rounded once
    assert float(eps) != 1e-3
    for j in range(3):
        sc = f(f(1) / np.sqrt(f(f(L["var"][j]) + eps))) * f(L["gamma"][j])
        assert scale[j] == f(sc)
        # fmaf(bias - mean, scale, beta): the exact product plus beta, rounded once
        want = f(np.float64(f(f(L["b"][j]) - f(L["mean"][j]))) * np.float64(scale[j]) + np.float64(L["beta"][j]))
        assert shift[j] == want
    # var 0: scale 1 / sqrt(float32(1e-3)) = 31.622776..., not 1 / sqrt(1e-3) in double rounded
    assert O.oracle_mlp_affine_f32(_one([[1.0]], b=[0.0], mean=[0.0], var=[0.0], eps=1e-3))[0][0] == f(1) / np.sqrt(eps)
    # no batch norm: scale 1, shift = bias; no affine: beta 0, gamma 1
    assert O.oracle_mlp_affine_f32(_one([[1.0]], b=[0.75]))[0][0] == 1 and O.oracle_mlp_affine_f32(_one([[1.0]], b=[0.75]))[1][0] == f(0.75)
    sc, sh = O.oracle_mlp_affine_f32(_one([[1.0]], b=[1.0], mean=[0.5], var=[3.0], eps=1.0))
    assert sc[0] == 0.5 and sh[0] == 0.25


def test_oracle_nan_relu_and_max():
    x = np.array([[np.nan, 1.0], [-1.0, 0.0], [2.0, -3.0]], np.float32)
    got = O.oracle_mlp_rows_f32(x, [_one([[1.0, 1.0], [-1.0, 0.0]], relu=1)])
    assert np.isnan(got[0]).all()                      # NaN passes the ReLU
    assert got[1, 0] == 0 and got[1, 1] == 1          # -1 -> 0
    assert np.signbit(O.oracle_mlp_rows_f32(np.array([[-0.0]], np.float32), [_one([[1.0]], relu=1)])[0, 0]) is np.False_
    pooled = MO.max_pool(got, 3)
    assert np.isnan(pooled).all()                      # the max keeps NaN, as the kernel's integer keys do
    assert (MO.max_pool(got[1:], 2) == [[0.0, 1.0]]).all()


def test_oracle_against_float64():
    rs = np.random.RandomState(3)
    for cin, cout in ((1, 1), (7, 65), (33, 129), (300, 17)):
        x = (rs.standard_normal((40, cin)) * np.exp(rs.uniform(-5, 5, cin))).astype(np.float32)
        w = rs.standard_normal((cout, cin)).astype(np.float32)
        b = rs.standard_normal(cout).astype(np.float32)
        got = O.oracle_mlp_rows_f32(x, [_one(w, b=b)])
        lin = torch.nn.Linear(cin, cout).double()
        with torch.no_grad():
            lin.weight.copy_(torch.from_numpy(w.astype(np.float64)))
            lin.bias.copy_(torch.from_numpy(b.astype(np.float64)))
            ref = lin(torch.from_numpy(x.astype(np.float64))).numpy()
        mass = np.abs(x.astype(np.float64)) @ np.abs(w.astype(np.float64)).T + np.abs(b)
        assert NUM.within_bound(got, ref, mass, cin + 1, "f32").all(), (cin, cout)
    # several layers with batch norms against the torch modules in float64
    layers = F.draw_layers(rs, 37, [96, 80, 5], "f32")
    x = rs.standard_normal((50, 37)).astype(np.float32)
    ref = _torch_float64(x, layers)
    got = O.oracle_mlp_rows_f32(x, F.oracle_layers(layers))
    np.testing.assert_allclose(got, ref, rtol=1e-4, atol=1e-4 * np.abs(ref).max())


def _torch_float64(x, layers):
    mods = []
    for L in layers:
        lin = torch.nn.Linear(L["w"].shape[1], L["w"].shape[0]).double()
        with torch.no_grad():
            lin.weight.copy_(torch.from_numpy(L["w"].astype(np.float64)))
            lin.bias.copy_(torch.from_numpy(L["b"].astype(np.float64)))
        mods.append(lin)
        if "mean" in L:
            bn = torch.nn.BatchNorm1d(L["w"].shape[0], eps=float(np.float32(L["eps"])), affine="gamma" in L).double()
            with torch.no_grad():
                bn.running_mean.copy_(torch.from_numpy(L["mean"].astype(np.float64)))
                bn.running_var.copy_(torch.from_numpy(L["var"].astype(np.float64)))
                if "gamma" in L:
                    bn.weight.copy_(torch.from_numpy(L["gamma"].astype(np.float64)))
                    bn.bias.copy_(torch.from_numpy(L["beta"].astype(np.float64)))
            mods.append(bn.eval())
        if L["relu"]:
            mods.append(torch.nn.ReLU())
    with torch.no_grad():
        return torch.nn.Sequential(*mods)(torch.from_numpy(x.astype(np.float64))).numpy()


# ----------------------------------------------------------------------------------------------- 16-bit bound
@pytest.mark.parametrize("fmt", ["bf16", "f16"])
def test_bound_holds_on_a_cpu_model_of_the_16_bit_kernel(fmt):
    rs = np.random.RandomState(11 if fmt == "bf16" else 12)
    worst = 0.0
    for trial in range(12):
        cin = int(rs.choice([1, 3, 31, 33, 67, 130]))
        widths = [int(rs.choice([1, 8, 33, 65, 130])) for _ in range(int(rs.randint(1, 5)))]
        layers = F.draw_layers(rs, cin, widths, fmt)
        aff = [O.oracle_mlp_affine_f32(L) for L in F.oracle_layers(layers)]
        x = NUM.quantize(F._scaled(rs, (48, cin), fmt), fmt)
        pool_k = int(rs.choice([1, 3, 16])) if trial % 2 else None
        for _ in range(3):  # three summation orders
            got = MO.simulate16(x, layers, aff, fmt, rs, pool_k)
            ref, bound = MO.bound16(x, layers, aff, fmt, pool_k)
            ok, ratio = MO.check16(got, ref, bound)
            assert ok, (trial, ratio)
            worst = max(worst, ratio)
    print(f"{fmt}: worst err / bound on the CPU model {worst:.3g}")
    assert worst > 0.01  # the bound is not vacuous


@pytest.mark.parametrize("pool_k", [None, 8], ids=["rows", "sa"])
@pytest.mark.parametrize("fmt", ["bf16", "f16"])
def test_bound_rejects_every_mutation(fmt, pool_k):
    rs = np.random.RandomState(21)
    layers = F.mutation_layers(rs)
    x = NUM.quantize(rs.standard_normal((64, 37)).astype(np.float32), fmt)
    aff = lambda ls: [O.oracle_mlp_affine_f32(L) for L in F.oracle_layers(ls)]
    got = MO.simulate16(x, layers, aff(layers), fmt, rs, pool_k)
    ref, bound = MO.bound16(x, layers, aff(layers), fmt, pool_k)
    assert MO.check16(got, ref, bound)[0]
    for kind in MO.MUTATIONS:
        bad = MO.mutate(layers, kind)
        r, b = MO.bound16(x, bad, aff(bad), fmt, pool_k)
        if kind == "swap":
            r, b = MO.swap_partial_pass(r), MO.swap_partial_pass(b)
        assert not MO.check16(got, r, b)[0], kind


def test_float32_comparison_rejects_every_mutation():
    rs = np.random.RandomState(22)
    layers = F.mutation_layers(rs)
    x = rs.standard_normal((64, 37)).astype(np.float32)
    got = MO.max_pool(O.oracle_mlp_rows_f32(x, F.oracle_layers(layers)), 8)
    for kind in MO.MUTATIONS:
        want = MO.max_pool(O.oracle_mlp_rows_f32(x, F.oracle_layers(MO.mutate(layers, kind))), 8)
        if kind == "swap":
            want = MO.swap_partial_pass(want)
        assert not F.same_values(got, want), kind


def test_same_values_treats_signed_zeros_equal_and_nan_by_place():
    a = np.array([0.0, np.nan, 1.0], np.float32)
    assert F.same_values(a, np.array([-0.0, np.nan, 1.0], np.float32))
    assert not F.same_values(a, np.array([0.0, 1.0, 1.0], np.float32))
    assert not F.same_values(a, np.array([0.0, np.nan, np.nextafter(np.float32(1), np.float32(2))], np.float32))


def test_sa_rows_gather_in_float32():
    rs = np.random.RandomState(4)
    xyz = rs.random_sample((2, 9, 3)).astype(np.float32)
    ctr = rs.random_sample((2, 3, 3)).astype(np.float32)
    pts = rs.standard_normal((2, 9, 4)).astype(np.float32)
    idx = rs.randint(0, 9, (2, 3, 5))
    r = MO.sa_rows(xyz, ctr, pts, idx, True, True, "f32")
    assert r.shape == (2, 3, 5, 7)
    assert r[1, 2, 4, 0] == np.float32(xyz[1, idx[1, 2, 4], 0] - ctr[1, 2, 0])
    assert (r[1, 2, 4, 3:] == pts[1, idx[1, 2, 4]]).all()
    r = MO.sa_rows(xyz, ctr, pts, idx, False, True, "bf16")
    assert (r[..., 4:] == NUM.quantize(r[..., 4:], "bf16")).all() and (r[..., :4] == MO.sa_rows(xyz, ctr, pts, idx, True, False, "f32")).all()
    g = MO.sa_rows(xyz, None, None, None, True, True, "f32")
    assert g.shape == (2, 1, 9, 3) and (g[:, 0] == xyz).all()
