"""CPU checks of tests/fuzz_masked_bn_gpu.py, tests/bn_regimes.py and the masked batch-norm oracle (no device).

The fixed slice (fuzz_masked_bn_gpu.SLICE_SEEDS, SLICE_ITERATIONS cases each) is replayed through bn_regimes: every
<T, V, VEC> instantiation of masked_bn.cu must be launched by some case, with every named regime and a second
grid-stride trip of each elementwise kernel.  The restated constants must be those of masked_bn.cu; the oracle must
agree with float64 truth within float32 bounds (so it cannot share a wrong formula with the kernels); and the
comparators of the fuzz must catch planted defects."""
import os
import re

import numpy as np
import pytest

import bn_regimes as R
import fuzz_masked_bn_gpu as F
import numerics as NUM
from oracle import oracle as O

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "pointnet2_b200", "csrc")

REQUIRED_REGIMES = (
    {f"vec{v}_tx{t}" for v in (1, 4) for t in (1, 2, 4, 8, 16, 32)}
    | {"idle_lanes", "col_tiles_many", "partial_last_tile",
       "scalar_vec4_x", "scalar_vec4_y", "scalar_vec4_dy", "scalar_vec4_dx",
       "chunks_1", "rows_eq_chunk_rows", "chunks_32", "chunks_33", "chunks_ge_64_remainder",
       "keep_all", "empty_chunk", "late_rows_only", "keep_one", "keep_none",
       "f32", "bf16", "f16", "affine", "no_affine", "momentum", "cma1", "cma_large", "no_tracking", "null_dgrads",
       "data_constant", "data_far_mean", "data_overflow", "data_nonfinite", "data_subnormal", "data_ties",
       "f16_out_past_65504", "beta_neg_zero", "gamma_zero", "gamma_negative",
       "max_b1", "max_b31", "max_b32", "max_b33", "max_b70", "max_ragged_last_pass", "max_n_lt_ty",
       "max_row_trips_3_plus", "max_empty_cloud", "max_tie_within_thread", "max_tie_across_threads", "max_nan_row",
       "torch_plain", "torch_max", "torch_ops_plain", "torch_ops_max"}
    | {"refused_" + w for w in F.REFUSALS})
ELEMENTWISE = ["mbn_norm_relu_kernel", "mbn_bwd_dx_kernel", "mbn_max_bwd_dx_kernel", "mbn_norm_relu_max_kernel",
               "mbn_max_bwd_finalize_kernel"]


def plans(p):
    """(launches, regimes) of one drawn case"""
    case, reg = p["case"], set()
    if case == "refused":
        return [], {"refused_" + p["why"]}
    if case == "torch":
        return [], {("torch_ops_" if p["functional"] else "torch_") + p["form"]}
    fmt = p["fmt"]
    reg |= {fmt, "no_affine" if p["gamma"] is None else "affine", "no_tracking" if p["tracking"] == "none"
            else p["tracking"]}
    if p["null_dgrads"] and p["gamma"] is not None:
        reg.add("null_dgrads")
    if p["data"] != "normal":
        reg.add("data_" + p["data"])
    if p["gamma"] is not None:
        reg |= {"gamma_zero"} if (p["gamma"] == 0).any() else set()
        reg |= {"gamma_negative"} if (p["gamma"] < 0).any() else set()
        reg |= {"beta_neg_zero"} if (np.signbit(p["beta"]) & (p["beta"] == 0)).any() else set()
        if fmt == "f16" and p["affine"] == "huge":
            reg.add("f16_out_past_65504")
    off = p["off"]
    if case == "plain":
        c, rows = p["c"], p["rows"]
        al_f = not (off["x"] or off["y"])
        al_b = not any(off.values())
        d = R.plain_call(fmt, rows, c, p["keep"], al_f, al_b)
    else:
        c, rows = p["c"], p["b"] * p["n"]
        d = R.max_call(fmt, p["b"], p["n"], c, p["keep"], not off["x"], not (off["x"] or off["dx"]))
        reg |= F.tie_regimes(p)
    if d["geom"]["vec"] == 4:
        reg |= {f"scalar_vec4_{k}" for k, v in off.items() if v}
    return d["launches"], reg | d["regimes"]


def replay():
    kernels, regimes, trips = set(), set(), {}
    for seed in F.SLICE_SEEDS:
        for p in F.draws(seed, F.SLICE_ITERATIONS):
            L, reg = plans(p)
            regimes |= reg
            for g in L:
                kernels.add(g["kernel"])
                fam = g["kernel"].split("<")[0]
                trips[fam] = max(trips.get(fam, 0), g["trips"])
    return kernels, regimes, trips


@pytest.fixture(scope="module")
def reached():
    return replay()


def test_slice_reaches_every_instantiation(reached):
    kernels, _, _ = reached
    assert kernels <= set(R.instances()), kernels - set(R.instances())
    missing = sorted(set(R.instances()) - kernels)
    assert not missing, missing


def test_slice_reaches_every_regime(reached):
    _, regimes, _ = reached
    missing = sorted(REQUIRED_REGIMES - regimes)
    assert not missing, missing


def test_slice_takes_a_second_trip_in_every_elementwise_kernel(reached):
    _, _, trips = reached
    assert {f: trips.get(f, 0) >= 2 for f in ELEMENTWISE} == {f: True for f in ELEMENTWISE}, trips


def test_restated_constants_match_the_source():
    src = open(os.path.join(CSRC, "masked_bn.cu")).read()
    for name, v in (("kMbnThreads", R.THREADS), ("kMbnRows", R.ROWS), ("kMbnGroups", R.GROUPS),
                    ("kMbnMergeWarps", R.MERGE_WARPS), ("kMbnUnroll", R.UNROLL)):
        assert re.search(r"constexpr int %s = %d;" % (name, v), src), name
    assert "num_sms() * 8 / g.col_tiles + 1" in src  # elementwise_row_blocks' cap
    assert "g.col_tiles <= 65535" in src
    assert "(c % 4 == 0) ? 4 : 1" in src and "while (tx < lanes && tx < 32) tx <<= 1;" in src
    oracle = open(os.path.join(os.path.dirname(CSRC), "..", "oracle", "pn2_oracle.c")).read()
    for name, v in (("MBN_THREADS", R.THREADS), ("MBN_ROWS", R.ROWS), ("MBN_GROUPS", R.GROUPS),
                    ("MBN_MERGE_WARPS", R.MERGE_WARPS)):
        assert re.search(r"#define %s %d\b" % (name, v), oracle), name


def test_restated_kernels_match_the_launch_sites():
    src = open(os.path.join(CSRC, "masked_bn.cu")).read()
    launched = set(re.findall(r"\b(\w+_kernel)\s*(?:<[^<>]*>)?\s*<<<", src))
    assert launched == {k.split("<")[0] for k in R.instances()}


def test_geometry_by_hand():
    assert [R.geom(1, c)["tx"] for c in (1, 2, 3, 5, 9, 17)] == [1, 2, 4, 8, 16, 32]
    assert [R.geom(1, c)["tx"] for c in (4, 8, 12, 20, 36, 68)] == [1, 2, 4, 8, 16, 32]
    g = R.geom(1, 132)
    assert (g["vec"], g["lanes"], g["col_tiles"], g["ty"], g["chunk_rows"]) == (4, 33, 2, 8, 256)
    assert R.geom(10000, 1)["chunks"] == 2 and R.geom(8192, 1)["chunks"] == 1


# ------------------------------------------------------------------------------------- oracle against float64
def _f32_bound(n):
    return 4 * NUM.gamma(max(n, 1) + 8)


@pytest.mark.parametrize("seed", range(6))
def test_oracle_against_float64(seed):
    """mean, biased variance, y, dx, dgamma and dbeta of the oracle within float32 error bounds of float64 truth"""
    rs = np.random.RandomState(100 + seed)
    for c in (1, 5, 8, 13, 132):
        rows = int(rs.choice([1, 2, 9, 300, 9000]))
        keep = (rs.random_sample(rows) < 0.7).astype(np.uint8)
        keep[rs.randint(rows)] = 1
        x = (rs.standard_normal((rows, c)) * rs.uniform(0.5, 3) + rs.uniform(-20, 20)).astype(np.float32)
        eps = 1e-3
        mean, var_eps, cnt, _, _ = O.oracle_mbn_stats(x, keep, eps)
        xr = x[keep != 0].astype(np.float64)
        n = len(xr)
        assert cnt == n
        m64, v64 = xr.mean(0), xr.var(0)
        amax = np.abs(xr).max(0)
        gam = _f32_bound(n)
        assert np.all(np.abs(mean - m64) <= gam * amax)
        dm = gam * amax
        assert np.all(np.abs((var_eps.astype(np.float64) - eps) - v64) <= 2 * dm * np.sqrt(v64) + dm * dm + gam * v64
                      + NUM.ulp(var_eps, "f32"))
        invstd = (1 / np.sqrt(var_eps.astype(np.float64))).astype(np.float32)
        gamma = rs.uniform(0.5, 2, c).astype(np.float32)
        beta = rs.standard_normal(c).astype(np.float32)
        y = O.oracle_mbn_norm_relu(x, keep, mean, invstd, gamma, beta)
        xh64 = (x - m64) / np.sqrt(v64 + eps)
        y64 = np.where(keep[:, None] != 0, np.maximum(xh64 * gamma + beta, 0), 0)
        tol = 1e-4 * (np.abs(xh64 * gamma) + np.abs(beta) + 1)
        assert np.all(np.abs(y - y64) <= tol)
        dy = rs.standard_normal((rows, c)).astype(np.float32)
        dx, dg, db = O.oracle_mbn_backward(dy, x, y, keep, mean, invstd, gamma)
        g = np.where((keep[:, None] != 0) & (y > 0), dy, 0).astype(np.float64)
        xh = (x - mean.astype(np.float64)) * invstd.astype(np.float64)
        db64, dg64 = g.sum(0), (g * xh).sum(0)
        mass_g, mass_gx = np.abs(g).sum(0), np.abs(g * xh).sum(0)
        assert np.all(np.abs(db - db64) <= gam * mass_g + 1e-30)
        assert np.all(np.abs(dg - dg64) <= gam * mass_gx * 2 + 1e-30)
        dx64 = np.where(keep[:, None] != 0, gamma * invstd.astype(np.float64) * (g - db64 / n - xh * dg64 / n), 0)
        assert np.all(np.abs(dx - dx64) <= 1e-4 * (np.abs(gamma * invstd) * (np.abs(g) + mass_g / n + np.abs(xh) * mass_gx / n)
                                                   + 1e-30))


def test_oracle_max_pool_and_backward_against_float64():
    rs = np.random.RandomState(7)
    b, n, c = 5, 40, 6
    x = rs.randint(-3, 4, (b * n, c)).astype(np.float32)
    keep = (np.arange(n)[None] < np.array([40, 1, 0, 17, 33])[:, None]).astype(np.uint8).reshape(-1)
    mean, var_eps, cnt, _, _ = O.oracle_mbn_stats(x, keep, 1e-5)
    invstd = (1 / np.sqrt(var_eps.astype(np.float64))).astype(np.float32)
    y = O.oracle_mbn_norm_relu(x, keep, mean, invstd).reshape(b, n, c)
    out, arg = O.oracle_mbn_max_pool(y, keep)
    k = keep.reshape(b, n) != 0
    for i in range(b):
        for j in range(c):
            if not k[i].any():
                assert arg[i, j] == -1 and out[i, j] == 0
                continue
            real = np.flatnonzero(k[i])
            col = y[i, real, j]
            assert arg[i, j] == real[np.argmax(col)] and out[i, j] == col.max()
    dout = rs.standard_normal((b, c)).astype(np.float32)
    dx, dg, db = O.oracle_mbn_max_backward(dout, x.reshape(b, n, c), out, arg, keep, mean, invstd)
    g = np.where((arg >= 0) & (out > 0), dout, 0).astype(np.float64)
    assert np.allclose(db, g.sum(0), rtol=1e-6, atol=1e-6)


def test_zero_real_rows_give_nan_statistics_as_masked_batch_norm():
    """the rule include/pn2_api.h states for a batch without a real row: mean 0 / 0, running buffers NaN"""
    x = np.ones((10, 3), np.float32)
    mean, var_eps, cnt, rm, rv = O.oracle_mbn_stats(x, np.zeros(10), 1e-5, 0.1, 1, np.zeros(3), np.ones(3))
    assert cnt == 0 and np.isnan(mean).all() and np.isnan(var_eps).all() and np.isnan(rm).all() and np.isnan(rv).all()
    import torch
    from pointnet2_b200.layers import masked_batch_norm
    bn = torch.nn.BatchNorm1d(3).train()
    masked_batch_norm(bn, torch.zeros(10, 3), torch.zeros(10, 1, dtype=torch.bool))
    assert torch.isnan(bn.running_mean).all() and torch.isnan(bn.running_var).all()


def test_one_real_row_has_zero_variance():
    x = np.arange(30, dtype=np.float32).reshape(10, 3)
    keep = np.zeros(10, np.uint8)
    keep[7] = 1
    mean, var_eps, cnt, rm, rv = O.oracle_mbn_stats(x, keep, 0.25, 0.5, 1, np.zeros(3), np.ones(3))
    assert cnt == 1 and np.array_equal(mean, x[7]) and np.all(var_eps == np.float32(0.25))
    assert np.array_equal(rm, x[7] * np.float32(0.5)) and np.all(rv == np.float32(0.5))  # unbiased 0 / max(0, 1)


# ------------------------------------------------------------------------- the comparators catch planted defects
def test_comparators_catch_a_flipped_bit():
    rs = np.random.RandomState(3)
    want = rs.standard_normal(64).astype(np.float32)
    for fmt in F.FMTS:
        got = F.G.to_fmt_bits(want, fmt).copy()
        assert F.same(got, want, fmt)
        got[rs.randint(64)] ^= 1
        assert not F.same(got, want, fmt)
    nan = np.full(4, np.nan, np.float32)
    assert F.same(np.full(4, 0x7FFFFFFF, np.uint32), nan, "f32")  # any NaN equals any NaN


def test_invstd_comparator_holds_two_ulp():
    v = np.array([0.5, 2.0, 1e-5, np.inf, np.nan], np.float32)
    want = (1 / np.sqrt(v.astype(np.float64))).astype(np.float32)
    assert F.invstd_ok(want, v)
    off3 = want.copy()
    off3[1] = np.nextafter(np.nextafter(np.nextafter(want[1], np.float32(9)), np.float32(9)), np.float32(9))
    assert not F.invstd_ok(off3, v)


def test_max_pool_comparator_catches_a_wrong_tie():
    """y with ties across rows: the oracle takes the first; the last row of the tie must not pass"""
    y = np.zeros((1, 6, 1), np.float32)
    y[0, [1, 4], 0] = 2.0
    keep = np.ones(6, np.uint8)
    out, arg = O.oracle_mbn_max_pool(y, keep)
    assert arg[0, 0] == 1
    assert not np.array_equal(np.array([[4]], np.int32), arg)
    y[0, 3, 0] = np.nan  # NaN wins
    assert O.oracle_mbn_max_pool(y, keep)[1][0, 0] == 3
    z = np.array([[[-0.0], [0.0], [-0.0]]], np.float32)  # -0 < +0
    assert O.oracle_mbn_max_pool(z, np.ones(3, np.uint8))[1][0, 0] == 1


def test_padding_comparator_catches_an_unwritten_row():
    """a padding row of y left poisoned fails the 'padding rows come back 0' check, and a written guard fails too"""
    rows, c, fmt = 5, 3, "bf16"
    keep = np.array([1, 0, 1, 1, 0], np.uint8)
    body = np.zeros(rows * c, np.uint16)
    body.reshape(rows, c)[1] = F.POISON[fmt]
    assert not np.all(body.reshape(rows, c)[keep == 0] == 0)
    full = np.concatenate([np.zeros(rows * c, np.uint16), np.full(F.G.GUARD, F.POISON[fmt], np.uint16)])
    assert F.G.guarded(full, 0, rows * c, fmt)[1]
    full[rows * c] = 0
    assert not F.G.guarded(full, 0, rows * c, fmt)[1]
