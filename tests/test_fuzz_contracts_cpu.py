"""Without a GPU: the fixed-seed slice of tests/fuzz_contracts_gpu.py reaches every regime its contracts branch on,
and the reference arithmetic it checks against (tests/numerics.py) is right."""
import numpy as np
import pytest
import torch

import fuzz_contracts_gpu as F
import numerics as NUM


@pytest.fixture(scope="module")
def slice_params():
    return [p for seed in F.SLICE_SEEDS for p in F.draws(seed, F.SLICE_ITERATIONS)]


def regimes(p):
    """the named regimes one case's parameters reach"""
    tags = set()
    fmt = p.get("fmt") or (p["mode"].split("_")[1] if p["case"] == "interp_grad" else None)
    if fmt:
        tags.add("dtype_" + fmt)
    if p.get("offset") == 1:
        tags.add("offset_1")
    lens = p.get("lens")
    if lens:
        if 1 in lens["lengths"]:
            tags.add("length_1")
        npoint = p.get("npoint", p.get("m")) if p["case"] in ("fps_ragged", "layer_ragged") else None
        if npoint and min(lens["lengths"]) < npoint:
            tags.add("length_below_npoint")
        if lens["form"].startswith("clamp") and any(r < 1 or r > p["n"] for r in lens["raw"]):
            tags.add("clamped_device_lengths")
        tags.add("lengths_" + lens["form"])
    if p["case"] == "ball_ragged":
        tags.add(f"bq_mode_{p['mode']}")
    if p["case"] == "fps_ragged" and p["plan"] and p["plan"][2] >= 2:
        tags.add("fps_cluster_plan")
    if p["case"] in ("interp_grad", "group_grad") and p["longest"] > 256:
        tags.add("list_over_256_" + p["case"])
    if p["case"] == "interp_grad" and p["m"] > 16000:
        tags.add("m_over_16000")
    if p["case"] == "interp_ragged":
        tags.add("c1_0" if p["c1"] == 0 else "c1_positive")
    return tags


REQUIRED = {
    "dtype_f32", "dtype_bf16", "dtype_f16", "offset_1",
    "length_1", "length_below_npoint", "clamped_device_lengths",
    "lengths_host", "lengths_int32", "lengths_int64",
    "bq_mode_0", "bq_mode_1", "bq_mode_2", "fps_cluster_plan",
    "list_over_256_interp_grad", "list_over_256_group_grad", "m_over_16000",
    "c1_0", "c1_positive",
}


def test_slice_reaches_every_regime(slice_params):
    seen = set().union(*(regimes(p) for p in slice_params))
    assert REQUIRED <= seen, sorted(REQUIRED - seen)


def test_slice_runs_every_case_several_times_per_seed():
    assert F.SLICE_ITERATIONS % len(F.CASES) == 0 and F.SLICE_ITERATIONS // len(F.CASES) >= 3
    assert set(F.CASES) == set(F.DRAW) == set(F.RUN)


def test_draws_are_reproducible_and_bounded():
    a, b = F.draws(F.SLICE_SEEDS[0], 18), F.draws(F.SLICE_SEEDS[0], 18)
    for p, q in zip(a, b):
        assert F.public(p) == F.public(q)
    for p in F.draws(F.SLICE_SEEDS[1], 45):
        if p["case"] == "fps_ragged":
            assert p["n"] * p["npoint"] <= 2 * 10 ** 7  # the C oracle stays cheap
        if "lens" in p and p["lens"]:
            assert all(1 <= l <= p["n"] for l in p["lens"]["lengths"])
            assert len(p["lens"]["raw"]) == p["b"]


# ---------------------------------------------------------------------------------------------- rounding once
def test_round_once_matches_hand_values():
    x = np.array([1.0, 1 + 2 ** -8, 1 + 3 * 2 ** -8, 1 + 2 ** -8 + 2 ** -20, -2.0, 0.0], np.float32)
    # bf16 keeps 7 mantissa bits: 1 + 2^-8 is a tie between 1 and 1 + 2^-7 and goes to even (1); 1 + 3·2^-8 goes up to
    # 1 + 2^-6 (even); anything above the tie rounds up
    np.testing.assert_array_equal(NUM.round_once(x, "bf16"), np.array([0x3F80, 0x3F80, 0x3F82, 0x3F81, 0xC000, 0], np.uint16))
    # f16: 10 mantissa bits, ties at 2^-11
    y = np.array([1 + 2 ** -11, 1 + 3 * 2 ** -11, 65504.0, 65519.99, 65520.0, 2.0 ** -24, 2.0 ** -25, 2.0 ** -25 * 1.5],
                 np.float32)
    np.testing.assert_array_equal(NUM.round_once(y, "f16"),
                                  np.array([0x3C00, 0x3C02, 0x7BFF, 0x7BFF, 0x7C00, 0x0001, 0x0000, 0x0001], np.uint16))
    # bf16 overflow: the largest float32 rounds up into inf
    assert NUM.round_once(np.array([3.4028235e38], np.float32), "bf16")[0] == 0x7F80


@pytest.mark.parametrize("fmt,dtype", [("bf16", torch.bfloat16), ("f16", torch.float16)])
def test_round_once_agrees_with_torch(fmt, dtype):
    rs = np.random.RandomState(5)
    bits = rs.randint(0, 2 ** 32, 200000, dtype=np.uint64).astype(np.uint32)
    x = bits.view(np.float32)
    x = x[np.isfinite(x)]
    # add the edges: subnormals of both formats, values around the float16 overflow threshold, exact ties
    edges = np.array([2.0 ** -24, 2.0 ** -25, 3 * 2.0 ** -26, 2.0 ** -14 * 0.999, 2.0 ** -133, 2.0 ** -134, 65504, 65519.996,
                      65520, 70000, 1 + 2 ** -8, 1 + 2 ** -11, -(1 + 3 * 2 ** -11), 0.0, -0.0, np.inf, -np.inf], np.float32)
    x = np.concatenate([x, edges, x * np.float32(2.0 ** -100), x * np.float32(2.0 ** -120)])
    want = torch.from_numpy(x).to(dtype).view(torch.int16).numpy().view(np.uint16)
    np.testing.assert_array_equal(NUM.round_once(x, fmt), want)
    np.testing.assert_array_equal(NUM.decode(want, fmt), torch.from_numpy(x).to(dtype).float().numpy())


def test_ulp_hand_values():
    np.testing.assert_array_equal(NUM.ulp([1.0, 1.5, 2.0, 0.0], "bf16"), [2.0 ** -7, 2.0 ** -7, 2.0 ** -6, 2.0 ** -133])
    np.testing.assert_array_equal(NUM.ulp([1.0, 1024.0, 2.0 ** -20, 0.0], "f16"), [2.0 ** -10, 1.0, 2.0 ** -24, 2.0 ** -24])
    np.testing.assert_array_equal(NUM.ulp([1.0, 2.0 ** -130], "f32"), [2.0 ** -23, 2.0 ** -149])


# ------------------------------------------------------------------------------------------- float64 bound
def test_bound_hand_values():
    # three terms of mass 3: γ(3) = 4u / (1 - 4u)
    g = 4 * 2.0 ** -24 / (1 - 4 * 2.0 ** -24)
    assert NUM.within_bound(np.float32(1.0), 1.0 + 3 * g * 0.999, 3.0, 3, "f32")
    assert not NUM.within_bound(np.float32(1.0), 1.0 + 3 * g * 1.001, 3.0, 3, "f32")
    # a bf16 result may be off by half its ulp more: at 1.0, 2^-8
    assert NUM.within_bound(np.float32(1.0), 1.0 + 2.0 ** -8, 0.0, 1, "bf16")
    assert not NUM.within_bound(np.float32(1.0), 1.0 + 2.0 ** -8 * 1.01, 0.0, 1, "bf16")
    assert not NUM.within_bound(np.float32(np.nan), 0.0, 1.0, 1, "f32")


def test_bound_holds_for_float32_sums_in_any_order_and_catches_a_dropped_term():
    rs = np.random.RandomState(7)
    for trial in range(200):
        L = int(rs.randint(1, 3000))
        terms = (rs.standard_normal(L) * np.exp(rs.uniform(-20, 20, L))).astype(np.float32)
        w = rs.random_sample(L).astype(np.float32)
        prods = (w * terms).astype(np.float32)  # the kernel's rounded products
        ref, mass, count = NUM.scatter64(1, np.zeros(L, int), w.astype(np.float64) * terms)
        for order in (np.arange(L), rs.permutation(L)):
            s = np.float32(0)
            for v in prods[order]:
                s = np.float32(s + v)
            assert NUM.within_bound(s, ref[0, 0], mass[0, 0], count[0], "f32")
            for fmt in ("bf16", "f16"):
                if abs(float(s)) < 60000:
                    assert NUM.within_bound(NUM.quantize(np.array([s]), fmt)[0], ref[0, 0], mass[0, 0], count[0], fmt)
    # dropping the smallest-magnitude nonzero term of a short list with a small mass is caught
    terms = np.array([1.0, 1e-3, -0.5], np.float32)
    ref, mass, _ = NUM.scatter64(1, np.zeros(3, int), terms)
    assert not NUM.within_bound(np.float32(np.float32(1.0) + np.float32(-0.5)), ref[0, 0], mass[0, 0], 3, "f32")


def test_scatter64():
    ref, mass, count = NUM.scatter64(4, [0, 2, 2, 3, 2], np.array([[1.0, -1], [2, 2], [-3, 1], [4, 0], [0.5, 0.5]]))
    np.testing.assert_array_equal(ref, [[1, -1], [0, 0], [-0.5, 3.5], [4, 0]])
    np.testing.assert_array_equal(mass, [[1, 1], [0, 0], [5.5, 3.5], [4, 0]])
    np.testing.assert_array_equal(count, [1, 0, 3, 1])


# ----------------------------------------------------------------------------------------------- padding
@pytest.mark.parametrize("kind", ["poison", "copy"])
@pytest.mark.parametrize("shape", [(3, 50, 3), (3, 50, 7), (3, 50, 0), (3, 50)])
def test_padding_never_touches_a_real_row(kind, shape):
    rs = np.random.RandomState(3)
    x = rs.standard_normal(shape).astype(np.float32)
    lengths = [50, 1, 17]
    y = NUM.pad_rows(x, lengths, kind)
    for i, l in enumerate(lengths):
        np.testing.assert_array_equal(y[i, :l], x[i, :l])
        if kind == "poison" and l < 50 and y[i, l:].size:
            assert not np.isfinite(y[i, l:l + 3]).any() and np.abs(y[i, l + 3]).max() == NUM.FAR
        if kind == "copy":
            np.testing.assert_array_equal(y[i, l:], x[i, np.arange(l, 50) % l])
    idx = rs.randint(0, 9, (3, 50, 3)).astype(np.int32)
    w = rs.random_sample((3, 50, 3)).astype(np.float32)
    ii, ww = NUM.pad_index_rows(idx, w, lengths, kind, 9)
    for i, l in enumerate(lengths):
        np.testing.assert_array_equal(ii[i, :l], idx[i, :l])
        np.testing.assert_array_equal(ww[i, :l], w[i, :l])
        assert (ii[i] >= 0).all() and (ii[i] < 9).all()
