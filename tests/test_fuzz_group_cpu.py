"""CPU checks of tests/fuzz_group_gpu.py and tests/group_regimes.py (no device).

The fixed slice (fuzz_group_gpu.SLICE_SEEDS, SLICE_ITERATIONS cases each) is replayed through group_regimes: every
reachable kernel instantiation of group.cu, interpolate.cu (but three_nn_kernel) and scatter_det.cu must be launched
by some case, with every named regime, and a second grid-stride trip for each gather family.  The restated
instantiation lists must match the launch sites of the .cu files, and the restated ordered sums must equal the C
oracle wherever the oracle's sequential sum is the contract (every unweighted list, weighted lists up to 256)."""
import os
import re

import numpy as np
import pytest

import fuzz_group_gpu as F
import group_regimes as R

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "pointnet2_b200", "csrc")


REQUIRED_REGIMES = {
    # group_point / group_concat
    "narrow_c1", "narrow_c2", "narrow_c3", "narrow_c4", "narrow_c0", "flat_b_over_65535",
    "vec4_channel_steps_1", "vec4_channel_steps_2", "vec4_rows_mod4_1", "vec4_rows_mod4_2", "vec4_rows_mod4_3",
    "rows_channel_steps_1", "rows_channel_steps_2",
    "concat_head_0", "concat_head_1", "concat_head_2", "concat_head_3", "concat_xyz_first", "concat_xyz_last",
    "concat_grouped_xyz", "concat_no_grouped_xyz", "misaligned_points", "misaligned_out",
    # ordered sums
    "build_one_cta", "build_count_scan_fill", "offsets_chunks_1", "offsets_chunks_2", "offsets_chunks_3",
    "empty_list", "long_weighted_finite", "long_seq_finite", "bucket_1", "bucket_2", "bucket_4", "bucket_8", "long_weighted", "long_seq",
    "gather_channel_passes_2", "gather_channel_passes_3", "long_channel_passes_3", "seq_channel_passes_2",
    "seq_flushes_1", "seq_flushes_2", "seq_flushes_3", "ragged_cut", "weighted_f32", "weighted_bf16", "weighted_f16",
    "unweighted_f32", "unweighted_bf16", "unweighted_f16", "targets_1023", "targets_1024", "targets_1025",
    "targets_16000", "targets_16001",
    # atomic gradients, interpolation, selection sort, refusals, torch
    "atomic_exact", "atomic_bound", "interp_ragged", "interp_dense",
    "sort_n_lt_32", "sort_n_32", "sort_n_gt_32", "sort_k_ge_n", "sort_nan_at_s", "sort_nan", "sort_ties",
    "refused_group_point_b", "refused_group_concat_b", "refused_grad_det_ws", "refused_interp_grad_det_ws",
    "refused_bad_dtype", "refused_null_idx", "refused_null_out", "refused_null_points", "autograd_det",
    "autograd_atomic",
}
# the gather families whose grid-stride loop must take a second trip in the slice
TRIP_FAMILIES = ["group_rows_vec4_kernel", "group_rows_kernel", "group_concat_vec_kernel", "group_narrow_kernel",
                 "group_point_grad", "three_interp_vec4_kernel", "three_interp_scalar_kernel", "three_interp_grad",
                 "gather_point_grad_kernel"]


def plans(p):
    """(launches, regimes) of one drawn case"""
    case, L, reg = p["case"], [], set()
    if case == "group_point":
        g, _ = R.group_point_impl(p["b"], p["n"], p["c"], p["m"], p["s"], p["fmt"], p["points_off"], p["out_off"])
        L.append(g)
        reg |= set(g["regimes"])
        reg |= {"misaligned_points"} if p["points_off"] else set()
        reg |= {"misaligned_out"} if p["out_off"] else set()
    elif case == "group_concat":
        g, _ = R.group_concat_impl(p["b"], p["n"], p["c"], p["m"], p["s"], p["fmt"], p["points_off"], 0)
        L.append(g)
        reg |= set(g["regimes"])
        if g["kernel"].startswith("group_concat_vec"):
            reg |= {f"concat_head_{h}" for h in R.concat_heads(p["c"], p["m"], p["s"], p["b"], p["xyz_first"])}
        reg.add("concat_xyz_first" if p["xyz_first"] else "concat_xyz_last")
        reg.add("concat_grouped_xyz" if p["with_gx"] else "concat_no_grouped_xyz")
    elif case == "ordered_grad":
        counts = F.ordered_counts(p)
        d = R.inv_scatter_det(p["weighted"], p["b"], p["nt"], p["c"], p["fmt"], counts, p["ragged"], p["off"], p["off"],
                              idx=p["idx"].reshape(p["b"], -1))
        L += [dict(kernel=k, trips=1) for k in d["launches"]]
        reg |= set(d["regimes"])
        reg.add(("weighted_" if p["weighted"] else "unweighted_") + p["fmt"])
        reg.add(f"targets_{p['nt']}")
        if p["finite"] and d["long_lists"]:
            reg.add("long_weighted_finite" if p["weighted"] else "long_seq_finite")
        if p["weighted"] and p["ragged"]:
            for k, l in enumerate(p["lengths"]):
                cut_differs = -(-3 * l // R.PIECES) != -(-3 * p["n"] // R.PIECES)
                if cut_differs and (counts[k] > R.SORT_CAP).any():
                    reg.add("ragged_cut")  # a long list in a cloud whose 3 * len cut is not the 3n one
    elif case == "atomic_grad":
        b, n, m, c = p["b"], p["n"], p["m"], p["c"]
        if p["which"] == "group_point":
            s = p["idx"].shape[2]
            L += R.group_point_grad_impl(b, n, c, m, s, p["fmt"], p["off"], p["off"])
        elif p["which"] == "three_interp":
            L.append(R.three_interpolate_grad_atomic(b, n, c, p["ragged"], p["off"], p["off"]))
        else:
            L += [R.gather_point(b, m), R.gather_point(b, m, grad=True)]
        reg.add("atomic_exact" if p["exact"] else "atomic_bound")
    elif case == "interp":
        L.append(R.three_interpolate_launch(p["b"], p["m"], p["c"], p["n"], p["fmt"], p["ragged"], p["off"], p["off"]))
        reg.add("interp_ragged" if p["ragged"] else "interp_dense")
    elif case == "selection_sort":
        L.append(dict(kernel="selection_sort_kernel", trips=1))
        n, k, d = p["n"], p["k"], p["d"]
        reg.add("sort_n_lt_32" if n < 32 else "sort_n_32" if n == 32 else "sort_n_gt_32")
        reg |= {"sort_k_ge_n"} if k >= n else set()
        nan = np.isnan(d)
        if nan[..., :min(k, n)].any():
            reg.add("sort_nan_at_s")
        if nan.any():
            reg.add("sort_nan")
        if (d == 0).any() and np.signbit(d[d == 0]).any() and (~np.signbit(d[d == 0])).any():
            reg.add("sort_ties")
    elif case == "refused":
        reg.add("refused_" + p["why"])
    elif case == "autograd":
        reg.add("autograd_det" if p["det"] else "autograd_atomic")
    elif case == "fp_front":
        g = R.fp_front_launch(p["b"], p["n"], p["m"], p["fmt"], p["ragged"])
        assert g["g"] == p["g"], (p["g"], g)  # the draw reaches the G it was meant for
        L.append(g)
    return L, reg


def replay():
    kernels, regimes, trips = set(), set(), {}
    for seed in F.SLICE_SEEDS:
        for p in F.draws(seed, F.SLICE_ITERATIONS):
            L, reg = plans(p)
            regimes |= reg
            for g in L:
                kernels.add(g["kernel"])
                fam = next((f for f in TRIP_FAMILIES if g["kernel"].startswith(f)), None)
                if fam:
                    trips[fam] = max(trips.get(fam, 0), g.get("trips", 1))
    return kernels, regimes, trips


@pytest.fixture(scope="module")
def reached():
    return replay()


def test_slice_reaches_every_instantiation(reached):
    kernels, _, _ = reached
    assert kernels <= set(R.INSTANCES), kernels - set(R.INSTANCES)
    missing = sorted(set(R.REACHABLE) - kernels)
    assert not missing, missing


def test_slice_reaches_every_regime(reached):
    _, regimes, _ = reached
    missing = sorted(REQUIRED_REGIMES - regimes)
    assert not missing, missing


def test_slice_takes_a_second_grid_stride_trip_in_every_gather_family(reached):
    _, _, trips = reached
    assert {f: trips.get(f, 0) >= 2 for f in TRIP_FAMILIES} == {f: True for f in TRIP_FAMILIES}, trips


def _launched(fname):
    """kernel instantiations launched in a .cu file: literal template arguments resolved, macro arguments as
    written (the names of the restatement are compared template by template)"""
    src = open(os.path.join(CSRC, fname)).read()
    return sorted(set(re.findall(r"\b(\w+_kernel)\s*(?:<[^<>]*(?:<[^<>]*>[^<>]*)*>)?\s*<<<", src)))


def test_restated_kernels_match_the_launch_sites():
    restated = {k.split("<")[0] for k in R.INSTANCES}
    launched = set()
    for f in ("group.cu", "interpolate.cu", "scatter_det.cu"):
        launched |= set(_launched(f))
    # kernels launched through a function pointer or macro carry their names in the template-argument text
    if "inv_build_kernel<true> : inv_build_kernel<false>" in open(os.path.join(CSRC, "scatter_det.cu")).read():
        launched.add("inv_build_kernel")
    others = {"three_nn_kernel"}  # interpolate.cu's three-NN search alone: fuzz_contracts_gpu
    assert launched - others == restated - others, (sorted(launched - others - restated), sorted(restated - launched))


def test_restated_template_arguments_match_the_literal_launches():
    src = open(os.path.join(CSRC, "group.cu")).read()
    vec = set(re.findall(r"group_rows_vec4_kernel<(\d+), R><<<", src))
    cat = set(re.findall(r"group_concat_vec_kernel<(\d+), R><<<", src))
    rows = set(re.findall(r"PN2_GROUP_ROWS\((\d+)\);", src))
    assert {f"group_rows_vec4_kernel<{v},4>" for v in vec} == {k for k in R.INSTANCES if k.startswith("group_rows_vec4")}
    assert {f"group_concat_vec_kernel<{v},2>" for v in cat} == {k for k in R.INSTANCES if k.startswith("group_concat_vec")}
    assert {int(v) for v in rows} == {int(k.split("<")[1].split(",")[0]) for k in R.INSTANCES
                                     if k.startswith("group_rows_kernel<")}
    det = open(os.path.join(CSRC, "scatter_det.cu")).read()
    assert re.search(r"kInvSortCap = %d;" % R.SORT_CAP, det) and re.search(r"kInvBuildMaxM = %d;" % R.BUILD_MAX_M, det)
    assert re.search(r"kSeqScan = %d;" % R.SEQ_SCAN, det) and re.search(r"kInvThreads = %d;" % R.INV_THREADS, det)


def test_concat_vec_lanes_cover_every_row_in_one_pass():
    """group_concat_vec_kernel's 'last lane loads the next pass's first vector' needs LPR < c4: every width the
    dispatcher sends it has LPR >= c4, so each row is one pass"""
    for c in range(0, 400):
        for b in (1, 3):
            g = R.launch_group_rows(True, b, c, 4, 8, "f32", True)
            if g["kernel"].startswith("group_concat_vec"):
                assert g["lpr"] >= g["c4"], c


def test_ordered_sum_matches_the_oracle_where_it_is_sequential():
    from oracle import oracle as O
    rs = np.random.RandomState(5)
    for _ in range(30):
        nt, n, c = int(rs.randint(1, 40)), int(rs.randint(1, 400)), int(rs.randint(1, 6))
        go = F.special_f32(rs, (n, c))
        idx = rs.randint(0, nt, n).astype(np.int32)
        a = R.ordered_sum(go, idx, nt)
        b = O.oracle_group_point_grad((1, nt, c), idx.reshape(1, n, 1), go.reshape(1, n, 1, c))[0]
        assert F.same_or_nan(a.view(np.uint32), b, "f32")
        w = F.special_f32(rs, (n, 3))
        i3 = rs.randint(0, nt, (n, 3)).astype(np.int32)
        a = R.ordered_sum(go, i3, nt, weight=w)
        b = O.oracle_three_interpolate_grad((1, nt, c), i3[None], w[None], go[None])[0]
        short = np.bincount(i3.ravel(), minlength=nt) <= R.SORT_CAP
        assert F.same_or_nan(a[short].view(np.uint32), b[short], "f32")


def test_long_weighted_lists_are_eight_ordered_pieces():
    """a hand case: one target with 300 entries, 2^25 first and 1.0 after it.  One sequential float32 sum loses every
    1.0 (half an ulp of 2^25 is 2); the eight pieces of ceil(300 / 8) = 38 entries keep the 1.0s of pieces 1..7 as
    exact sums of 38 or 34, and add them to 2^25 in piece order"""
    n = 100
    idx = np.zeros((n, 3), np.int32)
    w = np.ones((n, 3), np.float32)
    go = np.ones((n, 1), np.float32)
    w[0, 0] = 2.0 ** 25
    got = R.ordered_sum(go, idx, 1, weight=w)[0, 0]
    want = np.float32(2.0 ** 25)
    for p in range(1, 8):
        want = np.float32(want + np.float32(min(300, 38 * (p + 1)) - 38 * p))
    assert got == want and got != np.float32(2.0 ** 25)
    # at most 256 entries: one ascending sum, which loses them all
    assert R.ordered_sum(go[:85], idx[:85], 1, weight=w[:85])[0, 0] == np.float32(2.0 ** 25)


def test_selection_sort_oracle_nan_semantics():
    """the reference's scan: a NaN at position s stays; elsewhere NaN is never taken"""
    from oracle import oracle as O
    d = np.array([[[3, np.nan, 5, 1]]], np.float32)
    i, v = O.oracle_selection_sort(1, d)
    assert i.tolist() == [[[3, 1, 2, 0]]]
    i, v = O.oracle_selection_sort(4, np.array([[[np.nan, 2, 1, np.nan, 0]]], np.float32))
    assert i[0, 0].tolist() == [0, 4, 2, 3, 1]


def test_ragged_cut_is_visible_in_the_slice():
    """on some slice case the eight pieces cut from 3 * len give other bits than pieces cut from 3n: a kernel that cut
    a ragged cloud's long lists like a full one would fail there"""
    for seed in F.SLICE_SEEDS:
        for p in F.draws(seed, F.SLICE_ITERATIONS):
            if p["case"] != "ordered_grad" or not (p["weighted"] and p["ragged"] and p["finite"]):
                continue
            for k, l in enumerate(p["lengths"]):
                if l == p["n"]:
                    continue
                args = (p["go"][k, :l], p["idx"][k, :l], p["nt"])
                good = R.ordered_sum(*args, weight=p["w"][k, :l])
                bad = R.ordered_sum(*args, weight=p["w"][k, :l], cut=3 * p["n"])
                if not np.array_equal(good.view(np.uint32), bad.view(np.uint32)):
                    return
    pytest.fail("no slice case tells the 3 * len cut from the 3n cut")


def test_every_fp_front_instantiation_is_drawn_with_its_g():
    seen = set()
    for seed in F.SLICE_SEEDS:
        for p in F.draws(seed, F.SLICE_ITERATIONS):
            if p["case"] == "fp_front":
                seen.add(R.fp_front_launch(p["b"], p["n"], p["m"], p["fmt"], p["ragged"])["kernel"])
    assert seen == {k for k in R.INSTANCES if k.startswith("fp_front_kernel")}
