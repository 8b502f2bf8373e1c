"""Without a GPU: the fixed-seed slice of tests/fuzz_fps_gpu.py reaches every FPS kernel, every stage where a kernel
decides a tie, and every data regime.  The draws are replayed with numpy and the C oracle's step trace
(``oracle_fps_trace``), and tests/fps_regimes.py says which kernel runs each case and which stage decides each tie.  A
new instantiation in csrc/fps.cu, or a draw that stops reaching a kernel, a tie stage or a regime, fails here before a
GPU is needed."""
import os
import re

import numpy as np
import pytest

import fps_regimes as R
import fuzz_fps_gpu as F
from oracle import oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INST = {i.name: i for i in R.INSTANCES}
UNDERFLOW = np.float32(2.0 ** -75)  # a difference at most this large squares to 0 (2^-150 rounds to even)


def macro_lists():
    """the X(...) argument tuples of each PN2_FPS_*_KERNELS macro in csrc/fps.cu"""
    src = open(os.path.join(ROOT, "pointnet2_b200", "csrc", "fps.cu")).read()
    out = {}
    for name in ("CTA", "CLUSTER", "BIG"):
        m = re.search(r"#define PN2_FPS_%s_KERNELS\(X\)((?:[^\n]*\\\n)*[^\n]*)" % name, src)
        assert m, name
        out[name] = [tuple(int(v) for v in a.split(",")) for a in re.findall(r"X\(([\d,\s]+)\)", m.group(1))]
    return out


def test_restated_kernel_lists_equal_fps_cu():
    got = macro_lists()
    assert got["CTA"] == R.CTA_KERNELS
    assert got["CLUSTER"] == R.CLUSTER_KERNELS
    assert got["BIG"] == R.BIG_KERNELS
    n_cta = sum(1 + pk for _, _, pk in R.CTA_KERNELS)
    n_cluster = sum(1 + pk for *_, pk in R.CLUSTER_KERNELS)
    assert len(R.INSTANCES) == n_cta + n_cluster + 2 * len(R.BIG_KERNELS) + 1 == 69
    assert len(set(R.INSTANCES)) == len(R.INSTANCES)
    assert {i for i, _ in F.COMBOS} == set(R.INSTANCES) - {R.INSTANCES[-1]}


# ------------------------------------------------------------------------------------------------ the replay
def empty_tags(inst, C, length):
    """threads (and CTAs of a cluster) that hold none of the cloud's points"""
    tags = set()
    per_cta = inst.T
    if length < per_cta * (C if inst.family in ("cluster", "big") else 1):
        tags.add("empty_threads")
    if inst.family in ("cluster", "big") and length <= inst.T * (C - 1):
        tags.add("empty_ctas")
    return tags


def cloud_tags(inst, C, c, m, kind):
    """the trace of one cloud c (1, L, 3): its tie stages under inst and its data regimes; and whether the trace's picks
    are oracle_fps's"""
    idx, top, count, tied = O.oracle_fps_trace(m, c)
    same = np.array_equal(idx, O.oracle_fps(m, c))
    L = c.shape[1]
    tags = set()
    if m > 1:
        t, cnt, tied = top[0, 1:], count[0, 1:], tied[0, 1:]
        fk = R.family_key(inst)
        rows = np.nonzero(cnt >= 2)[0]
        if len(rows):
            others = tied[rows, 1:]
            winners = np.broadcast_to(tied[rows, :1], others.shape)
            keep = others >= 0
            tags |= {f"stage:{fk}:{s}" for s in set(R.stages(inst, winners[keep], others[keep], C))}
        picks = idx[0, 1:]
        if (t == np.float32(1e38)).any():
            tags.add("win_1e38")
        if (t == 0).any():
            tags.add("max_zero")
        if np.isnan(c[0, picks]).any():
            tags.add("pick_nan")
        if np.isinf(c[0, picks]).any():
            tags.add("pick_inf")
        if L > 1 and (picks == L - 1).any():
            tags.add("winner_last")
        if kind in ("tiny", "ball_Z"):
            with np.errstate(invalid="ignore"):
                for q in np.unique(idx[0, :-1]):
                    d = np.abs((c[0] - c[0, q]).astype(np.float32)).max(1)
                    if ((d > 0) & (d <= UNDERFLOW)).any():
                        tags.add("underflow_zero")
                        break
    if np.isnan(c[0, 0]).any():
        tags.add("nan_point0")
    return tags, same


def case_inst(p):
    """(instantiation, cluster size) a case runs"""
    if p["case"] == "fps_forced":
        return INST[p["inst"]], p["C"]
    if p["case"] == "fps_scratch":
        return R.INSTANCES[-1], 1
    plan = R.plan_fps(p["b"], p["n"], capacity=R.h100_capacity)
    inst, why = R.dispatch(plan, p["n"])
    assert why is None, (p["b"], p["n"], plan, why)
    return inst, max(plan.cluster, 1)


def regimes(p):
    """(the named regimes one case reaches, whether every trace matched oracle_fps)"""
    b, n, m, lens = p["b"], p["n"], p["npoint"], p["lens"]
    if p["case"] == "fps_refused":
        return {"refused_" + p["why"]}, True
    inst, C = case_inst(p)
    mode = "ragged" if lens else "dense"
    tags = {f"ran:{inst.name}:{mode}", "kind_" + p["kind"]}
    if p["case"] == "fps_builtin":
        tags |= {"builtin_" + inst.family, f"builtin_{inst.family}_{mode}"}
    if inst.family in ("cluster", "big"):
        tags.add(f"C_{C}")
        if inst.family == "big" and C & (C - 1):
            tags.add("big_C_nonpow2")
    for name, v in (("1", 1), ("2", 2), ("n-1", n - 1), ("n", n), ("n+3", n + 3)):
        if m == v:
            tags.add("npoint_" + name)
    ls = lens["lengths"] if lens else [n] * b
    if lens:
        raw = lens["raw"]
        if any(r < 1 for r in raw):
            tags.add("len_clamped_low")
        if any(r > n for r in raw):
            tags.add("len_clamped_high")
        if 1 in ls:
            tags.add("len_1")
        if min(ls) < m:
            tags.add("len_lt_npoint")
        if min(ls) < n:
            tags.add(f"ragged_short_{inst.family}")
    if inst.family == "scratch" and b > R.SCRATCH_GRID:
        tags.add("scratch_reuse")
        if any(ls[i + R.SCRATCH_GRID] < ls[i] for i in range(b - R.SCRATCH_GRID)):
            tags.add("scratch_short_after_long")
    ok = True
    for i, ln in enumerate(ls):
        t, same = cloud_tags(inst, C, p["xyz"][i:i + 1, :ln], m, p["kind"])
        tags |= t | empty_tags(inst, C, ln)
        ok = ok and same
    return tags, ok


@pytest.fixture(scope="module")
def slice_params():
    return [p for seed in F.SLICE_SEEDS for p in F.draws(seed, F.SLICE_ITERATIONS)]


@pytest.fixture(scope="module")
def slice_replay(slice_params):
    return [regimes(p) for p in slice_params]


REQUIRED = {
    # the tie stages of each family, as its layout has them
    *{f"stage:{fk}:{s}" for fk, ss in R.STAGES.items() for s in ss},
    # cluster sizes
    "C_2", "C_4", "C_8", "C_16", "big_C_nonpow2",
    # the planner's own choice reaches every family, dense and ragged
    "builtin_cta_dense", "builtin_cta_ragged", "builtin_cluster_dense", "builtin_cluster_ragged", "builtin_big",
    "builtin_scratch",
    # the dispatcher's refusals
    *{"refused_" + w for w in F.REFUSALS},
    # data regimes
    "win_1e38", "pick_nan", "pick_inf", "nan_point0", "max_zero", "underflow_zero", "winner_last", "empty_threads",
    "empty_ctas", "len_clamped_low", "len_clamped_high", "len_1", "len_lt_npoint", "scratch_reuse",
    "scratch_short_after_long", "ragged_short_cta", "ragged_short_cluster", "ragged_short_big",
    "npoint_1", "npoint_2", "npoint_n-1", "npoint_n", "npoint_n+3",
    "kind_nan0", "kind_big", "kind_tiny", "kind_negzero", "kind_same", "kind_lattice2", "kind_ball_X", "kind_G", "kind_D",
}


def test_trace_picks_are_oracle_fps(slice_replay):
    assert all(ok for _, ok in slice_replay)


def test_slice_runs_every_instantiation_dense_and_ragged(slice_replay):
    seen = set().union(*(t for t, _ in slice_replay))
    want = {f"ran:{i.name}:{mode}" for i in R.INSTANCES for mode in ("dense", "ragged")}
    assert want <= seen, sorted(want - seen)


def test_slice_reaches_every_regime(slice_replay):
    seen = set().union(*(t for t, _ in slice_replay))
    assert REQUIRED <= seen, sorted(REQUIRED - seen)


def test_each_seed_forces_every_combination_once(slice_params):
    per_seed = len(slice_params) // len(F.SLICE_SEEDS)
    for s, seed in enumerate(F.SLICE_SEEDS):
        forced = [p for p in slice_params[s * per_seed:(s + 1) * per_seed] if p["case"] == "fps_forced"]
        assert len(forced) == len(F.COMBOS)
        assert {(p["inst"], p["lens"] is not None) for p in forced} == {(i.name, r) for i, r in F.COMBOS}


def test_draws_are_reproducible_and_bounded(slice_params):
    a, b = F.draws(F.SLICE_SEEDS[0], 10), F.draws(F.SLICE_SEEDS[0], 10)
    for p, q in zip(a, b):
        assert F.public(p) == F.public(q)
        assert np.array_equal(p["xyz"].view(np.int32), q["xyz"].view(np.int32))
    for p in slice_params:
        assert p["xyz"].dtype == np.float32 and p["xyz"].shape == (p["b"], p["n"], 3)
        if p["case"] != "fps_refused":
            assert p["npoint"] <= 8 or p["b"] * p["n"] * p["npoint"] <= F.MAX_WORK


def test_stage_classifier_by_hand():
    """Hand-placed pairs: each stage of each layout"""
    cta_plain = R.Inst("cta", 4, 128, 4, 0)  # DD = 4 residues, one point per residue
    assert R.stages(cta_plain, 0, [128, 1, 32]) == ["residue", "warp", "cross_warp"]
    cta_512 = R.Inst("cta", 16, 512, 16, 1)  # DD = 1, Q = 16, GS = 4: groups j // 4
    assert R.stages(cta_512, 0, [512 * 3, 512 * 4, 5]) == ["group", "group_other", "warp"]
    cta_256 = R.Inst("cta", 16, 256, 16, 1)  # DD = 2, Q = 8, GS = 4: residues alternate with j
    assert R.stages(cta_256, 0, [256 * 2, 256 * 8, 256]) == ["group", "group_other", "residue"]
    cl = R.Inst("cluster", 32, 512, 16, 0)  # k = t + 512 (r + C j)
    assert R.stages(cl, 0, [512 * 2 * 3, 512 * 2 * 16, 512, 64], C=2) == ["scan", "reg_stream", "cluster", "cross_warp"]
    big = R.Inst("big", 44, 512, 16, 1)
    assert R.stages(big, 7, [7 + 512 * 3 * 2, 7 + 512 * 3 * 4, 7 + 512 * 3 * 16], C=3) == ["group", "group_other",
                                                                                             "reg_stream"]
    assert R.stages(R.INSTANCES[-1], 3, [3 + 1024, 4, 3 + 64]) == ["scan", "warp", "cross_warp"]


def test_decoded_overrides():
    d = R.decode_override
    assert d(0, 16, 1) is None
    assert d(256, 16, -1) == R.Plan(256, 16, 1, 16, 0)
    assert d(256, 16, -2) == R.Plan(256, 16, 1, 16, 1)
    assert d(514, 32, 4) == R.Plan(512, 32, 4, 16, 0)   # +2: plain; 512 x 32: half the coordinates streamed
    assert d(257, 32, 4) == R.Plan(256, 32, 4, 32, 1)
    assert d(512, 44, 3, packed_cluster=0) == R.Plan(512, 44, 3, 16, 0)
    assert R.dispatch(d(512, 48, 3), 512 * 48 * 3)[0] == R.Inst("big", 48, 512, 12, 1)
    assert R.dispatch(d(512, 48, 3), 512 * 48 * 3 + 1) == (None, "capacity")


# ------------------------------------------------------------------------------------------- the planner sweep
def sweep_sizes():
    ns = {128, 256, 512, 1024, 2048, 4096, 8192, 262144, 512 * 52 * 16}
    for C in range(2, 17):
        ns.add(1024 * C)
        ns |= {512 * p * C for p in (44, 48, 52)}
    for C in (2, 4, 8, 16):
        t = 128 if C >= 4 else 256
        ns |= {C * t * pp for pp in (2, 4, 8, 16, 32)} | {C * 256 * 32, C * 512 * 32}
    return sorted({v + d for v in ns for d in (-1, 0, 1)})


def test_plan_equals_the_library_plan_over_every_threshold():
    """pn2_fps_plan against plan_fps at every threshold +- 1.  Without a device the library plans with 132 SMs and
    capacity 0; with one, with its SM count and pn2_fps_cluster_capacity."""
    import torch

    from pointnet2_b200 import _lib
    lib = _lib.load()
    lib.pn2_set_fps_config(0, 0, 0)
    sms, cap = R.SMS, None
    if torch.cuda.is_available():
        sms = torch.cuda.get_device_properties(0).multi_processor_count
        cap = F.live_capacity(lib)
    bad = []
    for b in (1, 2, 3, 5, 8, 9, 16, 17, 33, 66, 67, 132, 133, 500):
        for n in sweep_sizes():
            want = R.plan_fps(b, n, sms=sms, capacity=cap)
            got = F.device_plan(lib, b, n)
            if got != (want.threads, want.ppt, want.cluster):
                bad.append((b, n, got, want))
    assert not bad, bad[:10]
