"""CPU checks of tests/fuzz_samplers_gpu.py and tests/select_regimes.py (no device).

The fixed slice (fuzz_samplers_gpu.SLICE_SEEDS, SLICE_ITERATIONS cases each) is replayed through select_regimes: every
select call of every case is traced with select_trace, and every named regime must be reached, the select's finishing
passes 0 to 5 and "no select" included.  select_trace must agree with np.sort; the planted collisions must still
collide; the restated constants must be those of the .cu sources; and the comparators of the fuzz must catch planted
defects."""
import os
import re

import numpy as np
import pytest

import crop_oracle as CO
import fuzz_samplers_gpu as F
import scan_oracle as SO
import select_regimes as R
import voxel_oracle as VO

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "pointnet2_b200", "csrc")

REQUIRED = (
    {f"select_pass{k}" for k in range(6)} | {"select_none"}
    | {f"{op}_select_pass{k}" for op in ("voxel", "shapes", "crops", "vscan") for k in (0, 1)}
    | {f"voxel_select_pass{k}" for k in (2, 3, 4, 5)} | {f"shapes_select_pass{k}" for k in (4, 5)}
    | {f"{op}_select_none" for op in ("voxel", "shapes", "crops", "vscan")}
    | {"voxel_warp_w1", "voxel_warp_w2", "voxel_warp_w4", "voxel_warp_seeded", "voxel_warp_rows", "voxel_empty_cell",
       "voxel_cta", "voxel_cta_seeded", "voxel_cta_rows", "voxel_cta_reuse", "voxel_no_cta_launch", "voxel_s_not_x32"}
    | {f"voxel_c{v}" for v in (1, 31, 32, 33, 64, 65, 127, 128)}
    | {"voxel_pillars", "voxel_voxels", "voxel_nan", "voxel_quotient_in_minus1_0", "voxel_out_of_grid",
       "voxel_lengths_0", "voxel_lengths_1", "voxel_lengths_lt_n", "voxel_lengths_n", "voxel_lengths_out_of_range",
       "voxel_dense"} | {"voxel_kind_" + k for k in F.VOXEL_KINDS}
    | {"voxel_c_eq_m", "voxel_c_eq_m_plus_1", "voxel_m1", "voxel_m_max", "voxel_m_pow2", "voxel_m_pow2_plus_1"}
    | {"shapes_subset_first", "shapes_subset_random", "shapes_votes", "shapes_normals", "shapes_no_normals",
       "shapes_parts", "shapes_no_parts", "shapes_dropout", "shapes_no_dropout", "shapes_out_of_range",
       "shapes_pool_lt_npoints", "shapes_c_eq_m", "shapes_c_eq_m_plus_1", "shapes_m1", "shapes_m_pow2",
       "shapes_compact_over_1024"}
    | {"crops_npoints_" + k for k in ("below", "equal", "one_under", "far_under")}
    | {"crops_attempt9", "crops_unlabelled", "crops_duplicates", "crops_out_of_range", "crops_m_max",
       "crops_compact_over_1024", "crops_c_eq_m", "crops_c_eq_m_plus_1", "crops_rotate", "crops_dropout"}
    | {"vscan_few_near", "vscan_invalid", "vscan_vis_gt_npoints", "vscan_vis_le_npoints", "vscan_out_of_range",
       "vscan_sparse_select"} | {f"vscan_mode_{m}" for m in range(-1, 8)}
    | {"seed_" + k for k in ("negative", "high", "small", "device")} | {"api_c", "api_wrapper"}
    | {"refused_" + w for w in F.REFUSALS})


def _select(op, keys, m, reg):
    tr = R.select_trace(keys, m)
    assert tr["gathered"] == m, (op, len(keys), m)
    assert np.array_equal(tr["out"], np.sort(np.asarray(keys, np.uint64))[:m]), (op, len(keys), m)
    assert tr["pass"] == R.boundary_pass(keys, m)
    tag = "none" if tr["pass"] is None else f"pass{tr['pass']}"
    reg |= {f"select_{tag}", f"{op}_select_{tag}"} | R.edge_regimes(len(keys), m, op)


def voxel_regimes(p):
    b, n, dim, dims, S = p["b"], p["n"], p["dim"], p["dims"], p["nsample"]
    cells = dim ** dims
    reg = {"voxel_pillars" if dims == 2 else "voxel_voxels", "voxel_kind_" + p["kind"]}
    count = np.zeros((b, cells), np.int64)
    members = []
    for i in range(b):
        ln = n if p["lengths"] is None else min(max(int(p["lengths"][i]), 0), n)
        if p["lengths"] is None:
            reg.add("voxel_dense")
        else:
            raw = int(p["lengths"][i])
            reg.add({0: "voxel_lengths_0", 1: "voxel_lengths_1", n: "voxel_lengths_n"}.get(raw, "voxel_lengths_lt_n"
                                                                                          if 0 < raw < n else
                                                                                          "voxel_lengths_out_of_range"))
        pts = p["xyz"][i, :ln]
        cell = VO.cells_of(pts, dim, p["radius"], dims)
        q = (pts[:, :dims] + np.float32(p["radius"])) / np.float32(2 * p["radius"] / dim)
        if np.isnan(pts).any():
            reg.add("voxel_nan")
        with np.errstate(invalid="ignore"):
            if ((q > -1) & (q < 0)).any():
                reg.add("voxel_quotient_in_minus1_0")
            if ((q >= dim) | (q <= -1)).any():
                reg.add("voxel_out_of_grid")
        count[i] = np.bincount(cell[cell >= 0], minlength=cells)
        members.append(cell)
    plan = R.voxel_plan(count, n, S)
    reg |= plan["regimes"]
    assert plan["smem"] == 8 * R.pow2_at_least(S)
    for e, c, _ in plan["selects"]:
        i, cell = divmod(e, cells)
        rows = np.nonzero(members[i] == cell)[0]
        keys = VO.order_keys(rows, np.ones(len(rows), bool), p["seed"] & R.M64, np.full(len(rows), e))
        _select("voxel", keys, S, reg)
    flat = count.reshape(-1)
    for e in np.nonzero((flat > 0) & (flat <= S))[0]:
        reg |= {"select_none", "voxel_select_none"} | R.edge_regimes(int(flat[e]), int(flat[e]), "voxel")
    for e in np.nonzero((flat > S) & (flat <= R.WARP_CELL))[0]:  # sorted whole by one warp
        reg |= R.edge_regimes(int(flat[e]), S, "voxel")
    return reg


def shapes_regimes(p):
    reg = {"shapes_subset_" + p["subset"], "shapes_normals" if p["with_normals"] else "shapes_no_normals",
           "shapes_parts" if p["parts"] else "shapes_no_parts",
           "shapes_dropout" if p["max_dropout"] > 0 else "shapes_no_dropout"}
    if p["votes"]:
        reg.add("shapes_votes")
    sizes = np.asarray(p["sizes"])
    if ((p["shape_idx"] < 0) | (p["shape_idx"] >= len(sizes))).any():
        reg.add("shapes_out_of_range")
    plan = R.shapes_plan(sizes, p["shape_idx"], p["npoints"], p["subset"] == "random", p["votes"])
    if plan["pool"] < p["npoints"]:
        reg.add("shapes_pool_lt_npoints")
    assert plan["smem"] == 8 * R.pow2_at_least(min(plan["pool"], p["npoints"]))
    for e, (q, m, sel) in enumerate(plan["entries"]):
        if q == 0:
            continue
        if sel:
            _select("shapes", R.row_keys(p["seed"], R.STREAM["shapes"], e, np.arange(q)), m, reg)
        else:
            reg |= {"select_none", "shapes_select_none"} | R.edge_regimes(q, m, "shapes")
    return reg


def crops_regimes(p):
    reg = {"crops_npoints_" + p["npoints_kind"]} | {"crops_" + k for k in p["kinds"] if k != "room"}
    reg |= {"crops_rotate"} if p["rotate"] else set()
    reg |= {"crops_dropout"} if p["max_dropout"] > 0 else set()
    for b, s in enumerate(p["crop_scene"]):
        if not 0 <= s < len(p["scenes"]):
            reg.add("crops_out_of_range")
            continue
        pts, lab = p["scenes"][s]
        att = CO.crop_attempts(pts, lab, pts[:, 2].min(), pts[:, 2].max(), p["seed"], b)
        a = CO.choose(att)
        if not att[a]["valid"]:
            reg.add("crops_attempt9")
        mem = att[a]["members"]
        c, m = len(mem), min(len(mem), p["npoints"])
        if c > m:
            _select("crops", R.row_keys(p["seed"], R.STREAM["crops"], b, mem), m, reg)
        else:
            reg |= {"select_none", "crops_select_none"} | R.edge_regimes(c, m, "crops")
    return reg


def vscan_regimes(p):
    reg = set()
    for b, (s, mode) in enumerate(zip(p["scan_scene"], p["scan_mode"])):
        if not 0 <= s < len(p["scenes"]):
            reg.add("vscan_out_of_range")
            continue
        pts = p["scenes"][s][0]
        reg.add(f"vscan_mode_{int(mode)}")
        got = SO.scan(pts, pts.astype(np.float64).mean(0), int(mode),
                      SO.view_draws(p["seed"], b) if mode == -1 else None)
        vis = got["smpidx"]
        if got["near"] < SO.MIN_NEAR:
            reg.add("vscan_few_near")
        if len(vis) < p["min_points"]:
            reg.add("vscan_invalid")
        m = min(len(vis), p["npoints"])
        if len(vis) > p["npoints"]:
            reg.add("vscan_vis_gt_npoints")
            if len(vis) < len(pts):
                reg.add("vscan_sparse_select")  # n = ps rows, c = vis of them set in the bitmap
            _select("vscan", R.row_keys(p["seed"], R.STREAM["vscan"], b, vis), m, reg)
        else:
            reg |= {"vscan_vis_le_npoints", "select_none", "vscan_select_none"}
    return reg


def refused_regimes(p):
    reg = set()
    for why in p["whys"]:
        op, rest = why.split("_", 1)
        bad = {"npoints_0": 0, "npoints_16385": R.MAX_ROWS + 1, "nsample_0": 0, "nsample_16385": R.MAX_ROWS + 1}
        if op == "voxel":
            b, n, dim, S = (2, 1 << 30, 3, 32) if rest == "bn_2_31" else (2, 300, 1025, 32) if rest == "bc_2_31" else \
                (1, 300, 3, bad.get(rest, 32))
            wsb = R.voxel_workspace_bytes(1, 300, 3, 3) - (rest == "ws_short")
            assert R.voxel_refusal(b, n, dim, 3, 1.0, S, wsb, rest != "ws_misaligned"), why
            assert R.voxel_refusal(1, 300, 3, 3, 1.0, 32, wsb + 1, True) is None
        elif op == "shapes":
            b, npts = (65536, R.MAX_ROWS) if rest == "be_2_31" else (2, bad[rest])
            assert R.shapes_refusal(100, b, 0, npts, False), why
            assert R.shapes_refusal(100, 2, 0, 64, False) is None
        elif op == "crops":
            b, npts = (65535, R.MAX_ROWS) if rest == "bn_2_31" else (2, bad.get(rest, 64))
            wsb = R.crops_workspace_bytes(2, 64) - (rest == "ws_short")
            assert R.crops_refusal(b, npts, wsb, rest != "ws_misaligned", 0.5), why
            assert R.crops_refusal(2, 64, wsb + 1, True, 0.5) is None
        else:
            b, npts = (R.SCAN_MAX_BATCH + 1, 64) if rest == "b_4097" else (2, bad.get(rest, 64))
            wsb = R.vscan_workspace_bytes(2, 100, 64) - (rest == "ws_short")
            assert R.vscan_refusal(b, 100, npts, wsb, rest != "ws_misaligned", 300), why
            assert R.vscan_refusal(2, 100, 64, wsb + 1, True, 300) is None
        reg.add("refused_" + why)
    return reg


REGIMES = {"voxel": voxel_regimes, "voxel_planted": voxel_regimes, "shapes": shapes_regimes,
           "shapes_planted": shapes_regimes, "crops": crops_regimes, "vscan": vscan_regimes,
           "refused": refused_regimes}


def case_regimes(p):
    reg = REGIMES[p["case"]](p)
    if "seed_kind" in p:
        reg |= {"seed_" + p["seed_kind"], "api_" + p["api"]}
    return reg


@pytest.fixture(scope="module")
def slice_regimes():
    reached = {}
    for seed in F.SLICE_SEEDS:
        for it, p in enumerate(F.draws(seed, F.SLICE_ITERATIONS)):
            for r in case_regimes(p):
                reached.setdefault(r, (seed, it))
    return reached


def test_slice_reaches_every_regime(slice_regimes):
    missing = sorted(REQUIRED - set(slice_regimes))
    assert not missing, missing


def test_planted_cells_finish_at_their_pass():
    for seed in F.SLICE_SEEDS:
        for p in F.draws(seed, F.SLICE_ITERATIONS):
            if p["case"] not in ("voxel_planted", "shapes_planted"):
                continue
            reg = case_regimes(p)
            op = p["case"].split("_")[0]
            for want in p["planted"].values():
                assert f"{op}_select_pass{want}" in reg, (p["case"], want)


def test_select_trace_agrees_with_sort():
    rs = np.random.RandomState(3)
    for _ in range(60):
        c = int(rs.choice([1, 2, 3, 100, 1025, 5000, 40000]))
        keys = np.unique(rs.randint(0, 1 << 63, c, dtype=np.int64).astype(np.uint64) << np.uint64(rs.randint(0, 2)))
        m = int(rs.randint(1, len(keys) + 1))
        tr = R.select_trace(keys, m)
        assert np.array_equal(tr["out"], np.sort(keys)[:m]) and tr["gathered"] == m
        assert tr["select"] == (len(keys) > m) and tr["sort_n"] == R.pow2_at_least(m)
        assert tr["pass"] == R.boundary_pass(keys, m)
    # the m-th and (m+1)-th orders differing first in bit 53, 42, 32, 21, 10 or 0: every finishing pass
    for ps, shift in enumerate((53, 42, 32, 21, 10, 0)):
        top = int(rs.randint(1 << 62)) << 2 | 1 << 63
        a = top >> (shift + 1) << (shift + 1) | (int(rs.randint(1 << 20)) & ((1 << shift) - 1))  # bit `shift` clear
        b = a | 1 << shift
        low = [int(rs.randint(0, 1 << 62)) % a for _ in range(40)]
        high = [b + 1 + int(rs.randint(0, (R.M64 - b) // 2)) for _ in range(40)]
        keys = np.unique(np.array(low + [a, b] + high, np.uint64))
        m = int((keys <= np.uint64(a)).sum())
        tr = R.select_trace(keys, m)
        assert tr["pass"] == ps and np.array_equal(tr["out"], np.sort(keys)[:m]), (ps, tr["pass"])


def test_planted_constants_still_collide():
    for (op, ps), (seed, e, j1, j2) in R.PLANTED.items():
        stream = R.STREAM[op]
        k = R.row_keys(seed, stream, e, [j1, j2]) >> np.uint64(32)
        assert k[0] == k[1], (op, ps)
        assert R.pair_pass(j1, j2) == ps
        if op == "voxel":
            lo, cnt = R.VOXEL_WINDOW
            assert lo <= j1 < j2 < lo + cnt <= F.PLANT_N
        else:
            assert j2 < R.MAX_ROWS
    # the search that found them (one (seed, entry) of each is enough)
    assert (2019872, 2283615) in R.collisions(7, 9, 0, *R.VOXEL_WINDOW)
    assert (14608, 15333) in R.collisions(4, 1, 15, 0, R.MAX_ROWS)


def _const(path, name):
    src = open(os.path.join(CSRC, path)).read()
    m = re.search(rf"\b{name}\s*=\s*(\d+)", src)
    assert m, (path, name)
    return int(m.group(1))


def test_constants_match_the_sources():
    assert _const("pn2_common.cuh", "kSelectMaxRows") == R.MAX_ROWS
    assert _const("pn2_common.cuh", "kSelectRadixBins") == R.RADIX_BINS == 2 * R.SELECT_THREADS
    assert _const("voxel.cu", "kWarpKeys") == R.WARP_KEYS
    assert _const("voxel.cu", "kCtaThreads") == R.SELECT_THREADS
    assert _const("voxel.cu", "kRowThreads") == R.ROW_THREADS and _const("voxel.cu", "kWarpThreads") == R.WARP_THREADS
    assert _const("voxel.cu", "kStreamCell") == R.STREAM["voxel"] == VO.STREAM_CELL
    assert _const("shapes.cu", "kShapeThreads") == R.SELECT_THREADS
    assert _const("shapes.cu", "kStreamKey") == R.STREAM["shapes"]
    assert _const("crops.cu", "kSelectThreads") == R.SELECT_THREADS
    assert _const("crops.cu", "kKeyWords") == R.KEY_WORDS and _const("crops.cu", "kAttempts") == R.ATTEMPTS
    assert "rng_row_key(seed, 2," in open(os.path.join(CSRC, "crops.cu")).read() and R.STREAM["crops"] == CO.STREAM_KEY
    assert _const("vscan.cu", "kSelectThreads") == R.SELECT_THREADS
    assert _const("vscan.cu", "kStreamKey") == R.STREAM["vscan"] == SO.STREAM_KEY
    assert _const("vscan.cu", "kScanMaxBatch") == R.SCAN_MAX_BATCH
    src = open(os.path.join(CSRC, "pn2_common.cuh")).read()
    assert "pass % 3 == 2 ? 10 : 11" in src and "pass < 6" in src  # the digit widths of WIDTHS
    assert "n / (kWarpCell + 1)" in open(os.path.join(CSRC, "voxel.cu")).read()  # big_cap of voxel_layout


def _oracle_voxel_case():
    rs = np.random.RandomState(5)
    xyz = rs.uniform(-1, 1, (2, 3000, 3)).astype(np.float32)
    p = dict(xyz=xyz, dim=3, radius=1.0, nsample=150, seed=9, dims=3, lengths=None)
    return F.want_voxel(p)


def test_comparators_catch_planted_defects():
    want = _oracle_voxel_case()
    fields = ("count", "idx", "grouped")
    ok = {k: v.copy() for k, v in want.items()}
    assert F.compare(ok, want, fields) == []
    full = np.argwhere(want["count"] > 1)
    i, c = full[0]
    # two rows of a cell swapped
    g = {k: v.copy() for k, v in want.items()}
    g["idx"][i, c, [0, 1]] = g["idx"][i, c, [1, 0]]
    assert "idx" in F.compare(g, want, fields)
    # a wrong row index
    g = {k: v.copy() for k, v in want.items()}
    g["idx"][i, c, 0] += 1
    assert "idx" in F.compare(g, want, fields)
    # one row too many in a cell
    g = {k: v.copy() for k, v in want.items()}
    g["count"][i, c] += 1
    assert "count" in F.compare(g, want, fields)
    # a guard written past the end
    g = dict(ok, guards={"idx": False})
    assert F.compare(g, want, fields) == ["idx"]
    # the last pad row of a ragged batch left as poison: exact and ulp fields
    pidx = np.full((2, 5), -1, np.int32)
    pidx[0, :3] = [4, 9, 2]
    wantp = dict(point_idx=pidx, xyz=np.zeros((2, 5, 3), np.float32), lengths=np.array([3, 0], np.int32))
    g = {k: v.copy() for k, v in wantp.items()}
    g["point_idx"][0, 4] = np.frombuffer(bytes([F.POISON] * 4), np.int32)[0]
    assert "point_idx" in F.compare(g, wantp, ("point_idx", "lengths"))
    g = {k: v.copy() for k, v in wantp.items()}
    g["xyz"][0, 4] = np.frombuffer(bytes([F.POISON] * 12), np.float32)
    assert "xyz" in F.compare(g, wantp, (), {"xyz": wantp["xyz"].astype(np.float64)})
    # one row too many in an entry
    g = {k: v.copy() for k, v in wantp.items()}
    g["lengths"][0] = 4
    g["point_idx"][0, 3] = 7
    assert set(F.compare(g, wantp, ("point_idx", "lengths"))) == {"point_idx", "lengths"}
    # flags read back as bytes: a poisoned flag is not "true"
    assert F.compare({"valid": np.array([F.POISON], np.uint8)}, {"valid": np.array([True])}, ("valid",)) == ["valid"]


def test_workspace_restatements_follow_the_layouts():
    assert R.voxel_workspace_bytes(1, 128, 3, 3) == R.voxel_layout(1, 128, 27)["total"]
    assert R.voxel_layout(1, 128, 27)["big_cap"] == 0 and R.voxel_layout(2, 129, 27)["big_cap"] == 2
    assert R.voxel_workspace_bytes(2, 1 << 30, 3, 3) == 0 and R.voxel_workspace_bytes(2, 10, 1025, 3) == 0
    assert R.crops_workspace_bytes(65535, R.MAX_ROWS) == 0 and R.crops_workspace_bytes(1, 1) % 256 == 0
    assert R.vscan_workspace_bytes(R.SCAN_MAX_BATCH + 1, 10, 10) == 0 and R.vscan_workspace_bytes(1, 1, 1) % 256 == 0
