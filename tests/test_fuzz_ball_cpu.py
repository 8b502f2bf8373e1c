"""Without a GPU: the fixed-seed slice of tests/fuzz_ball_gpu.py reaches every regime of the three ball-query kernels.
The draws are replayed with numpy and the C oracle only (oracle_fps gives the layer's centroids), and every cloud and
query is tagged by tests/ball_regimes.py.  A draw that stops reaching a branch fails here, before a GPU is needed."""
import numpy as np
import pytest

import ball_regimes as R
import fuzz_ball_gpu as F
from oracle import oracle as O


def _bg_tags(pts, q, radius, nsample, stride):
    """ball_group_kernel on one cloud: cloud tags and the union of the query tags, prefixed bg_"""
    cl = R.BgCloud(pts, radius, stride)
    tags = {"bg_cloud_" + cl.reason}
    if cl.use_grid:
        tags.add("bg_dual" if cl.dual else "bg_single_layout")
    hits = R.hit_rows(radius, pts, q)
    for j in range(len(q)):
        tags |= {"bg_" + t for t in R.bg_query(cl, q[j], hits[j], nsample)}
    return tags


def _geo_tags(pts, radius):
    g = R.geometry(pts, radius)
    tags = set()
    if not g["finite_box"]:
        tags.add("geo_nonfinite_box")
    elif np.any(g["ext"] == 0):
        tags.add("geo_degenerate_axis")
    if np.isnan(pts).all(0).any():
        tags.add("geo_nan_axis")
    if max(g["dims"]) == R.MAX_DIM:
        tags.add("geo_dims_16")
    return tags


def _global_tags(x, q, radius, nsample, group):
    """the global-grid path (build + query + brute force for the clouds it leaves)"""
    b, n = x.shape[:2]
    flags = [R.global_flag(x[i], radius, nsample) for i in range(b)]
    tags = {"gb_" + why for _, why in flags}
    if any(f is None for f, _ in flags):
        return tags
    use = R.batch_uses_grid([f for f, _ in flags])
    if any(f for f, _ in flags):
        tags.add("gq_batch_grid" if use else "bf_flagged_cloud_by_batch_rule")
    if use and not all(f for f, _ in flags):
        tags.add("bf_skips_grid_cloud")
    G = R.pick_group(b, q.shape[1], group)
    for i in range(b):
        hits = R.hit_rows(radius, x[i], q[i])
        if use and flags[i][0]:
            geo = R.geometry(x[i], radius)
            for j in range(q.shape[1]):
                tags |= {"gq_" + t for t in R.gq_query(x[i], geo, q[i, j], hits[j], nsample)}
        else:
            tags |= {"bf_" + t for t in R.bf_tags(n, q.shape[1], nsample, G, hits)}
    return tags


def _bf(x, q, nsample, group, radius):
    b, n = x.shape[:2]
    G = R.pick_group(b, q.shape[1], group)
    tags = set()
    for i in range(b):
        tags |= {"bf_" + t for t in R.bf_tags(n, q.shape[1], nsample, G, R.hit_rows(radius, x[i], q[i]))}
    return tags


def regimes(p):
    """the named regimes one case reaches"""
    b, n = p["b"], p["n"]
    x = p["xyz"]
    tags = set()
    if p["case"] == "bq_op":
        r, s, q = p["radius"], p["nsample"], p["q"]
        for i in range(b):
            tags |= _geo_tags(x[i], r)
        if O.oracle_ball_threshold(r) < 0:
            return tags | {"split_refused" if p["split"] else "bf_memset"}
        if p["split"]:
            return tags | {"split"} | _global_tags(x, q, r, s, p["group"])
        if p["mode"] == 0 and n >= R.GRID_MIN_N and R.bg_fits(n):
            if b * p["m"] >= 4096:
                tags.add("op_auto_ball_group")
                for i in range(b):
                    tags |= _bg_tags(x[i], q[i], r, s, n)
                return tags
            return tags | _bf(x, q, s, p["group"], r)
        if p["mode"] == 1 or n < R.GRID_MIN_N:
            return tags | _bf(x, q, s, p["group"], r)
        return tags | {"op_global_grid"} | _global_tags(x, q, r, s, p["group"])
    if p["case"] == "ball_group":
        r, s, q = p["radius"], p["nsample"], p["q"]
        if O.oracle_ball_threshold(r) < 0:
            return {"bg_refused"}
        _, by_m = R.bg_ctas_per_cloud(b, p["m"])
        tags.add("bg_ctas_by_m" if by_m else "bg_ctas_by_sms")
        if not p["center"]:
            tags.add("center_false")
        if not p["want_grouped"]:
            tags.add("no_grouped")
        for i in range(b):
            tags |= _geo_tags(x[i], r) | _bg_tags(x[i], q[i], r, s, n)
            if n >= R.BG_MIN_GRID_N and np.isnan(x[i]).all(0).any() and np.isfinite(q[i]).all(1).any():
                tags.add("bg_nan_axis_finite_query")  # every point is a hit: a grid walk would miss most of them
        return tags
    # bq_layer: the overlapped consumer's rows (centroids are data points)
    over = F.layer_overlapped(n, p["radii"])
    tags.add("layer_overlapped" if over else "layer_sequential")
    tags.add(f"layer_consumer_ctas_{p['consumer_ctas']}")
    if len(p["radii"]) > 1:
        tags.add("layer_msg")
    if over and 8192 <= n:
        tags.add("layer_overlapped_n8192")
    if not over and n > 8192:
        tags.add("layer_sequential_n" + ("9728" if n > 9727 else "8193_9727"))
    if any(O.oracle_ball_threshold(r) < 0 for r in p["radii"]):
        tags.add("layer_threshold_negative")
    ls = p["lengths"] or [n] * b
    if p["lengths"]:
        tags.add("layer_ragged")
    if not over:
        return tags
    for i, ln in enumerate(ls):
        c = x[i, :ln]
        nx = O.oracle_gather_point(c[None], O.oracle_fps(p["npoint"], c[None]))[0]
        if p["lengths"]:
            by_len = R.BgCloud(c, p["radii"][0], n).use_grid
            by_stride = R.BgCloud(x[i], p["radii"][0], n).use_grid
            if by_len != by_stride:
                tags.add("layer_length_flips_use_grid")
        for r, s in zip(p["radii"], p["ns"]):
            tags |= {"layer_" + t for t in _bg_tags(c, nx, r, s, n)}
    return tags


# Every regime of ball_regimes.py, per kernel
REQUIRED = {
    # grid_geometry
    "geo_nonfinite_box", "geo_degenerate_axis", "geo_nan_axis", "geo_dims_16",
    # bq_grid_build_kernel's flag and each reason it clears it; the batch rule
    "gb_grid", "gb_box", "gb_prune", "gb_expect", "gb_heavy", "gb_expect_local", "gq_batch_grid",
    "bf_flagged_cloud_by_batch_rule", "bf_skips_grid_cloud", "split", "split_refused", "op_global_grid",
    # bq_grid_query_kernel
    "gq_query_nonfinite", "gq_hit_overflow", "gq_rank_sort", "gq_empty_row", "gq_full_row",
    # ball_query_kernel<G>
    "bf_G1", "bf_G2", "bf_G4", "bf_G8", "bf_G16", "bf_G32", "bf_multi_tile", "bf_odd_n", "bf_early_exit", "bf_memset",
    # ball_group_kernel, per cloud
    "op_auto_ball_group", "bg_cloud_grid", "bg_cloud_box", "bg_cloud_small_n", "bg_cloud_prune", "bg_dual",
    "bg_single_layout", "bg_ctas_by_m", "bg_ctas_by_sms", "bg_refused", "center_false", "no_grouped",
    # ball_group_kernel, per query
    "bg_query_nonfinite", "bg_scan_instead", "bg_walk_balanced", "bg_walk_crowded", "bg_compact", "bg_compact_again",
    "bg_tau_reject", "bg_overflow_cost", "bg_overflow_nsample", "bg_sort1", "bg_sort2", "bg_sort4", "bg_sort8",
    "bg_scan_shared_buffered", "bg_scan_shared_unbuffered", "bg_scan_global_buffered", "bg_scan_global_unbuffered",
    "bg_empty_row", "bg_full_row", "bg_nan_axis_finite_query",
    # the layer
    "layer_overlapped", "layer_sequential", "layer_consumer_ctas_0", "layer_consumer_ctas_1", "layer_consumer_ctas_3",
    "layer_msg", "layer_ragged", "layer_length_flips_use_grid", "layer_overlapped_n8192", "layer_sequential_n8193_9727",
    "layer_sequential_n9728", "layer_threshold_negative", "layer_bg_cloud_grid", "layer_bg_scan_shared_unbuffered",
    "layer_bg_walk_balanced", "layer_bg_full_row",
}


@pytest.fixture(scope="module")
def slice_params():
    return [p for seed in F.SLICE_SEEDS for p in F.draws(seed, F.SLICE_ITERATIONS)]


@pytest.fixture(scope="module")
def slice_tags(slice_params):
    return [regimes(p) for p in slice_params]


def test_slice_reaches_every_regime(slice_tags):
    seen = set().union(*slice_tags)
    # the overlapped layer runs ball_group_kernel too: its query regimes count for the kernel
    seen |= {t[len("layer_"):] for t in seen if t.startswith("layer_bg_")}
    assert REQUIRED <= seen, sorted(REQUIRED - seen)


def test_slice_runs_every_case_the_same_number_of_times():
    assert F.SLICE_ITERATIONS % len(F.CASES) == 0 and F.SLICE_ITERATIONS // len(F.CASES) >= 10
    assert set(F.CASES) == set(F.DRAW) == set(F.RUN) == {"bq_op", "ball_group", "bq_layer"}


def test_draws_are_reproducible_and_bounded(slice_params):
    a, b = F.draws(F.SLICE_SEEDS[0], 6), F.draws(F.SLICE_SEEDS[0], 6)
    for p, q in zip(a, b):
        assert F.public(p) == F.public(q)
        for key in ("xyz", "q"):
            if key in p:
                assert np.array_equal(p[key].view(np.int32), q[key].view(np.int32))
    for p in slice_params:
        m = p.get("m", p.get("npoint"))
        assert m >= 1 and p["b"] * m * p["n"] <= F.MAX_POINTS
        assert p["xyz"].dtype == np.float32 and p["xyz"].shape == (p["b"], p["n"], 3)
        if "q" in p:
            assert p["q"].dtype == np.float32 and p["q"].shape == (p["b"], m, 3)


def test_slice_draws_the_edges(slice_params):
    """nsample on the hit-buffer edges, n on the kernels' edges, the radius on both sides of 1e-20 and at 1e30"""
    ss = {s for p in slice_params for s in p.get("ns", [p.get("nsample")])}
    assert {128, 129, 256, 257} <= ss and any(s > 256 for s in ss)
    ns = {p["n"] for p in slice_params}
    assert len(ns & set(F.N_EDGES)) >= 7, sorted(ns & set(F.N_EDGES))
    assert any(n % 2 for n in ns)
    rs = {r for p in slice_params for r in p.get("radii", [p.get("radius")])}
    assert any(O.oracle_ball_threshold(r) < 0 for r in rs) and any(r > 1e-20 and r < 1.1e-20 for r in rs)
    assert 1e30 in rs
