"""Without a GPU: the fixed-seed slice of tests/fuzz_knn_gpu.py reaches every regime of KnnWarp (knn_warp.cuh) in
both kNN kernels.  The draws are replayed with numpy and the C oracle only (oracle_fps gives the layer's centroids),
and every query row is tagged by tests/knn_regimes.py.  A draw that stops reaching a branch fails here, before a GPU
is needed."""
import numpy as np
import pytest

import fuzz_knn_gpu as F
import knn_regimes as R
from oracle import oracle as O


def row_tags(xyz, q, k, tile):
    """the union of knn_regimes.analyse over the query rows of one cloud, plus zero_distance_ties: two or more
    distances that round to 0 from points that are not the query"""
    tags = set()
    d = R.dist_rows(xyz, q)
    for j in range(len(q)):
        tags |= R.analyse(d[j], k, tile)[1]
        off = (xyz != q[j]).any(1)
        if k > 1 and np.count_nonzero((d[j] == 0) & off) >= 2:
            tags.add("zero_distance_ties")
    return tags


def regimes(p):
    """the named regimes one case reaches"""
    b, n, k = p["b"], p["n"], p["k"]
    tags = set()
    if p["case"] == "knn_op":
        for i in range(b):
            tags |= row_tags(p["xyz"][i], p["q"][i], k, R.TILE)
        if n > 2 * R.TILE:
            tags.add("three_tiles")
        if R.group_tail_lt_32(n, k):
            tags.add("group_tail_lt_32")
        if p["m"] % 8:
            tags.add("m_mod_8")
        return tags
    can = F.overlapped_can_run(b, n, k)
    if p["path"] == 1 and can:
        tags |= {"path_forced_overlapped", "layer_kc1" if k <= 32 else "layer_kc2"}
        if p["consumer_ctas"] == 1:
            tags.add("consumer_ctas_1")
    if p["path"] == 2:
        tags.add("path_forced_sequential")
    if not p["center"]:
        tags.add("center_false")
    if not p["want_grouped"]:
        tags.add("no_grouped")
    if not p["want_dist"]:
        tags.add("no_dist")
    if p["path"] == 1 and can:  # the rows of knn_group_kernel: one offer of the whole cloud
        nx = O.oracle_gather_point(p["xyz"], O.oracle_fps(p["npoint"], p["xyz"]))
        for i in range(b):
            tags |= {"overlapped_" + t for t in row_tags(p["xyz"][i], nx[i], k, n)}
    return tags


REQUIRED = {
    "kc1", "kc2", "kc4", "kc2_partial_b_nonempty", "kc4_partial_b_nonempty", "layer_kc1", "layer_kc2", "k_eq_n",
    "b_never_full", "evict_tie", "reject_eq_tau", "fast_path", "tie_boundary_only", "tie_in_prefix", "inf_in_prefix",
    "nan_in_A", "nan_beyond_k", "nan_query", "zero_distance_ties", "three_tiles", "group_tail_lt_32", "m_mod_8",
    "path_forced_overlapped", "path_forced_sequential", "consumer_ctas_1", "center_false", "no_grouped", "no_dist",
    # knn_group_kernel's own scan (one offer of the whole cloud, trips that run on across 1024 points)
    "overlapped_evict_tie", "overlapped_reject_eq_tau", "overlapped_tie_in_prefix", "overlapped_nan_in_A",
    "overlapped_kc2_partial_b_nonempty", "overlapped_fast_path",
}


@pytest.fixture(scope="module")
def slice_params():
    return [p for seed in F.SLICE_SEEDS for p in F.draws(seed, F.SLICE_ITERATIONS)]


@pytest.fixture(scope="module")
def slice_tags(slice_params):
    return [regimes(p) for p in slice_params]


def test_slice_reaches_every_regime(slice_tags):
    seen = set().union(*slice_tags)
    assert REQUIRED <= seen, sorted(REQUIRED - seen)


def test_slice_runs_both_cases_the_same_number_of_times():
    assert F.SLICE_ITERATIONS % len(F.CASES) == 0 and F.SLICE_ITERATIONS // len(F.CASES) >= 10
    assert set(F.CASES) == set(F.DRAW) == set(F.RUN) == {"knn_op", "knn_layer"}


def test_draws_are_reproducible_and_bounded(slice_params):
    a, b = F.draws(F.SLICE_SEEDS[0], 10), F.draws(F.SLICE_SEEDS[0], 10)
    for p, q in zip(a, b):
        assert F.public(p) == F.public(q)
        for key in ("xyz", "q"):
            if key in p:
                assert np.array_equal(p[key].view(np.int32), q[key].view(np.int32))
    for p in slice_params:
        m = p.get("m", p.get("npoint"))
        assert 1 <= p["k"] <= min(p["n"], 128) and m >= 1
        assert p["b"] * m * p["n"] <= F.MAX_POINTS and p["b"] * m * p["k"] * p["n"] <= F.MAX_ROW_ROUNDS
        assert p["xyz"].dtype == np.float32 and p["xyz"].shape == (p["b"], p["n"], 3)
        if p["case"] == "knn_layer":
            assert p["n"] <= 8192 and (p["path"] != 1 or p["k"] <= 64)
        else:
            assert p["q"].dtype == np.float32 and p["q"].shape == (p["b"], m, 3)


def test_slice_draws_the_edges(slice_params):
    """k on every boundary of the KC instances, n on the tile and group edges"""
    ks = {p["k"] for p in slice_params}
    assert {1, 32, 33, 64, 65, 128} <= ks
    ns = {(p["n"], p["k"]) for p in slice_params}
    assert any(n == 2 * k for n, k in ns) and any(n == k + 1 for n, k in ns)
    assert {1024, 1025} & {n for n, _ in ns}


def test_kg_warps_restates_the_layer():
    """overlapped_can_run is what tests/test_knn_layer_gpu.py pins on the device for pn2_sa_knn_layer_fits"""
    assert F.kg_warps(20000, 8) == 0 and F.kg_warps(4096, 64) > 0 and F.kg_warps(4096, 128) == 0
    assert F.kg_warps(8192, 64) == 32 and F.kg_warps(16, 17) == 0
