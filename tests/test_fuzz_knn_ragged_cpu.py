"""Without a GPU: the fixed-seed slice of tests/fuzz_knn_ragged_gpu.py reaches every regime of per-cloud lengths in
both kNN kernels — clouds shorter than k, as long as k, and longer with a partial last tile; every KC instance; both
layer paths; query padding and self-kNN; out-of-range device lengths; and, on rows of truncated clouds, both KnnWarp
finishes (the sorted fast path and the replay).  The draws are replayed with numpy and the C oracle only (oracle_fps
gives the layer's centroids), and the query rows of the truncated clouds are tagged by tests/knn_regimes.py."""
import numpy as np

import fuzz_knn_gpu as F
import fuzz_knn_ragged_gpu as G
import knn_regimes as R
from oracle import oracle as O

ROWS = 48  # query rows analysed per cloud


def kc(k):
    return 1 if k <= 32 else 2 if k <= 64 else 4


def cloud_tags(x, q, ln, n, k, tile):
    tags = set()
    kq = min(k, ln)
    tags.add("len_lt_k" if ln < k else "len_eq_k" if ln == k else "len_gt_k")
    if ln > k and ln % tile and ln < n:
        tags.add("len_gt_k_partial_tile")
    if ln < n:
        d = R.dist_rows(x[:ln], q[:ROWS])
        for j in range(len(d)):
            taken = "fast_path" in R.analyse(d[j], kq, tile)[1]
            tags.add("ragged_fast_path" if taken else "ragged_replay")
    return tags


def regimes(p):
    b, n, k = p["b"], p["n"], p["k"]
    tags = set()
    if p["raw_lengths"] != p["lengths"]:
        tags.add("clamped")
    if p["case"] == "knn_ragged":
        tags.add(f"op_kc{kc(k)}")
        lens = p["lengths"] if p["data_lengths"] else [n] * b
        qlens = p["query_lengths"] or [p["m"]] * b
        if any(ql < p["m"] for ql in qlens):
            tags.add("query_padding")
        if p["self_knn"]:
            tags.add("self_knn")
        for i in range(b):
            tags |= cloud_tags(p["xyz"][i], p["q"][i][:qlens[i]], lens[i], n, k, R.TILE)
        return tags
    tags.add(f"layer_kc{kc(k)}")
    if p["path"] == 2 or (p["path"] == 1 and not F.overlapped_can_run(b, n, k)):
        tags.add("sequential")
    elif p["path"] == 1:
        tags.add("overlapped")
    for i, ln in enumerate(p["lengths"]):
        c = p["xyz"][i:i + 1, :ln]
        q = O.oracle_gather_point(c, O.oracle_fps(p["npoint"], c))[0]
        tile = R.TILE if "sequential" in tags else max(n, 1)  # the overlapped layer offers the whole cloud at once
        tags |= {"layer_" + t for t in cloud_tags(p["xyz"][i], q, ln, n, k, tile)}
    return tags


REQUIRED = {"len_lt_k", "len_eq_k", "len_gt_k", "len_gt_k_partial_tile", "op_kc1", "op_kc2", "op_kc4", "query_padding",
            "self_knn", "ragged_fast_path", "ragged_replay", "clamped", "layer_kc1", "layer_kc2", "layer_kc4", "overlapped",
            "sequential", "layer_len_lt_k", "layer_len_eq_k", "layer_len_gt_k_partial_tile", "layer_ragged_fast_path",
            "layer_ragged_replay"}


def test_fixed_slice_reaches_every_regime():
    tags = set()
    for seed in G.SLICE_SEEDS:
        for p in G.draws(seed, G.SLICE_ITERATIONS):
            tags |= regimes(p)
    missing = REQUIRED - tags
    assert not missing, f"the fixed slice no longer reaches {sorted(missing)}"


def test_draws_are_reproducible_and_well_formed():
    a, b = G.draws(81, 6), G.draws(81, 6)
    for p, q in zip(a, b):
        assert F.public(p) == F.public(q)
        assert np.array_equal(p["xyz"], q["xyz"], equal_nan=True)
        assert all(1 <= ln <= p["n"] for ln in p["lengths"]) and 1 <= p["k"] <= min(p["n"], 128)
