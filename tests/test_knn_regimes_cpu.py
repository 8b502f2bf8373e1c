"""Without a GPU: the derivation both kNN kernels rest on (knn.cu, knn_warp.cuh), restated by tests/knn_regimes.py,
against the reference's selection sort (oracle.oracle_selection_sort) over the whole row, on thousands of
adversarial rows.

- ``offer``'s insertion order ends with B = the k smallest non-NaN values at positions >= k under (value, position),
  with the knn_kernel tiles and with the whole cloud in one offer;
- the k selection-sort rounds replayed on W = A ∪ B alone give the first k columns of the full sort, values and
  indices;
- whenever ``finish``'s fast-path condition holds, the sorted W gives them too.
"""
import numpy as np
import pytest

import knn_regimes as R
from oracle import oracle as O


def full_sort(v, k):
    i, x = O.oracle_selection_sort(k, np.asarray(v, np.float32)[None, None, :])
    return x[0, 0, :k], i[0, 0, :k]


def row(rs, n, k):
    """one adversarial row of n 'distances': few distinct levels, all equal, integer levels or continuous values,
    with NaN at a position < k, at k or last, and ±inf"""
    kind = rs.randint(6)
    if kind == 0:
        v = np.full(n, np.float32(rs.choice([0.0, 1.0, 2.5])))
    elif kind == 1:
        v = rs.randint(0, int(rs.choice([2, 3, 5])), n).astype(np.float32)
    elif kind == 2:
        v = rs.randint(0, int(rs.choice([8, 30, 1000])), n).astype(np.float32)
    elif kind == 3:
        v = rs.random_sample(n).astype(np.float32)
    elif kind == 4:  # the k-th and (k+1)-th smallest of W planted equal: a distinct row otherwise
        v = rs.permutation(n).astype(np.float32)
        j = int(rs.randint(n))
        v[j] = v[(j + 1) % n] if n > 1 else v[j]
    else:  # an ascending run at the front: A (partly) sorted already, few swaps
        v = rs.randint(0, 50, n).astype(np.float32)
        j = int(rs.randint(1, n + 1))
        v[:j] = np.sort(v[:j])
    for _ in range(int(rs.choice([0, 0, 1, 2]))):
        where = rs.randint(4)
        p = [int(rs.randint(k)), k, n - 1, int(rs.randint(n))][where]
        if p < n:
            v[p] = np.float32(rs.choice([np.nan, np.inf, np.inf, -np.inf]))
    return v


def n_for(rs, k):
    return int(rs.choice([k, k + 1, 2 * k - 1, 2 * k, k + int(rs.randint(1, 64)), int(rs.randint(k, 3 * k + 70))]))


def check_row(v, k):
    """every claim on one row; returns the row's tags"""
    want_v, want_i = full_sort(v, k)
    expect_b = R.expected_b(v, k)
    for tile in (R.TILE, len(v)):
        bp, _ = R.build_b(v, k, tile)
        assert set(bp) == expect_b and len(bp) == len(expect_b), (k, tile, v)
    w, tags = R.analyse(v, k)
    got_v, got_i = R.replay(v, k, w)
    assert np.array_equal(got_i, want_i) and np.array_equal(got_v.view(np.int32), want_v.view(np.int32)), (k, v)
    if "fast_path" in tags:
        sv, si = R.sorted_prefix(v, k, w)
        assert np.array_equal(si, want_i) and np.array_equal(sv.view(np.int32), want_v.view(np.int32)), (k, v)
    return tags


def test_replay_on_w_equals_the_full_selection_sort_for_every_k():
    rs = np.random.RandomState(2024)
    seen = set()
    rows = 0
    for k in range(1, 129):
        for _ in range(24):
            n = max(1, n_for(rs, k))
            k_ = min(k, n)
            seen |= check_row(row(rs, n, k_), k_)
            rows += 1
    assert rows >= 3000
    want = {"kc1", "kc2", "kc4", "kc2_partial_b_nonempty", "kc4_partial_b_nonempty", "k_eq_n", "b_never_full",
            "evict_tie", "reject_eq_tau", "fast_path", "tie_boundary_only", "tie_in_prefix", "inf_in_prefix",
            "nan_in_A", "nan_beyond_k"}
    assert want <= seen, sorted(want - seen)


@pytest.mark.parametrize("n", [300, 1100, 2100])
def test_long_rows_across_tiles(n):
    """rows longer than one and two knn_kernel tiles, with few levels: B evicts across tile boundaries"""
    rs = np.random.RandomState(n)
    for k in (1, 31, 33, 64, 65, 100, 128):
        for levels in (2, 40, 100000):
            v = rs.randint(0, levels, n).astype(np.float32)
            if rs.rand() < 0.5:
                v[rs.randint(n, size=3)] = np.nan
            check_row(v, k)


def test_all_nan_row():
    """a NaN query: every distance is NaN, each one is output in its own round, in position order"""
    for k, n in ((1, 1), (5, 40), (33, 33), (128, 300)):
        v = np.full(n, np.nan, np.float32)
        tags = check_row(v, k)
        assert {"nan_query", "nan_in_A"} <= tags
        _, i = full_sort(v, k)
        np.testing.assert_array_equal(i, np.arange(k))


def test_nan_positions():
    """NaN before k is output in its own column; at k or beyond it is never taken"""
    v = np.array([5, np.nan, 1, 7, np.nan, 0, 3, np.nan], np.float32)
    for k in range(1, 9):
        check_row(v, k)
    _, i = full_sort(v, 3)
    np.testing.assert_array_equal(i, [5, 1, 2])


def test_a_boundary_tie_needs_the_replay():
    """W = {9, 9 | 1}, k = 2: sorted W gives positions [2, 0], the selection sort [2, 1] (round 0 swaps the 9 from
    position 0 to position 2, so the 9 at position 1 wins round 1 by position).  A tie between ranks k-1 and k alone
    must leave the fast path."""
    v = np.array([9, 9, 1], np.float32)
    w, tags = R.analyse(v, 2)
    assert "tie_boundary_only" in tags and "fast_path" not in tags
    _, want_i = full_sort(v, 2)
    np.testing.assert_array_equal(want_i, [2, 1])
    np.testing.assert_array_equal(R.replay(v, 2, w)[1], [2, 1])
    np.testing.assert_array_equal(R.sorted_prefix(v, 2, w)[1], [2, 0])


def test_boundary_ties_often_change_the_answer():
    """not a single construction: random rows with a boundary-only tie have wrong sorted prefixes too"""
    rs = np.random.RandomState(5)
    wrong = total = 0
    for _ in range(3000):
        k = int(rs.randint(1, 40))
        n = int(rs.randint(k + 1, 3 * k + 10))
        v = rs.randint(0, 12, n).astype(np.float32)
        w, tags = R.analyse(v, k)
        if tags & {"tie_boundary_only"}:
            total += 1
            _, want_i = full_sort(v, k)
            wrong += not np.array_equal(R.sorted_prefix(v, k, w)[1], want_i)
    assert total > 20 and wrong > 0, (wrong, total)


def test_b_insertion_events_by_hand():
    """k = 2, all in the trip that fills B, so every position is a candidate: B fills with positions 2, 3 (4, 4);
    position 4 (1) evicts the LATER of the two equal maxima, 3, while the maximum is shared; position 5 (4) equals
    tau = 4 and is rejected; position 6 (3) evicts 2; position 7 (3) equals tau = 3 and is rejected."""
    v = np.array([0, 0, 4, 4, 1, 4, 3, 3], np.float32)
    for tile in (R.TILE, len(v)):
        bp, ev = R.build_b(v, 2, tile)
        assert sorted(bp) == [4, 6] and set(bp) == R.expected_b(v, 2)
        assert ev == dict(full=True, evictions=2, evict_tie=1, reject_eq_tau=2)


def test_later_trips_are_balloted_against_tau():
    """once B is full, a trip's candidates are the values below tau at its start: an equal value in a later trip
    never reaches the comparison (no reject_eq_tau), one below it does"""
    k = 2
    v = np.full(200, 50, np.float32)
    v[:4] = [0, 0, 7, 7]  # B = {2, 3}, tau = 7, filled in the first trip (positions 2..65)
    v[100] = 7            # a later trip: not a candidate
    bp, ev = R.build_b(v, k)
    assert sorted(bp) == [2, 3] and ev["reject_eq_tau"] == 0 and ev["evictions"] == 0
    v[150] = 3
    bp, ev = R.build_b(v, k)
    assert sorted(bp) == [2, 150] and ev["evict_tie"] == 1
