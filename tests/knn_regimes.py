"""KnnWarp (pointnet2_b200/csrc/knn_warp.cuh) restated in numpy, for one row of squared distances: which elements
form the sets A and B, in what order B takes them and what each insertion hits, whether ``finish`` takes the sorted
fast path or the replay and why, and the replay itself on W = A ∪ B.  No device is needed.

The kernels' claim (knn.cu) is that the first k columns of the reference's selection sort over the whole row can be
computed from W alone.  ``replay`` and ``sorted_prefix`` compute them that way; tests/test_knn_regimes_cpu.py holds
both to ``oracle.oracle_selection_sort`` on the whole row, and tests/test_fuzz_knn_cpu.py uses ``analyse`` to show
that the fixed GPU slice of tests/fuzz_knn_gpu.py reaches every branch.

Values are compared as floats.  The kernel orders B and W by the bits of the value, which is the same order for the
non-negative distances it sees (a distance is never −0.0 or negative).
"""
from __future__ import annotations

import numpy as np

TILE = 1024  # knn_kernel's shared-memory tile (knn.cu kKnnTile); the overlapped layer offers the whole cloud at once


def dist_row(xyz, q):
    """float32 squared distances of the points xyz (n, 3) from q (3,), as oracle.oracle_knn_point computes them:
    ((dx² + dy²) + dz²), every difference, product and sum rounded to float32."""
    return dist_rows(xyz, np.asarray(q, np.float32)[None])[0]


def dist_rows(xyz, q):
    """dist_row for every query of q (m, 3): (m, n)"""
    with np.errstate(over="ignore", invalid="ignore"):  # inf and NaN distances are part of the contract
        d = (np.asarray(xyz, np.float32)[None, :, :] - np.asarray(q, np.float32)[:, None, :]).astype(np.float32)
        sq = (d * d).astype(np.float32)
        return ((sq[..., 0] + sq[..., 1]).astype(np.float32) + sq[..., 2]).astype(np.float32)


def _trip(p, k, tile):
    """the 64-position trip of ``offer`` that position p (>= k) is scanned in, as one sortable integer: tiles of
    ``tile`` points, each scanned in trips of 64 from max(0, k - base)"""
    base = (p // tile) * tile
    return (p // tile) * (tile + 64) + (p - base - np.maximum(0, k - base)) // 64


def build_b(v, k, tile=TILE):
    """Set B as ``offer`` builds it.  Positions >= k are scanned in trips of two 32-point groups; one ballot per
    group, taken with the state at the start of the trip, picks the candidates (every non-NaN value while B is open,
    values < tau once it is full), and each candidate, in ascending position, is appended while B is open or else
    replaces B's maximum under (value, position) if it is still < tau.

    Returns (positions of B in slot order, events) with events: ``full`` (B filled), ``evictions``, ``evict_tie``
    (evictions made while B's maximum value was held by several entries), ``reject_eq_tau`` (candidates that passed
    the ballot and were then equal to tau)."""
    v = np.asarray(v, np.float32)
    n = len(v)
    ev = dict(full=False, evictions=0, evict_tie=0, reject_eq_tau=0)
    pos = np.arange(k, n)
    pos = pos[~np.isnan(v[k:])] if n > k else pos
    if len(pos) < k:  # B never fills: every non-NaN position >= k, in scan order
        return [int(p) for p in pos], ev
    ev["full"] = True
    bp = [int(p) for p in pos[:k]]
    bv = [float(v[p]) for p in bp]

    def find_max():
        tau = max(bv)
        return tau, max(p for p, x in zip(bp, bv) if x == tau)

    def offer_one(p, tau, ev_pos):
        x = float(v[p])
        if x < tau:
            ev["evictions"] += 1
            if sum(1 for y in bv if y == tau) > 1:
                ev["evict_tie"] += 1
            j = bp.index(ev_pos)
            bp[j], bv[j] = int(p), x
            return find_max()
        if x == tau:
            ev["reject_eq_tau"] += 1
        return tau, ev_pos

    tau, ev_pos = find_max()
    rest = pos[k:]
    if len(rest) == 0:
        return bp, ev
    trips = _trip(rest, k, tile)
    # the trip in which B filled was balloted while B was open: all its later non-NaN positions are candidates
    same = trips == _trip(np.array([pos[k - 1]]), k, tile)[0]
    for p in rest[same]:
        tau, ev_pos = offer_one(p, tau, ev_pos)
    rest, trips = rest[~same], trips[~same]
    keep = v[rest] < tau
    rest, trips = rest[keep], trips[keep]
    while len(rest):  # each later trip: the candidates are the values below tau at its start
        t = trips[0]
        cnt = int(np.searchsorted(trips, t, side="right"))
        for p in rest[:cnt]:
            tau, ev_pos = offer_one(p, tau, ev_pos)
        rest, trips = rest[cnt:], trips[cnt:]
        keep = v[rest] < tau
        rest, trips = rest[keep], trips[keep]
    return bp, ev


def expected_b(v, k):
    """the k smallest non-NaN values at positions >= k under (value, position), as a set of positions"""
    v = np.asarray(v, np.float32)
    pos = np.arange(k, len(v))
    pos = pos[~np.isnan(v[k:])] if len(v) > k else pos
    order = np.lexsort((pos, v[pos]))
    return set(int(p) for p in pos[order[:k]])


def fast_path(v, k, w):
    """``finish``'s decision on W (original positions ``w``): (taken, reasons, sorted W).  The fast path needs |A| = k,
    the k smallest of W finite and pairwise different, the k-th and (k+1)-th different, and no NaN in W.  Reasons:
    ``nan_in_A``, ``inf_in_prefix``, ``tie_in_prefix`` (two equal values among the k smallest),
    ``tie_boundary_only`` (the only tie is between ranks k-1 and k)."""
    v = np.asarray(v, np.float32)
    w = np.asarray(w, np.int64)
    vals = v[w]
    order = np.lexsort((w, vals, np.isnan(vals)))  # NaN last, as its bits sort
    sw, sv = w[order], vals[order]
    reasons = set()
    if np.isnan(vals).any():
        reasons.add("nan_in_A")  # NaN never enters B
    head = sv[:k]
    if np.isinf(head).any():
        reasons.add("inf_in_prefix")
    if k > 1 and (head[1:] == head[:-1]).any():
        reasons.add("tie_in_prefix")
    if len(sv) > k and sv[k - 1] == sv[k]:
        reasons.add("tie_boundary" if reasons else "tie_boundary_only")
    ka = min(k, len(v))
    return ka == k and not reasons, reasons, (sv, sw)


def replay(v, k, w):
    """The k selection-sort rounds on W alone, with current positions (``finish``'s replay): a NaN at position s wins
    round s, a NaN elsewhere is never taken, otherwise the smallest value wins and ties go to the lowest current
    position; the winner swaps with the element at s.  Returns (values float32 (ka,), indices int32 (ka,))."""
    v = np.asarray(v, np.float32)
    w = np.asarray(w, np.int64)
    vals = v[w]
    nan = np.isnan(vals)
    cur = w.copy()  # current positions: nothing has moved yet
    ka = min(k, len(v))
    out_v = np.empty(ka, np.float32)
    out_i = np.empty(ka, np.int32)
    for s in range(ka):
        at_s = int(np.flatnonzero(cur == s)[0])
        if nan[at_s]:
            win = at_s
        else:
            cand = np.flatnonzero((cur >= s) & ~nan)
            best = vals[cand].min()
            ties = cand[vals[cand] == best]
            win = int(ties[np.argmin(cur[ties])])
        cur[at_s], cur[win] = cur[win], s
        out_v[s], out_i[s] = vals[win], w[win]
    return out_v, out_i


def sorted_prefix(v, k, w):
    """the fast path's answer: the k smallest of W under (value, position)"""
    _, _, (sv, sw) = fast_path(v, k, w)
    return sv[:k].astype(np.float32), sw[:k].astype(np.int32)


def analyse(v, k, tile=TILE):
    """Everything KnnWarp does with one row v (float32 (n,)) and k <= n, as (W positions, tags).  Tags name the
    regimes the row reaches: ``kc1`` / ``kc2`` / ``kc4`` (the instance, k <= 32 * KC), ``kcN_partial_b_nonempty``
    (k not a multiple of 32 and B filled: the lane masks of the partial last register run), ``k_eq_n``,
    ``b_never_full``, ``evict_tie``, ``reject_eq_tau``, ``fast_path`` or the reasons it is not taken,
    ``nan_beyond_k`` and ``nan_query`` (every distance NaN)."""
    v = np.asarray(v, np.float32)
    n = len(v)
    kc = 1 if k <= 32 else 2 if k <= 64 else 4
    tags = {f"kc{kc}"}
    bp, ev = build_b(v, k, tile)
    if ev["full"] and k % 32:
        tags.add(f"kc{kc}_partial_b_nonempty")
    if k == n:
        tags.add("k_eq_n")
    elif not ev["full"]:
        tags.add("b_never_full")
    if ev["evict_tie"]:
        tags.add("evict_tie")
    if ev["reject_eq_tau"]:
        tags.add("reject_eq_tau")
    w = list(range(min(k, n))) + bp
    taken, reasons, _ = fast_path(v, k, w)
    tags |= {"fast_path"} if taken else reasons
    nan = np.isnan(v)
    if nan[k:].any():
        tags.add("nan_beyond_k")
    if nan.all():
        tags.add("nan_query")
    return w, tags


def group_tail_lt_32(n, k, tile=TILE):
    """the cloud ends inside the first 32-point group of a trip of its last tile: the second group is empty and the
    first partial"""
    base = (n - 1) // tile * tile
    p0 = max(0, k - base)
    tn = n - base
    return p0 < tn and 0 < (tn - p0) % 64 < 32
