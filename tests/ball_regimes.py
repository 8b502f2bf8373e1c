"""The path decisions of the three ball-query kernels restated in numpy, per cloud and per query.  No device is needed.

- ``geometry`` / ``cells``: grid_geometry and grid_cell (csrc/pn2_common.cuh), in float32 and in the kernels' operation
  order (the build uses -fmad=false and no fast math: IEEE division, no contraction).
- ``global_flag``: bq_grid_build_kernel's per-cloud flag (csrc/ball_query_grid.cu) and the reason it is cleared;
  ``batch_uses_grid``: the ¼ rule both global-grid kernels apply to the batch.
- ``BgCloud`` / ``bg_query``: ball_group_kernel (csrc/sa_fused.cu), the shared-memory grid: whether a cloud is binned,
  whether it keeps both layouts, and per query the 9 candidate ranges, the walk, the hit buffer's compactions, the
  overflow, the sort and the ordered scan.
- ``gq_query``: bq_grid_query_kernel: non-finite query, hit-buffer overflow, rank sort.
- ``pick_group`` / ``bf_tags``: the brute-force ball_query_kernel<G> (csrc/ball_query.cu).

Inside a cell the order of the points comes from an atomicAdd scatter and differs from run to run, so the walk's
counters at the first compaction are not fixed.  ``bg_query`` walks the neighbourhood twice, with the hits first in
every cell and with the hits last, and reports a decision only when both walks agree; it also checks that both walks
emit the oracle's row.  The hits themselves (``hit_rows``) come from the C oracle.
"""
from __future__ import annotations

import numpy as np

from oracle import oracle as O

f32 = np.float32
MAX_DIM = 16          # kGridMaxDim
BG_HIT_CAP = 256      # kBgHitCap
BG_COMPACT_MAX = 128  # kBgCompactMax
BG_MIN_GRID_N = 512   # kBgMinGridN
GQ_HIT_CAP = 128      # kHitCap
GRID_MIN_N = 2048     # kGridMinN
BQ_TILE = 2048        # kBqTile
SMS = 132             # the H100's SM count (pick_group, ball_group's CTAs per cloud)


def _fdiv(a, b):
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        return f32(f32(a) / f32(b))


def _fmul(a, b):
    with np.errstate(invalid="ignore", over="ignore"):
        return f32(f32(a) * f32(b))


def _to_int(x):
    """(int) of a float as the device converts it: NaN -> 0, saturating"""
    x = float(x)
    if x != x:
        return 0
    return int(max(min(x, 2.0 ** 31 - 1), -(2.0 ** 31)))


def geometry(pts, radius):
    """grid_geometry over the points pts (n, 3): a dict with mn, ext, emax, h, inv_h, finite_box, dims, ncell, nb"""
    pts = np.asarray(pts, f32)
    radius = f32(radius)
    nan = np.isnan(pts)
    with np.errstate(invalid="ignore", over="ignore"):
        mn = np.where(nan, f32(np.inf), pts).min(0).astype(f32)  # fminf skips NaN
        mx = np.where(nan, f32(np.inf), pts).max(0).astype(f32)  # a NaN coordinate makes the max +inf
        ext = (mx - mn).astype(f32)
    emax = f32(np.fmax(np.fmax(ext[0], ext[1]), ext[2]))
    h = f32(np.fmax(_fmul(f32(1.01), radius), _fdiv(emax, f32(MAX_DIM - 1))))
    finite_box = bool(not np.isnan(ext).any() and emax >= 0 and emax < f32(1e30) and h > 0 and h < f32(1e30))
    if not finite_box:
        h = f32(1.0)
    inv_h = _fdiv(f32(1.0), h)
    dims = []
    for c in range(3):
        d = _to_int(np.floor(_fmul(ext[c], inv_h))) + 1 if finite_box else 1
        dims.append(min(max(d, 1), MAX_DIM))
    nb = min(dims[0], 3) * min(dims[1], 3) * min(dims[2], 3)
    return dict(mn=mn, ext=ext, emax=emax, h=h, inv_h=inv_h, finite_box=finite_box, dims=dims,
                ncell=dims[0] * dims[1] * dims[2], nb=nb)


def cells(x, geo, query=False):
    """grid_cell of the coordinates x (..., 3): clamped to [-1, dim] (queries) or to [0, dim - 1] (points)"""
    x = np.asarray(x, f32)
    with np.errstate(invalid="ignore", over="ignore"):
        f = np.floor(((x - geo["mn"]).astype(f32) * geo["inv_h"]).astype(f32))
    dims = np.array(geo["dims"], f32)
    f = np.fmin(np.fmax(f, f32(-1)), dims)  # fmaxf(NaN, -1) = -1
    c = f.astype(np.int64)
    return c if query else np.minimum(np.maximum(c, 0), np.array(geo["dims"]) - 1)


def hit_rows(radius, pts, q):
    """(m, n) boolean: point k passes query j's test, from the C oracle (every hit, not just the first nsample)"""
    pts, q = np.asarray(pts, f32), np.asarray(q, f32)
    n, m = len(pts), len(q)
    out = np.zeros((m, n), bool)
    for a in range(0, m, 512):
        qq = q[a:a + 512]
        idx, cnt = O.oracle_query_ball_point(float(radius), n, pts[None], qq[None])
        for j in range(len(qq)):
            out[a + j, idx[0, j, :cnt[0, j]]] = True
    return out


# ----------------------------------------------------------------------------------------------- global grid
def global_flag(pts, radius, nsample):
    """bq_grid_build_kernel on one cloud: (flag, reason).  flag is None where float sums leave it undecided (the sum of
    c_i² beyond 2^24 with the margin to 0.9 nsample not clear)."""
    pts = np.asarray(pts, f32)
    n = len(pts)
    geo = geometry(pts, radius)
    r = f32(radius)
    vol = _fmul(_fmul(np.fmax(geo["ext"][0], geo["h"]), np.fmax(geo["ext"][1], geo["h"])), np.fmax(geo["ext"][2], geo["h"]))
    expect = _fdiv(_fmul(_fmul(_fmul(_fmul(f32(n), f32(4.18879)), r), r), r), vol)
    if not geo["finite_box"]:
        return False, "box"
    if n < GRID_MIN_N:
        return False, "small_n"
    if 10 * geo["nb"] > 3 * geo["ncell"]:
        return False, "prune"
    if not expect < _fmul(f32(0.75), f32(nsample)):
        return False, "expect"
    cnt = cell_counts(pts, geo)
    if cnt.max() > 256:
        return False, "heavy"
    sq = int((cnt.astype(np.int64) ** 2).sum())
    rh = _fmul(r, geo["inv_h"])
    lim = _fmul(f32(0.9), f32(nsample))
    el = _fdiv(_fmul(_fmul(_fmul(_fmul(f32(4.18879), rh), rh), rh), f32(sq)), f32(n))
    if sq >= 1 << 24 and abs(float(el) - float(lim)) <= 1e-3 * float(lim):
        return None, "expect_local_undecided"
    if not el < lim:
        return False, "expect_local"
    return True, "grid"


def cell_counts(pts, geo):
    c = cells(pts, geo)
    d = geo["dims"]
    return np.bincount((c[:, 2] * d[1] + c[:, 1]) * d[0] + c[:, 0], minlength=geo["ncell"])


def batch_uses_grid(flags):
    bb = min(len(flags), 1024)
    return 4 * sum(1 for f in flags[:bb] if f) >= bb


# ------------------------------------------------------------------------------------------- ball_group_kernel
def bg_dual_layout(stride):
    """both layouts fit in shared memory: 32 n + 49168 <= 200 KiB, i.e. n <= 4863 (the row stride, not the length)"""
    return 16 * stride + (4096 + 4) * 4 + 32 * 256 * 4 + 16 * stride <= 200 * 1024


def bg_fits(n):
    """pn2_ball_group_fits: n <= 9727"""
    return 0 < n < (1 << 14) and 16 * n + (4096 + 4) * 4 + 32 * 256 * 4 <= 200 * 1024


def bg_ctas_per_cloud(b, m):
    """ball_group's CTAs per cloud when all queries are known: SMs per cloud, at most one warp per query"""
    r = SMS // min(b, SMS)
    return max(1, min(r, (m + 31) // 32)), r > (m + 31) // 32


class BgCloud:
    """ball_group_kernel's state for one cloud of ``length`` points in a batch of row stride ``stride``"""

    def __init__(self, pts, radius, stride):
        self.pts = np.asarray(pts, f32)
        self.n = len(self.pts)
        self.geo = geometry(self.pts, radius)
        g = self.geo
        self.use_grid = g["finite_box"] and self.n >= BG_MIN_GRID_N and 10 * g["nb"] <= 3 * g["ncell"]
        self.dual = bg_dual_layout(stride)
        self.reason = ("grid" if self.use_grid else "box" if not g["finite_box"] else "small_n" if self.n < BG_MIN_GRID_N
                       else "prune")
        if self.use_grid:
            c = cells(self.pts, g)
            d = g["dims"]
            self.cell = (c[:, 2] * d[1] + c[:, 1]) * d[0] + c[:, 0]
            cnt = np.bincount(self.cell, minlength=g["ncell"])
            self.start = np.concatenate([[0], np.cumsum(cnt)])

    def ranges(self, q):
        """the 9 candidate ranges of query q: a list of lists of cell ids (each a row of up to 3 x-adjacent cells)"""
        g = self.geo
        dx, dy, dz = g["dims"]
        cx, cy, cz = (int(v) for v in cells(np.asarray(q, f32)[None], g, query=True)[0])
        x0, x1 = max(cx - 1, 0), min(cx + 1, dx - 1)
        out = []
        for rr in range(9):
            y, z = cy + rr % 3 - 1, cz + rr // 3 - 1
            if x0 <= x1 and 0 <= y < dy and 0 <= z < dz:
                base = (z * dy + y) * dx
                out.append(list(range(base + x0, base + x1 + 1)))
            else:
                out.append([])
        return out


def _qfinite(q):
    return bool(np.all(np.abs(np.asarray(q, np.float64)) <= float(f32(3.0e38))))


def _walk(cl, lists, crowded, hits, total, nsample):
    """one walk of the neighbourhood with the candidate order ``lists`` (9 lists of point indices): the events, the
    final buffer and whether it overflowed"""
    n = cl.n
    ev = set()
    buf, hcount, tau, tested, dense = [], 0, None, 0, False
    if crowded:
        steps = [lst[a:a + 32] for lst in lists for a in range(0, len(lst), 32)]
    else:
        lanes = [lists[r][s::3] for r in range(9) for s in range(3)]
        steps = [[ln[t] for ln in lanes if t < len(ln)] for t in range(max(len(ln) for ln in lanes))]
    for step in steps:
        if hcount > BG_HIT_CAP - 32:
            with np.errstate(over="ignore"):
                sc = _fdiv(_fmul(_fmul(_fmul(f32(1.0 if cl.dual else 3.0), f32(n)), f32(nsample)), f32(tested)),
                           _fmul(f32(hcount), f32(total)))
            gc = f32(f32(total - tested) + f32(2240.0))
            if nsample > BG_COMPACT_MAX:
                ev.add("overflow_nsample")
                return ev, None, None
            if not dense and sc < gc:
                ev.add("overflow_cost")
                return ev, None, None
            ev.add("compact" if not dense else "compact_again")
            buf = sorted(buf)
            tau = buf[nsample - 1]
            buf = buf[:nsample]
            hcount, dense = nsample, True
        for k in step:
            tested += 1
            if hits[k]:
                if tau is not None and not k < tau:
                    ev.add("tau_reject")
                    continue
                buf.append(k)
                hcount += 1
    return ev, sorted(buf), dense


def bg_query(cl, q, hits, nsample):
    """ball_group_kernel on one query of cloud ``cl`` (a BgCloud); ``hits`` is the query's boolean hit row.  Returns the
    set of regime tags (decisions on which the two extreme within-cell orders disagree are left out)."""
    tags = set()
    n = cl.n
    nh = int(hits.sum())
    cnt = min(nh, nsample)
    tags.add("empty_row" if cnt == 0 else "full_row" if cnt == nsample else "short_row")
    scan = True
    if cl.use_grid and not _qfinite(q):
        tags.add("query_nonfinite")
    elif cl.use_grid:
        rngs = cl.ranges(q)
        lens = [int(cl.start[c[-1] + 1] - cl.start[c[0]]) if c else 0 for c in rngs]
        total, longest = sum(lens), max(lens)
        if cl.dual and 4 * total > n:
            tags.add("scan_instead")
        else:
            crowded = longest > 48
            tags.add("walk_crowded" if crowded else "walk_balanced")
            nb_hits = []
            runs = []
            for order in ("first", "last"):
                lists = []
                for c in rngs:
                    lst = []
                    for cell in c:
                        members = np.nonzero(cl.cell == cell)[0]
                        hm = members[hits[members]]
                        rest = members[~hits[members]]
                        lst += list(hm) + list(rest) if order == "first" else list(rest) + list(hm[::-1])
                    lists.append(lst)
                runs.append(_walk(cl, lists, crowded, hits, total, nsample))
            (e0, b0, d0), (e1, b1, d1) = runs
            tags |= e0 & e1
            over0, over1 = b0 is None, b1 is None
            want = list(np.nonzero(hits)[0][:nsample])
            for b_, d_ in ((b0, d0), (b1, d1)):
                if b_ is not None:  # the walk's row is the oracle's, whatever the order
                    got = b_[:nsample] if d_ else b_[:min(len(b_), nsample)]
                    assert got == want, ("walk row differs from the oracle", got[:8], want[:8])
                    nb_hits.append(len(b_))
            if not over0 and not over1:
                scan = False
                hc = nb_hits[0] if nb_hits[0] == nb_hits[1] else None
                if hc is not None:
                    nreg = (hc + 31) >> 5
                    tags.add("sort1" if nreg <= 1 else "sort2" if nreg == 2 else "sort4" if nreg <= 4 else "sort8")
            elif over0 != over1:  # overflow or not depends on the order: no scan tag
                return tags | {"overflow_order_dependent"}
    if scan:
        src = "shared" if (not cl.use_grid or cl.dual) else "global"
        tags.add(f"scan_{src}_{'buffered' if nsample <= BG_HIT_CAP else 'unbuffered'}")
    return tags


# ----------------------------------------------------------------------------------------- bq_grid_query_kernel
def gq_query(pts, geo, q, hits, nsample):
    """bq_grid_query_kernel on one query of a flagged cloud"""
    tags = set()
    nh = int(hits.sum())
    cnt = min(nh, nsample)
    tags.add("empty_row" if cnt == 0 else "full_row" if cnt == nsample else "short_row")
    if not _qfinite(q):
        return tags | {"query_nonfinite"}
    c = cells(pts, geo)
    qc = cells(np.asarray(q, f32)[None], geo, query=True)[0]
    near = np.ones(len(pts), bool)
    for a in range(3):
        lo, hi = max(qc[a] - 1, 0), min(qc[a] + 1, geo["dims"][a] - 1)
        near &= (c[:, a] >= lo) & (c[:, a] <= hi)
    hn = int((hits & near).sum())
    assert hn == nh, "a hit outside the query's 3x3x3 neighbourhood"
    tags.add("hit_overflow" if hn > GQ_HIT_CAP else "rank_sort")
    return tags


# ------------------------------------------------------------------------------------------- ball_query_kernel
def pick_group(b, m, forced=0):
    if forced > 0:
        return forced
    g = 1
    while g < 32 and b * m * g < SMS * 2048:
        g *= 2
    return g


def bf_tags(n, m, nsample, G, hit_mat):
    """ball_query_kernel<G> on one cloud: tiles, odd n, and CTAs whose rows are all full before the last tile"""
    tags = {f"G{G}"}
    if n > BQ_TILE:
        tags.add("multi_tile")
    if n % 2:
        tags.add("odd_n")
    if n > BQ_TILE:
        last = ((n - 1) // BQ_TILE) * BQ_TILE
        qpb = 256 // G
        for a in range(0, m, qpb):
            rows = hit_mat[a:a + qpb]
            if all(np.count_nonzero(r[:last]) >= nsample for r in rows):
                tags.add("early_exit")
                break
    return tags
