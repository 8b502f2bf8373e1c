#!/usr/bin/env python
"""Randomised differential test of the three ball-query kernels against the C oracle (TEST TOOL, runs on a GPU box).

    python tests/fuzz_ball_gpu.py [--seconds 120] [--seed 0] [--json out.json]

Three cases, each ``draw_<case>(rs)`` (parameters and inputs with numpy alone, no device) and ``run_<case>(p)``:

- ``bq_op``: ``query_ball_point`` under ``pn2_set_bq_mode`` 0 (automatic), 1 (brute force) or 2 (global grid) and
  ``pn2_set_bq_group`` 0 or a forced G; or the split ``pn2_ball_grid_build`` + ``pn2_query_ball_point_prebuilt``,
  whose per-cloud parameter block (flag, dims, origin, inv_h) is also held to tests/ball_regimes.py bit for bit;
- ``ball_group``: ``ball_group`` (ball_group_kernel with free queries), centred or raw, with or without grouped_xyz;
- ``bq_layer``: ``sample_group`` / ``sample_group_msg`` (the overlapped ball_group_kernel, or the sequential ops past
  n = 8192), with ``pn2_set_sa_consumer_ctas`` in {0, 1, 3} and sometimes per-cloud lengths.  The path that ran is
  recorded from the launch count and checked against the rule.

Everything is bit-exact against ``oracle_query_ball_point`` / ``oracle_group_point`` (and oracle_fps for the layer):
raw grouped coordinates as bit patterns (a gather copies NaN payloads), centred ones with one float32 subtraction,
where any NaN equals any NaN (the device's subtraction returns its canonical NaN).  Besides fuzz_gpu's U/S/D/G/L
clouds the draws plant NaN and ±inf points, NaN / ±inf / −0.0 queries, shells at r ± a few ulps, lattices on the
cell edges, coincident clusters of more than 256 points, coordinates near 1e19 (d² overflows) and 1e-22 apart (d²
underflows), clouds NaN on a whole axis, radii on both sides of 1e-20 and 1e30, nsample on the hit-buffer edges and
n on the kernels' edges.  tests/test_fuzz_ball_cpu.py replays the draws of the fixed slice and requires that they
reach every regime of tests/ball_regimes.py.  A failure is printed with the seed, the iteration and its parameters;
``run(seed, iteration + 1)`` reproduces it on any machine.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.abspath(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import ball_regimes as R  # noqa: E402
from fuzz_gpu import cloud, log_n  # noqa: E402  (the U/S/D/G/L cloud distributions)
from oracle import oracle as O  # noqa: E402
from pointnet2_b200 import _lib  # noqa: E402

dev = torch.device("cuda:0")  # only dereferenced when a case runs

# the slice tests/test_fuzz_ball_gpu.py runs, and tests/test_fuzz_ball_cpu.py checks the coverage of
SLICE_SEEDS = (71, 75, 76)
SLICE_ITERATIONS = 60  # twenty of each case per seed

NSAMPLE_EDGES = [1, 2, 127, 128, 129, 224, 225, 256, 257, 300]
N_EDGES = [511, 512, 2047, 2048, 4863, 4864, 8192, 8193, 9727, 9728]
MAX_POINTS = 24_000_000  # b * m * n: the oracle's distance tests (and the CPU replay's full hit rows)
NAN_BITS = np.int32(0x7FC12345)  # a quiet NaN with a payload a gather must copy


def T(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


def N(t):
    return t.detach().cpu().numpy()


def same_floats(got, want):
    """bit-identical, except that any NaN equals any NaN"""
    got, want = np.asarray(got, np.float32), np.asarray(want, np.float32)
    if got.shape != want.shape:
        return False
    same = got.view(np.int32) == want.view(np.int32)
    return bool(np.all(same | (np.isnan(got) & np.isnan(want))))


def _nan():
    return NAN_BITS.view(np.float32)


# ------------------------------------------------------------------------------------------------------ clouds
def _ulps(x, k):
    x = np.float32(x)
    for _ in range(abs(k)):
        x = np.nextafter(x, np.float32(np.inf if k > 0 else -np.inf), dtype=np.float32)
    return np.float32(x)


def draw_cloud(rs, b, n, kind=None):
    """(kind, xyz (b, n, 3), scale, query pool or None, radius hint or None): a base kind of fuzz_gpu.cloud or an
    adversarial one, its extent, the queries it is built around and the radius it is built for"""
    if kind is None:
        kind = str(rs.choice(["base", "C", "K", "E", "Z", "O", "X", "F"], p=[0.3, 0.14, 0.16, 0.1, 0.07, 0.07, 0.05, 0.11]))
    pool, hint = None, None
    if kind == "base":
        kind, xyz = cloud(rs, b, n)
    elif kind == "C":  # coincident clusters of more than 256 points: heavy cells, crowded walks, dense balls
        xyz = rs.random_sample((b, n, 3)).astype(np.float32)
        for i in range(b):
            for _ in range(int(rs.randint(1, 4))):
                cnt = min(n, int(rs.randint(257, 700)))
                xyz[i, rs.choice(n, cnt, replace=False)] = rs.random_sample(3).astype(np.float32)
    elif kind == "K":  # a blob of ~1000 points a few radii wide in a sparse cloud: hit buffers that fill and compact
        xyz = rs.random_sample((b, n, 3)).astype(np.float32)
        hint = 0.04
        pool = np.zeros((b, 2, 3), np.float32)
        for i in range(b):
            for j in range(2):
                c = rs.uniform(0.2, 0.8, 3).astype(np.float32)
                pool[i, j] = c
                cnt = min(n // 3, int(rs.randint(600, 1500)))
                at = np.sort(rs.choice(n, cnt, replace=False))
                blob = (c + rs.uniform(-1.2, 1.2, (cnt, 3)) * hint).astype(np.float32)
                # higher z, lower index: after the first compaction the walk's later ranges still bring hits below tau
                xyz[i, at] = blob[np.argsort(-blob[:, 2], kind="stable")]
    elif kind == "E":  # a lattice on the cell edges: 15 cells of 1/16 per axis, every point at mn + k h
        xyz = (rs.randint(0, 16, (b, n, 3)) * np.float32(1 / 16)).astype(np.float32)
        xyz[:, 0] = 0.0
        xyz[:, -1] = np.float32(15 / 16)
    elif kind == "Z":  # coordinates ~1e-22 apart: squares of 2^-75 round to 0
        xyz = (rs.randint(-6, 7, (b, n, 3)) * np.float32(2.0 ** -75)).astype(np.float32)
    elif kind == "O":  # coordinates ~1e19: most squared distances overflow to inf
        xyz = (rs.uniform(-1, 1, (b, n, 3)) * 2e19).astype(np.float32)
    elif kind == "X":  # every point NaN on one axis: a hit in every ball, whatever the other two coordinates
        xyz = rs.random_sample((b, n, 3)).astype(np.float32)
        xyz[:, :, int(rs.randint(3))] = _nan()
        hint = 0.05  # small enough for a 16-cell grid on the other two axes
    else:  # "F": per cloud, grid-friendly (spread) or grid-hostile (a tight blob): both sides of the ¼ rule
        xyz = rs.random_sample((b, n, 3)).astype(np.float32)
        hostile = rs.rand(b) < rs.choice([0.2, 0.5, 0.85])
        xyz[hostile] = (xyz[hostile] * np.float32(0.001)).astype(np.float32)
    if kind not in ("X", "K") and rs.rand() < 0.25:  # NaN / ±inf points
        for i in range(b):
            for _ in range(int(rs.randint(1, 3))):
                bad = np.float32(rs.choice([np.nan, np.nan, np.inf, -np.inf]))
                bad = _nan() if np.isnan(bad) else bad
                p = int(rs.randint(n))
                if rs.rand() < 0.5:
                    xyz[i, p] = bad
                else:
                    xyz[i, p, rs.randint(3)] = bad
    fin = xyz[np.isfinite(xyz)]
    scale = float(fin.max() - fin.min()) if fin.size else 1.0
    return kind, xyz, (scale if scale > 0 else 1.0), pool, hint


def draw_radius(rs, scale, hint=None):
    u = rs.rand()
    if hint is not None and u > 0.2:
        return float(np.float32(hint))
    if u < 0.05:
        return float(_ulps(np.float32(1e-20), int(rs.choice([-1, 0, 1, 2]))))  # the threshold < 0 edge
    if u < 0.08:
        return 1e30  # threshold = FLT_MAX
    return float(np.float32(scale * np.exp(rs.uniform(np.log(0.005), np.log(0.7)))))


def draw_nsample(rs, n):
    if rs.rand() < 0.7:
        return int(rs.choice(NSAMPLE_EDGES + [n + int(rs.randint(1, 4))]))
    return int(rs.randint(1, 400))


def draw_n(rs, lo, hi):
    if rs.rand() < 0.6:
        e = [v for v in N_EDGES if lo <= v <= hi]
        return int(rs.choice(e)) if e else log_n(rs, lo, hi)
    n = log_n(rs, lo, hi)
    return n | 1 if rs.rand() < 0.5 and n < hi else n


def shell(rs, xyz, q, radius):
    """points at r ± a few ulps along one axis from chosen queries: the threshold decides each of them"""
    b, n, _ = xyz.shape
    r = np.float32(radius)
    for i in range(b):
        for j in rs.randint(0, q.shape[1], min(q.shape[1], 6)):
            c = q[i, j]
            if not np.all(np.isfinite(c)):
                continue
            for _ in range(int(rs.randint(2, 9))):
                a = int(rs.randint(3))
                p = c.copy()
                p[a] = np.float32(c[a] + _ulps(r, int(rs.randint(-8, 9))))
                xyz[i, int(rs.randint(n))] = p
            p = exact_threshold_point(c, int(j) % 3, radius)
            if p is not None:  # d² == the threshold exactly: a hit, by the narrowest margin
                xyz[i, (int(j) * 7919 + i) % n] = p


def exact_threshold_point(c, a0, radius):
    """a point on one axis from c (axis a0 first) whose squared distance, as the kernels round it, equals the threshold
    (None if the 64 floats nearest c + r on each axis hold none)"""
    thr = np.float32(O.oracle_ball_threshold(radius))
    if not thr > 0:
        return None
    with np.errstate(over="ignore", invalid="ignore"):
        for a in (a0, (a0 + 1) % 3, (a0 + 2) % 3):
            x = np.float32(c[a] + np.float32(np.sqrt(thr)))
            for k in range(-32, 33):
                px = _ulps(x, k)
                d = np.float32(c[a] - px)
                if np.float32(d * d) == thr:
                    p = c.copy()
                    p[a] = px
                    return p
    return None


def draw_queries(rs, xyz, m, pool=None):
    """the kind's own centres, copies of cloud points, free points over (and beyond) the box; then −0.0 coordinates
    and NaN / ±inf queries"""
    b, n, _ = xyz.shape
    if pool is not None and rs.rand() < 0.6:
        q = np.stack([pool[i, rs.randint(0, pool.shape[1], m)] for i in range(b)])
    elif rs.rand() < 0.5:
        q = xyz[:, rs.randint(0, n, m)].copy()
    else:
        fin = xyz[np.isfinite(xyz)]
        lo, hi = (float(fin.min()), float(fin.max())) if fin.size else (0.0, 1.0)
        q = (lo + (hi - lo) * (rs.random_sample((b, m, 3)) * 1.4 - 0.2)).astype(np.float32)
    q = q.astype(np.float32)
    if rs.rand() < 0.25:
        q[q == 0] = np.float32(-0.0)
        q[:, rs.randint(0, m, max(1, m // 4)), rs.randint(3)] = np.float32(-0.0)
    if rs.rand() < 0.25:
        bad = np.float32(rs.choice([np.nan, np.inf, -np.inf]))
        q[rs.randint(b), rs.randint(0, m, int(rs.randint(1, 4))), rs.randint(3)] = bad
    return q


def _bound_m(b, n, m):
    return max(1, min(m, MAX_POINTS // (b * n)))


# ------------------------------------------------------------------------------------------------------ bq_op
def draw_bq_op(rs):
    mode = int(rs.choice([0, 0, 1, 2]))
    group = int(rs.choice([1, 2, 4, 8, 16, 32])) if rs.rand() < 0.35 else 0
    recipe = str(rs.choice(["free", "wide", "global"], p=[0.4, 0.25, 0.35]))
    kind = None
    if recipe == "global":  # the global-memory grid: build + query + brute force, or the split entries
        b = int(rs.choice([1, 2, 4, 8]))
        n = int(rs.choice([2048, 2049, 3001, 4864, 9728]))
        m = _bound_m(b, n, log_n(rs, 1, 600))
        mode = 2
        kind = str(rs.choice(["K", "F", "C", "base"]))
        if kind == "F":  # enough clouds for the ¼ rule to go either way
            b, m = 8, _bound_m(8, n, m)
    elif recipe == "wide":  # b * m >= 4096 at 2048 <= n <= 9727: the automatic mode runs ball_group_kernel
        b = int(rs.choice([1, 2, 4, 8]))
        n = draw_n(rs, 2048, 4864)
        m = _bound_m(b, n, -(-4096 // b) + int(rs.randint(0, 64)))
    else:
        b = int(rs.randint(1, 9)) if rs.rand() < 0.3 else int(rs.randint(1, 4))
        n = draw_n(rs, 1, 16000)
        m = _bound_m(b, n, log_n(rs, 1, 600))
    split = bool(R.GRID_MIN_N <= n and rs.rand() < (0.5 if recipe == "global" else 0.15))
    kind, xyz, scale, pool, hint = draw_cloud(rs, b, n, kind)
    radius = draw_radius(rs, scale, hint)
    if split and rs.rand() < 0.1:
        radius = float(np.float32(1e-20))  # both split entries refuse it
    s = draw_nsample(rs, n)
    q = draw_queries(rs, xyz, m, pool)
    if rs.rand() < 0.3:
        shell(rs, xyz, q, radius)
    return dict(case="bq_op", b=b, n=n, m=m, nsample=s, radius=radius, kind=kind, mode=mode, group=group, split=split,
                xyz=xyz, q=q)


def params_block(ws, b, n):
    """the per-cloud parameter blocks of the global grid's workspace: (b, 8) int32"""
    stride = 8 + n + 16 ** 3 + 1  # grid_ws_ints_per_cloud
    return N(ws).view(np.int32).reshape(b, stride)[:, :8]


def model_block(pts, radius, nsample):
    """what bq_grid_build_kernel writes into a cloud's parameter block (flag None: undecided)"""
    g = R.geometry(pts, radius)
    flag, _ = R.global_flag(pts, radius, nsample)
    bits = [int(np.float32(v).view(np.int32)) for v in (*g["mn"], g["inv_h"])]
    return flag, [*g["dims"], *bits[:3], bits[3]]


def run_bq_op(p):
    from pointnet2_b200.tf_grouping import query_ball_point
    lib = _lib.load()
    b, n, m, s, r, x, q = p["b"], p["n"], p["m"], p["nsample"], p["radius"], p["xyz"], p["q"]
    ok = True
    try:
        lib.pn2_set_bq_mode(p["mode"])
        lib.pn2_set_bq_group(p["group"])
        if p["split"]:
            wsb = int(lib.pn2_query_ball_point_workspace_bytes(b, n))
            ws = torch.zeros(wsb, dtype=torch.uint8, device=dev)
            tx, tq = T(x), T(q)
            idx = torch.empty((b, m, s), dtype=torch.int32, device=dev)
            cnt = torch.empty((b, m), dtype=torch.int32, device=dev)
            rc = lib.pn2_ball_grid_build(b, n, r, s, tx.data_ptr(), ws.data_ptr(), wsb, None)
            if rc == 0:
                rc = lib.pn2_query_ball_point_prebuilt(b, n, m, r, s, tx.data_ptr(), tq.data_ptr(), idx.data_ptr(),
                                                       cnt.data_ptr(), ws.data_ptr(), wsb, None)
            torch.cuda.synchronize(dev)
            if O.oracle_ball_threshold(r) < 0:  # radius <= 1e-20: both halves refuse it
                return rc != 0
            ok = rc == 0
            blocks = params_block(ws, b, n)
            for i in range(b):
                flag, rest = model_block(x[i], r, s)
                got = [int(v) for v in blocks[i]]
                # the origin as a value: which of +0 and -0 fminf keeps depends on the reduction order, and both bin
                # every coordinate into the same cell
                origin_ok = np.array_equal(np.int32(got[4:7]).view(np.float32), np.int32(rest[3:6]).view(np.float32))
                ok = ok and got[1:4] == rest[:3] and origin_ok and got[7] == rest[6]
                ok = ok and (flag is None or got[0] == int(flag))
        else:
            idx, cnt = query_ball_point(r, s, T(x), T(q))
            torch.cuda.synchronize(dev)
    finally:
        lib.pn2_set_bq_mode(0)
        lib.pn2_set_bq_group(0)
    oi, oc = O.oracle_query_ball_point(r, s, x, q)
    return bool(ok and np.array_equal(N(idx), oi) and np.array_equal(N(cnt), oc))


# -------------------------------------------------------------------------------------------------- ball_group
def grouped_oracle(x, oi, centre, center):
    og = O.oracle_group_point(x, oi)
    if center:
        with np.errstate(invalid="ignore"):  # inf - inf: NaN, as on the device
            og = (og - centre[:, :, None, :]).astype(np.float32)
    return og


def same_grouped(got, want, center):
    if center:
        return same_floats(got, want)
    return got.shape == want.shape and np.array_equal(got.view(np.int32), want.view(np.int32))


def draw_ball_group(rs):
    b = int(rs.choice([1, 2, 3, 5, 8, 33, 140])) if rs.rand() < 0.4 else int(rs.randint(1, 5))
    u = rs.rand()
    compact = u < 0.3  # a blob in a large single-layout cloud: hit buffers that compact, then filter by tau
    nan_axis = 0.3 <= u < 0.4  # a cloud NaN on a whole axis: every point is a hit in every ball
    n = int(rs.randint(4864, 9728)) if compact else int(rs.randint(512, 9728)) if nan_axis else draw_n(rs, 1, 9727)
    # b * m on both sides of the CTAs-per-cloud ramp (132 // b CTAs, at most one warp per query)
    m = int(rs.choice([1, 31, 33, 200, 32 * (132 // b) + 1, log_n(rs, 1, 5000)]))
    m = _bound_m(b, n, max(1, m))
    kind, xyz, scale, pool, hint = draw_cloud(rs, b, n, "K" if compact else "X" if nan_axis else None)
    radius = draw_radius(rs, scale, hint)
    q = draw_queries(rs, xyz, m, pool)
    if rs.rand() < 0.3:
        shell(rs, xyz, q, radius)
    s = int(rs.choice([32, 64, 127, 128])) if compact else draw_nsample(rs, n)
    return dict(case="ball_group", b=b, n=n, m=m, nsample=s, radius=radius, kind=kind,
                center=bool(rs.rand() < 0.6), want_grouped=bool(rs.rand() < 0.8), xyz=xyz, q=q)


def run_ball_group(p):
    from pointnet2_b200.sa_layer import ball_group
    x, q, r, s = p["xyz"], p["q"], p["radius"], p["nsample"]
    if O.oracle_ball_threshold(r) < 0:  # ball_group refuses a radius no distance can pass
        try:
            ball_group(r, s, T(x), T(q), center=p["center"], want_grouped=p["want_grouped"])
        except RuntimeError:
            return True
        return False
    idx, cnt, g = ball_group(r, s, T(x), T(q), center=p["center"], want_grouped=p["want_grouped"])
    torch.cuda.synchronize(dev)
    oi, oc = O.oracle_query_ball_point(r, s, x, q)
    ok = np.array_equal(N(idx), oi) and np.array_equal(N(cnt), oc) and (g is None) != p["want_grouped"]
    if g is not None:
        ok = ok and same_grouped(N(g), grouped_oracle(x, oi, q, p["center"]), p["center"])
    return bool(ok)


# ---------------------------------------------------------------------------------------------------- bq_layer
def layer_overlapped(n, radii):
    """sa_layer_msg's rule: one sampling CTA per cloud (n <= 8192), the cloud fits ball_group_kernel, every threshold
    >= 0"""
    return n <= 8192 and R.bg_fits(n) and all(O.oracle_ball_threshold(r) >= 0 for r in radii)


def qbp_launches(b, n, m, radius):
    """kernel launches of query_ball_point_ws in the automatic mode with the layer's workspace"""
    if O.oracle_ball_threshold(radius) < 0:
        return 0  # two memsets
    if n >= R.GRID_MIN_N and R.bg_fits(n):
        return 1  # ball_group_kernel, or the brute-force kernel below 4096 queries
    return 3 if R.GRID_MIN_N <= n <= (1 << 20) else 1


def layer_launches(p):
    b, n, m, radii = p["b"], p["n"], p["npoint"], p["radii"]
    if layer_overlapped(n, radii):
        return 1 + len(radii)
    return 1 + sum(qbp_launches(b, n, m, r) + (1 if p["want_grouped"] else 0) for r in radii)


def draw_bq_layer(rs):
    b = int(rs.randint(1, 5))
    n = draw_n(rs, 1, 9728)
    ragged = bool(rs.rand() < 0.3)
    lengths = None
    if ragged:  # lengths on both sides of 512: use_grid follows the length, the layout the stride
        lengths = [int(min(n, max(1, v))) for v in rs.choice([n, n - 1, 511, 512, 700, int(rs.randint(1, n + 1))], b)]
    npoint = int(rs.choice([1, 2, 64, 200, n // 4 + 1, n + 2]))
    npoint = _bound_m(b, n, min(npoint, 400))
    kind, xyz, scale, _, hint = draw_cloud(rs, b, n)
    scales = int(rs.choice([1, 1, 2, 3]))
    radii = [draw_radius(rs, scale, hint) for _ in range(scales)]
    ns = [draw_nsample(rs, n) for _ in range(scales)]
    return dict(case="bq_layer", b=b, n=n, npoint=npoint, radii=radii, ns=ns, kind=kind, lengths=lengths,
                consumer_ctas=int(rs.choice([0, 1, 3])), center=bool(rs.rand() < 0.6),
                want_grouped=bool(rs.rand() < 0.8), xyz=xyz)


PATHS = {"overlapped": 0, "sequential": 0}  # which path the bq_layer cases took


def run_bq_layer(p):
    from pointnet2_b200.sa_layer import sample_group, sample_group_msg
    lib = _lib.load()
    b, n, m, x = p["b"], p["n"], p["npoint"], p["xyz"]
    ls = p["lengths"] or [n] * b
    lens = torch.tensor(ls, dtype=torch.int32, device=dev) if p["lengths"] else None
    try:
        lib.pn2_set_sa_consumer_ctas(p["consumer_ctas"])
        before = _lib.launch_count()
        if len(p["radii"]) == 1:
            fi, nx, idx, cnt, g = sample_group(m, p["radii"][0], p["ns"][0], T(x), center=p["center"],
                                               want_grouped=p["want_grouped"], lengths=lens)
            idx, cnt, g = [idx], [cnt], [g] if g is not None else None
        else:
            fi, nx, idx, cnt, g = sample_group_msg(m, p["radii"], p["ns"], T(x), center=p["center"],
                                                   want_grouped=p["want_grouped"], lengths=lens)
        torch.cuda.synchronize(dev)
        launches = _lib.launch_count() - before
    finally:
        lib.pn2_set_sa_consumer_ctas(0)
    overlapped = layer_overlapped(n, p["radii"])
    p["overlapped"] = overlapped
    PATHS["overlapped" if overlapped else "sequential"] += 1
    ok = launches == layer_launches(p)  # the path that ran is the one the rule names
    ok = ok and (g is None) != p["want_grouped"]
    fi, nx = N(fi), N(nx)
    for i, ln in enumerate(ls):
        c = x[i:i + 1, :ln]
        o_fi = O.oracle_fps(m, c)
        o_nx = O.oracle_gather_point(c, o_fi)
        ok = ok and np.array_equal(fi[i:i + 1], o_fi) and np.array_equal(nx[i:i + 1].view(np.int32), o_nx.view(np.int32))
        for k, (r, s) in enumerate(zip(p["radii"], p["ns"])):
            oi, oc = O.oracle_query_ball_point(r, s, c, o_nx)
            ok = ok and np.array_equal(N(idx[k][i:i + 1]), oi) and np.array_equal(N(cnt[k][i:i + 1]), oc)
            if g is not None:
                ok = ok and same_grouped(N(g[k][i:i + 1]), grouped_oracle(c, oi, o_nx, p["center"]), p["center"])
    return bool(ok)


CASES = ["bq_op", "ball_group", "bq_layer"]
DRAW = {name: globals()["draw_" + name] for name in CASES}
RUN = {name: globals()["run_" + name] for name in CASES}


def draws(seed: int, iterations: int):
    """The parameters ``run(seed, iterations)`` uses, without a device (the run_* functions draw nothing)."""
    rs = np.random.RandomState(seed)
    return [DRAW[CASES[it % len(CASES)]](rs) for it in range(iterations)]


def public(p):
    """the parameters of a case without its input arrays (they follow from the seed and the iteration)"""
    return {k: v for k, v in p.items() if not isinstance(v, np.ndarray)}


def _one(rs, it, seed, counts, fails, catch):
    name = CASES[it % len(CASES)]
    p = DRAW[name](rs)
    try:
        ok = RUN[name](p)
    except Exception as e:  # noqa: BLE001 — report the exception as a failure of that case
        if not catch:
            raise
        ok = False
        p = dict(p, error=f"{type(e).__name__}: {e}")
    counts[name] = counts.get(name, 0) + 1
    if not ok:
        fails.append(dict(public(p), seed=seed, iteration=it))
    return ok, fails[-1] if not ok else None


def run(seed: int, iterations: int):
    """``iterations`` random cases (bq_op, ball_group and bq_layer in turn); returns (counts, failures)."""
    rs = np.random.RandomState(seed)
    counts, fails = {}, []
    for it in range(iterations):
        _one(rs, it, seed, counts, fails, catch=False)
    return counts, fails


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=float, default=120)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--json", type=str, default=None)
    args = ap.parse_args()
    rs = np.random.RandomState(args.seed)
    counts, fails, secs = {}, [], {}
    t0 = time.time()
    it = 0
    while time.time() - t0 < args.seconds:
        t1 = time.time()
        ok, fail = _one(rs, it, args.seed, counts, fails, catch=True)
        name = CASES[it % len(CASES)]
        secs[name] = secs.get(name, 0.0) + time.time() - t1
        if not ok:
            print("FAIL", json.dumps(fail), flush=True)
        it += 1
    summary = dict(seed=args.seed, seconds=round(time.time() - t0, 1), cases=counts, layer_paths=dict(PATHS),
                   case_seconds={k: round(v, 1) for k, v in secs.items()}, failures=fails)
    print(json.dumps(summary))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(summary, f, indent=1)
    sys.exit(1 if fails else 0)


if __name__ == "__main__":
    main()
