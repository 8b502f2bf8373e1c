#!/usr/bin/env python
"""Randomised differential test of both kNN kernels against the selection-sort oracle (TEST TOOL, runs on a GPU box).

    python tests/fuzz_knn_gpu.py [--seconds 120] [--seed 0] [--json out.json]

Two cases, each ``draw_<case>(rs)`` (parameters and inputs with numpy alone, no device) and ``run_<case>(p)``:

- ``knn_op``: ``knn_point(k, xyz1, xyz2)`` (knn_kernel<1/2/4>, csrc/knn.cu) against ``oracle_knn_point``;
- ``knn_layer``: ``sample_knn`` (the overlapped knn_group_kernel<1/2> of csrc/sa_fused.cu, or the sequential ops)
  against the oracle chain oracle_fps -> oracle_gather_point -> oracle_knn_point -> oracle_group_point, never against
  the op sequence (both would run the same KnnWarp).

Indices must be bit-exact, and so must every float, except that a NaN equals any NaN: the device's arithmetic returns
its canonical NaN where numpy keeps the payload of the input NaN.  The clouds are fuzz_gpu's U/S/D/G/L kinds plus
generators aimed at the branches of KnnWarp (knn_warp.cuh): mirrored pairs that plant equal distances at chosen
ranks, lattice shells at one exact distance, coordinates 1e-22 apart (distances underflow to 0), coordinates near
1e19 (distances overflow to inf), NaN / ±inf points before k, at k, in the first candidate group and last, and
queries that copy cloud points, carry −0.0 or are NaN.  tests/test_fuzz_knn_cpu.py replays the draws of the fixed
slice and requires that they reach every regime.  A failure is printed with the seed, the iteration and its
parameters; ``run(seed, iteration + 1)`` reproduces it on any machine.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from fuzz_gpu import cloud, log_n  # noqa: E402  (the U/S/D/G/L cloud distributions)
from knn_regimes import dist_rows  # noqa: E402
from oracle import oracle as O  # noqa: E402
from pointnet2_b200 import _lib  # noqa: E402
from pointnet2_b200.sa_layer import sample_knn  # noqa: E402
from pointnet2_b200.tf_grouping import knn_point  # noqa: E402

dev = torch.device("cuda:0")  # only dereferenced when a case runs

# the slice tests/test_fuzz_knn_gpu.py runs, and tests/test_fuzz_knn_cpu.py checks the coverage of
SLICE_SEEDS = (61, 62, 63)
SLICE_ITERATIONS = 40  # twenty of each case per seed

K_EDGES = [1, 31, 32, 33, 63, 64, 65, 96, 127, 128]  # the KC instances (k <= 32, 64, 128), full and partial
MAX_POINTS = 3_000_000      # b * m * n: the oracle's (b, m, n, 3) difference array
MAX_ROW_ROUNDS = 1.5e8      # b * m * k * n: k selection-sort rounds over whole rows
SMS = 132                   # the H100's SM count, for the layer's path prediction (knn_room)


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


# ------------------------------------------------------------------------------------------------------ clouds
def _dyadic(rs, shape, bits, hi):
    return (rs.randint(0, hi, shape) * np.float32(2.0 ** -bits)).astype(np.float32)


def _shell_offsets(r2):
    o = np.arange(-9, 10)
    g = np.stack(np.meshgrid(o, o, o, indexing="ij"), -1).reshape(-1, 3)
    return g[(g * g).sum(1) == r2]


def _plant_mirrors(rs, xyz, anchors, k):
    """for each anchor query q: the point p at a chosen rank (k - 2, k - 1, k or any) gets its exact reflection
    2q - p written over a random position, so two equal distances sit at (about) that rank"""
    n = xyz.shape[0]
    for q in anchors:
        d = dist_rows(xyz, q[None])[0]
        order = np.lexsort((np.arange(n), d))
        r = int(rs.choice([k - 2, k - 1, k - 1, k, int(rs.randint(n))]))
        r = min(max(r, 0), n - 1)
        j = int(rs.randint(n))
        if j != order[r]:
            xyz[j] = (2 * q - xyz[order[r]]).astype(np.float32)


def draw_cloud(rs, b, n, k, m):
    """(kind, xyz (b, n, 3), query pool (b, mp, 3) or None): the base kinds of fuzz_gpu.cloud or an adversarial one.
    The pool holds the queries the kind is built around (mirror anchors, shell centres)."""
    kind = str(rs.choice(["base", "M", "H", "Z", "O"], p=[0.4, 0.2, 0.15, 0.13, 0.12]))
    pool = None
    if kind == "base":
        kind, xyz = cloud(rs, b, n)
    elif kind == "M":  # mirrored pairs on a dyadic grid: every distance exact
        xyz = _dyadic(rs, (b, n, 3), 10, 1024)
        pool = _dyadic(rs, (b, int(rs.randint(1, 9)), 3), 8, 256)
        for i in range(b):
            for _ in range(int(rs.randint(1, 4))):
                _plant_mirrors(rs, xyz[i], pool[i], k)
    elif kind == "H":  # lattice shells: many points at one exact distance from a lattice query
        xyz = (rs.randint(0, 16, (b, n, 3)) * 0.125).astype(np.float32)
        pool = (rs.randint(3, 13, (b, int(rs.randint(1, 4)), 3)) * 0.125).astype(np.float32)
        for i in range(b):
            for c in pool[i]:
                off = _shell_offsets(int(rs.choice([9, 25, 50, 81])))
                cnt = int(rs.randint(1, min(n, 3 * len(off)) + 1))
                at = rs.choice(n, cnt, replace=False)
                xyz[i, at] = c + off[rs.randint(0, len(off), cnt)] * np.float32(0.125)
    elif kind == "Z":  # coordinates ~1e-22 apart: squares of 2^-75 round to 0, a few subnormals survive
        xyz = (rs.randint(-6, 7, (b, n, 3)) * np.float32(2.0 ** -75)).astype(np.float32)
        pool = (rs.randint(-6, 7, (b, 4, 3)) * np.float32(2.0 ** -75)).astype(np.float32)
    else:  # "O": coordinates ~1e19: most squared distances overflow to inf
        xyz = (rs.uniform(-1, 1, (b, n, 3)) * 2e19).astype(np.float32)
    if rs.rand() < 0.35:  # NaN / ±inf points before k, at k, in the first candidate group, last
        for i in range(b):
            for _ in range(int(rs.randint(1, 4))):
                p = int(rs.choice([rs.randint(k), k, k + rs.randint(32), n - 1]))
                if p < n:
                    bad = np.float32(rs.choice([np.nan, np.nan, np.inf, -np.inf]))
                    if rs.rand() < 0.5:
                        xyz[i, p] = bad
                    else:
                        xyz[i, p, rs.randint(3)] = bad
    return kind, xyz, pool


def draw_queries(rs, xyz, pool, m):
    """copies of cloud points (NaN rows included), the kind's own queries, free points; then −0.0 coordinates and
    NaN queries"""
    b, n, _ = xyz.shape
    r = rs.rand()
    if pool is not None and r < 0.6:
        q = np.stack([pool[i, rs.randint(0, pool.shape[1], m)] for i in range(b)])
    elif r < 0.8:
        q = xyz[:, rs.randint(0, n, m)].copy()
    else:
        fin = xyz[np.isfinite(xyz)]
        lo, hi = (float(fin.min()), float(fin.max())) if fin.size else (0.0, 1.0)
        q = (lo + (hi - lo) * rs.random_sample((b, m, 3))).astype(np.float32)
    q = q.astype(np.float32)
    if rs.rand() < 0.3:
        q[q == 0] = np.float32(-0.0)
        q[:, rs.randint(0, m, max(1, m // 4)), rs.randint(3)] = np.float32(-0.0)
    if rs.rand() < 0.2:
        q[rs.randint(b), rs.randint(0, m, int(rs.randint(1, 4))), rs.randint(3)] = np.nan
    return q


def _bound_m(b, n, k, m):
    return max(1, min(m, MAX_POINTS // (b * n), int(MAX_ROW_ROUNDS // (b * k * n))))


def draw_k(rs, kmax):
    return int(rs.choice([e for e in K_EDGES if e <= kmax])) if rs.rand() < 0.5 else int(rs.randint(1, kmax + 1))


def draw_n(rs, k, hi):
    if rs.rand() < 0.55:
        return int(rs.choice([k, k + 1, 2 * k - 1, 2 * k, 1023, 1024, 1025, 1024 + k, 2048 + 33, 3072 + 63]))
    return log_n(rs, 1, hi)


def fit_k(rs, k, n):
    return k if k <= n else (n if rs.rand() < 0.5 else int(rs.randint(1, n + 1)))


# ------------------------------------------------------------------------------------------------------ knn_op
def draw_knn_op(rs):
    b = int(rs.randint(1, 4))
    k = draw_k(rs, 128)
    n = draw_n(rs, k, 6000)
    k = fit_k(rs, k, n)
    m = _bound_m(b, n, k, log_n(rs, 1, 300))
    kind, xyz, pool = draw_cloud(rs, b, n, k, m)
    return dict(case="knn_op", b=b, n=n, m=m, k=k, kind=kind, xyz=xyz, q=draw_queries(rs, xyz, pool, m))


def run_knn_op(p):
    val, idx = knn_point(p["k"], T(p["xyz"]), T(p["q"]))
    wv, wi = O.oracle_knn_point(p["k"], p["xyz"], p["q"])
    return bool(np.array_equal(N(idx), wi) and same_floats(N(val), wv))


# --------------------------------------------------------------------------------------------------- knn_layer
def kg_warps(n, k):
    """sa_fused.cu kg_warps: warps per consumer CTA of the overlapped layer, 0 where it cannot hold (n, k)"""
    if n <= 0 or k <= 0 or k > 64 or k > n:
        return 0
    cloud_bytes = (n * 12 + 15) // 16 * 16
    if cloud_bytes >= 200 * 1024:
        return 0
    nw = min((200 * 1024 - cloud_bytes) // (24 * k), 32)
    return nw if nw >= 4 else 0


def overlapped_can_run(b, n, k):
    """the overlapped layer can run: kg_warps, one idle SM per cloud left by the sampling, one sampling CTA per
    cloud (n <= 8192)"""
    return kg_warps(n, k) > 0 and (SMS - b) // b >= 1 and n <= 8192


def draw_knn_layer(rs):
    path, ctas = int(rs.choice([0, 1, 2])), int(rs.choice([0, 1, 1000]))
    b = int(rs.randint(1, 4))
    k = draw_k(rs, 64 if path == 1 else 128)
    n = min(draw_n(rs, k, 8192), 8192)
    k = fit_k(rs, k, n)
    npoint = int(rs.choice([1, 2, n // 4 + 1, n // 2 + 1, n, n + 3, log_n(rs, 1, n + 3)]))
    npoint = _bound_m(b, n, k, min(npoint, 600))
    kind, xyz, _ = draw_cloud(rs, b, n, k, npoint)
    return dict(case="knn_layer", b=b, n=n, npoint=npoint, k=k, kind=kind, path=path, consumer_ctas=ctas,
                center=bool(rs.rand() < 0.6), want_grouped=bool(rs.rand() < 0.7), want_dist=bool(rs.rand() < 0.6),
                xyz=xyz)


PATHS = {"overlapped": 0, "sequential": 0}  # which path the knn_layer cases took


def run_knn_layer(p):
    lib = _lib.load()
    b, n, m, k, x = p["b"], p["n"], p["npoint"], p["k"], p["xyz"]
    try:
        lib.pn2_set_sa_knn_path(p["path"])
        lib.pn2_set_sa_consumer_ctas(p["consumer_ctas"])
        overlapped = int(lib.pn2_sa_knn_layer_workspace_bytes(b, n, m, k)) == 0
        fi, nx, idx, dist, g = sample_knn(m, k, T(x), center=p["center"], want_grouped=p["want_grouped"],
                                          want_dist=p["want_dist"])
        torch.cuda.synchronize(dev)
    finally:
        lib.pn2_set_sa_knn_path(0)
        lib.pn2_set_sa_consumer_ctas(0)
    p["overlapped"] = overlapped
    PATHS["overlapped" if overlapped else "sequential"] += 1
    ok = True
    if p["path"] == 1:  # the forced path is the one the CPU coverage test predicts
        ok = overlapped == overlapped_can_run(b, n, k)
    elif p["path"] == 2:
        ok = not overlapped
    o_fi = O.oracle_fps(m, x)
    o_nx = O.oracle_gather_point(x, o_fi)
    o_val, o_idx = O.oracle_knn_point(k, x, o_nx)
    ok = ok and np.array_equal(N(fi), o_fi) and np.array_equal(N(nx).view(np.int32), o_nx.view(np.int32))
    ok = ok and np.array_equal(N(idx), o_idx)
    ok = ok and (dist is None) != p["want_dist"] and (g is None) != p["want_grouped"]
    if dist is not None:
        ok = ok and same_floats(N(dist), o_val)
    if g is not None:
        og = O.oracle_group_point(x, o_idx)
        if p["center"]:
            with np.errstate(invalid="ignore"):  # inf - inf: NaN, as on the device
                og = (og - o_nx[:, :, None, :]).astype(np.float32)
        ok = ok and same_floats(N(g), og)
    return bool(ok)


CASES = ["knn_op", "knn_layer"]
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
    """``iterations`` random cases (alternating knn_op and knn_layer); returns (counts, failures)."""
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
