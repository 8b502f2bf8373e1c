#!/usr/bin/env python
"""Randomised differential test of per-cloud lengths in both kNN kernels (TEST TOOL, runs on a GPU box).

    python tests/fuzz_knn_ragged_gpu.py [--seconds 120] [--seed 0] [--json out.json]

Two cases, each ``draw_<case>(rs)`` (parameters and inputs with numpy alone, no device) and ``run_<case>(p)``:

- ``knn_ragged``: ``knn_point(k, xyz1, xyz2, lengths=, query_lengths=)`` (knn_kernel<KC, true>, csrc/knn.cu), self-kNN
  included, against tests/knn_ragged_oracle.py's restatement of the contract on the C oracle;
- ``layer_ragged``: ``sample_knn(lengths=)`` (the overlapped knn_group_kernel<KC, true> of csrc/sa_fused.cu, or the
  sequential ops) against the oracle chain on each truncated cloud, plus the column-0 filler.

The clouds, queries, k and n come from tests/fuzz_knn_gpu.py's generators (imported, not copied: its own draws are
untouched).  Lengths aim at the edges: 1, k - 1, k, k + 1, the 1024-point tile edges, n and random values; device
lengths are sometimes out of range (the kernels clamp them).  The padding is poisoned (NaN, ±inf, a far point) or a
copy of real points.  Indices must be bit-exact and so must every float, except that a NaN equals any NaN.
tests/test_fuzz_knn_ragged_cpu.py replays the draws of the fixed slice and requires that they reach every regime.
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
import fuzz_knn_gpu as F  # noqa: E402  (cloud, query, k and n generators)
from fuzz_gpu import log_n  # noqa: E402
from knn_ragged_oracle import oracle_knn_ragged, oracle_sample_knn_ragged  # noqa: E402
from pointnet2_b200 import _lib  # noqa: E402
from pointnet2_b200.sa_layer import sample_knn  # noqa: E402
from pointnet2_b200.tf_grouping import knn_point  # noqa: E402

dev = torch.device("cuda:0")  # only dereferenced when a case runs

# the slice tests/test_fuzz_knn_ragged_gpu.py runs, and tests/test_fuzz_knn_ragged_cpu.py checks the coverage of
SLICE_SEEDS = (81, 82, 83)
SLICE_ITERATIONS = 24  # twelve of each case per seed


def draw_lengths(rs, b, n, k):
    """per-cloud lengths at the edges; sometimes out of range (``raw``: what the device tensor holds)"""
    edges = [1, k - 1, k, k + 1, 1023, 1024, 1025, n, n - 1, int(rs.randint(1, n + 1))]
    lens = [min(max(int(rs.choice(edges)), 1), n) for _ in range(b)]
    raw = list(lens)
    if rs.rand() < 0.2:
        j = int(rs.randint(b))
        raw[j] = int(rs.choice([0, -5])) if lens[j] == 1 else n + int(rs.randint(1, 50)) if lens[j] == n else lens[j]
    return lens, raw


def draw_pad(rs):
    return str(rs.choice(["poison", "copy"]))


def apply_pad(x, lengths, kind, rs_seed):
    rs = np.random.RandomState(rs_seed)
    x = x.copy()
    for i, ln in enumerate(lengths):
        rows = np.arange(ln, x.shape[1])
        if not len(rows):
            continue
        if kind == "poison":
            x[i, rows] = np.float32(rs.choice([np.nan, np.inf, -np.inf, 1e30]))
            x[i, rows[::2]] = (50.0, -50.0, 50.0)
        else:
            x[i, rows] = x[i, rows % ln]
    return x


# ------------------------------------------------------------------------------------------------------ knn_ragged
def draw_knn_ragged(rs):
    b = int(rs.randint(1, 4))
    k = F.draw_k(rs, 128)
    n = F.draw_n(rs, k, 4000)
    k = min(k, n)  # the row stride bounds k; the lengths may not
    self_knn = bool(rs.rand() < 0.25) and b * n * n * k <= F.MAX_ROW_ROUNDS  # the oracle sorts n rows of n
    m = n if self_knn else F._bound_m(b, n, k, log_n(rs, 1, 300))
    kind, xyz, pool = F.draw_cloud(rs, b, n, k, m)
    lens, raw = draw_lengths(rs, b, n, k)
    if self_knn:
        q, qlens, qraw = xyz, lens, raw
    else:
        q = F.draw_queries(rs, xyz, pool, m)
        qlens = [int(rs.randint(1, m + 1)) if rs.rand() < 0.5 else m for _ in range(b)] if rs.rand() < 0.5 else None
        qraw = qlens
    return dict(case="knn_ragged", b=b, n=n, m=m, k=k, kind=kind, self_knn=self_knn, lengths=lens, raw_lengths=raw,
                query_lengths=qlens, raw_query_lengths=qraw, pad=draw_pad(rs), pad_seed=int(rs.randint(1 << 30)),
                data_lengths=bool(self_knn or qlens is None or rs.rand() < 0.8), xyz=xyz, q=q)


def run_knn_ragged(p):
    lens = p["lengths"] if p["data_lengths"] else None
    x = apply_pad(p["xyz"], lens or [p["n"]] * p["b"], p["pad"], p["pad_seed"])
    q = x if p["self_knn"] else (apply_pad(p["q"], p["query_lengths"], p["pad"], p["pad_seed"] + 1)
                                 if p["query_lengths"] else p["q"])
    dl = torch.tensor(p["raw_lengths"], dtype=torch.int32, device=dev) if lens else None
    ql = None
    if p["query_lengths"]:
        ql = dl if p["self_knn"] else torch.tensor(p["raw_query_lengths"], dtype=torch.int32, device=dev)
    xt = F.T(x)
    val, idx = knn_point(p["k"], xt, xt if p["self_knn"] else F.T(q), lengths=dl, query_lengths=ql)
    wv, wi = oracle_knn_ragged(p["k"], x, q, lens, p["query_lengths"])
    return bool(np.array_equal(F.N(idx), wi) and F.same_floats(F.N(val), wv))


# ---------------------------------------------------------------------------------------------------- layer_ragged
def draw_layer_ragged(rs):
    path, ctas = int(rs.choice([0, 1, 2])), int(rs.choice([0, 1, 1000]))
    b = int(rs.randint(1, 4))
    k = F.draw_k(rs, 64 if path == 1 else 128)
    n = min(F.draw_n(rs, k, 8192), 8192)
    k = min(k, n)
    npoint = int(rs.choice([1, 2, n // 4 + 1, n // 2 + 1, n, n + 3, log_n(rs, 1, n + 3)]))
    npoint = F._bound_m(b, n, k, min(npoint, 400))
    kind, xyz, _ = F.draw_cloud(rs, b, n, k, npoint)
    lens, raw = draw_lengths(rs, b, n, k)
    return dict(case="layer_ragged", b=b, n=n, npoint=npoint, k=k, kind=kind, path=path, consumer_ctas=ctas,
                lengths=lens, raw_lengths=raw, pad=draw_pad(rs), pad_seed=int(rs.randint(1 << 30)),
                center=bool(rs.rand() < 0.6), want_grouped=bool(rs.rand() < 0.7), want_dist=bool(rs.rand() < 0.6), xyz=xyz)


PATHS = {"overlapped": 0, "sequential": 0}  # which path the layer_ragged cases took


def run_layer_ragged(p):
    lib = _lib.load()
    b, n, m, k = p["b"], p["n"], p["npoint"], p["k"]
    x = apply_pad(p["xyz"], p["lengths"], p["pad"], p["pad_seed"])
    try:
        lib.pn2_set_sa_knn_path(p["path"])
        lib.pn2_set_sa_consumer_ctas(p["consumer_ctas"])
        overlapped = int(lib.pn2_sa_knn_layer_workspace_bytes(b, n, m, k)) == 0
        out = sample_knn(m, k, F.T(x), center=p["center"], want_grouped=p["want_grouped"], want_dist=p["want_dist"],
                         lengths=torch.tensor(p["raw_lengths"], dtype=torch.int32, device=dev))
        torch.cuda.synchronize(dev)
    finally:
        lib.pn2_set_sa_knn_path(0)
        lib.pn2_set_sa_consumer_ctas(0)
    PATHS["overlapped" if overlapped else "sequential"] += 1
    ok = True
    if p["path"] == 1:
        ok = overlapped == F.overlapped_can_run(b, n, k)
    elif p["path"] == 2:
        ok = not overlapped
    want = oracle_sample_knn_ragged(m, k, x, p["lengths"], p["center"])
    fi, nx, idx, dist, g = out
    ok = ok and np.array_equal(F.N(fi), want[0]) and np.array_equal(F.N(nx).view(np.int32), want[1].view(np.int32))
    ok = ok and np.array_equal(F.N(idx), want[2])
    ok = ok and (dist is None) != p["want_dist"] and (g is None) != p["want_grouped"]
    if dist is not None:
        ok = ok and F.same_floats(F.N(dist), want[3])
    if g is not None:
        ok = ok and F.same_floats(F.N(g), want[4])
    return bool(ok)


CASES = ["knn_ragged", "layer_ragged"]
DRAW = {name: globals()["draw_" + name] for name in CASES}
RUN = {name: globals()["run_" + name] for name in CASES}


def draws(seed: int, iterations: int):
    """The parameters ``run(seed, iterations)`` uses, without a device (the run_* functions draw nothing)."""
    rs = np.random.RandomState(seed)
    return [DRAW[CASES[it % len(CASES)]](rs) for it in range(iterations)]


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
        fails.append(dict(F.public(p), seed=seed, iteration=it))
    return ok, fails[-1] if not ok else None


def run(seed: int, iterations: int):
    """``iterations`` random cases (alternating knn_ragged and layer_ragged); returns (counts, failures)."""
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
    counts, fails = {}, []
    t0 = time.time()
    it = 0
    while time.time() - t0 < args.seconds:
        ok, fail = _one(rs, it, args.seed, counts, fails, catch=True)
        if not ok:
            print("FAIL", json.dumps(fail), flush=True)
        it += 1
    summary = dict(seed=args.seed, seconds=round(time.time() - t0, 1), cases=counts, layer_paths=dict(PATHS), failures=fails)
    print(json.dumps(summary))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(summary, f, indent=1)
    sys.exit(1 if fails else 0)


if __name__ == "__main__":
    main()
