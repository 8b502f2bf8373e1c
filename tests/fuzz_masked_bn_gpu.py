#!/usr/bin/env python
"""Randomised differential test of the masked batch-norm + ReLU kernels (csrc/masked_bn.cu), plain and max-pooled,
forward and backward, against the exact float32 oracle (oracle_mbn_*) and tests/bn_regimes.py (TEST TOOL, runs on a
GPU box).

    python tests/fuzz_masked_bn_gpu.py [--seconds 120] [--seed 0] [--json out.json]

Each case is ``draw_<case>(rs)`` (parameters and inputs with numpy alone, no device) and ``run_<case>(p)``.  Every
case but ``torch`` calls the C ABI with explicit pointers, so the alignment of each tensor, the workspace and the
dtype code are exactly what was drawn.  Outputs are filled with a poison pattern before each call and have a guard
after their end; the padding rows of y / dx must come back 0 and the guards untouched.

The oracle restates the documented order of every sum, so everything is compared bit for bit (any NaN equals any NaN,
16-bit results rounded once with numerics.round_once) except save_invstd: the device's rsqrtf is not correctly
rounded, so save_invstd is held within 2 ulp of 1 / sqrt(var + eps) in float64 (var + eps the oracle's float32 sum),
and the oracle takes the device's own save_invstd for y and dx.

- ``plain``: pn2_masked_bn_relu_forward_typed + backward_typed.  Each case runs twice: the padding rows of x and dy
  poisoned (NaN, ±inf, far values), then copied from real rows.  The two runs must agree bit for bit.
- ``max``: pn2_masked_bn_relu_max_forward_typed + backward_typed, twice as above; its statistics and running buffers
  must also equal the plain forward's bit for bit.
- ``refused``: a refused call returns cudaErrorInvalidValue, launches nothing and leaves the outputs poisoned.
- ``torch``: layers.masked_batch_norm_relu / masked_bn_relu_max with autograd, and the registered torch.ops.pn2 ops,
  against the C-ABI call's bits, with the same running buffers and num_batches_tracked incremented.

tests/test_fuzz_masked_bn_cpu.py replays the fixed slice through bn_regimes and requires every instantiation and
regime.  A failure is printed with the seed, the iteration and its parameters; ``run(seed, iteration + 1)``
reproduces it on any machine.
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
import bn_regimes as R  # noqa: E402
import fuzz_group_gpu as G  # noqa: E402  (device buffers with poison and guard)
import numerics as NUM  # noqa: E402
from oracle import oracle as O  # noqa: E402
from pointnet2_b200 import _lib  # noqa: E402
from pointnet2_b200._tensor import ptr, stream_ptr  # noqa: E402

dev = G.dev

# the slice tests/test_fuzz_masked_bn_gpu.py runs, and tests/test_fuzz_masked_bn_cpu.py checks the coverage of; the
# elementwise grids are planned with bn_regimes.SMS multiprocessors
SLICE_SEEDS = (61, 62)
SCHEDULE = ["plain", "max", "plain", "refused", "plain", "max", "torch", "plain", "refused", "max"]
SLICE_ITERATIONS = 14 * len(SCHEDULE)

FMTS = G.FMTS
CODE = G.DTYPE_CODE
RAW = G.RAW
POISON = G.POISON
CUDA_ERROR_INVALID_VALUE = 1
# every (vec, tx) pair, idle lanes and partial last column tiles
WIDTHS = [1, 2, 3, 5, 6, 7, 9, 10, 11, 13, 14, 15, 17, 31, 33, 130,   # vec 1: tx 1, 2, 4, 8, 16, 32
          4, 8, 12, 16, 20, 32, 36, 64, 68, 128, 132, 260]           # vec 4: tx 1, 2, 4, 8, 16, 32


def log_int(rs, lo, hi):
    return G.log_int(rs, lo, hi)


# ------------------------------------------------------------------------------------------------------- draws
def draw_rows(rs, c, kind=None):
    """rows for a width: one chunk, exactly chunk_rows, 32 / 33 chunks, >= 64 chunks with a remainder, or enough for
    a second grid-stride trip of the elementwise kernels"""
    g = R.geom(1, c)
    cr = g["chunk_rows"]
    kind = kind or str(rs.choice(["small", "exact", "c32", "c33", "many", "trips"], p=[.4, .1, .12, .12, .13, .13]))
    if kind == "small":
        rows = log_int(rs, 1, cr)
    elif kind == "exact":
        rows = cr
    elif kind == "c32":
        rows = 31 * cr + int(rs.randint(1, cr + 1))
    elif kind == "c33":
        rows = 32 * cr + int(rs.randint(1, cr + 1))
    elif kind == "many":
        rows = int(rs.randint(64, 80)) * cr + int(rs.randint(1, cr))
    else:  # past one trip of the capped elementwise grid
        per_trip = R.row_blocks(g, 1 << 30) * g["ty"] * R.UNROLL
        rows = per_trip + int(rs.randint(1, per_trip // 2 + 2))
    return kind, rows


def draw_keep(rs, rows, chunk_rows, kind=None):
    kind = kind or str(rs.choice(["all", "random", "empty_chunks", "late", "one", "none"],
                                 p=[.25, .3, .15, .15, .1, .05]))
    if kind == "all":
        k = np.ones(rows, np.uint8)
    elif kind == "random":
        k = (rs.random_sample(rows) < rs.uniform(0.2, 0.95)).astype(np.uint8)
    elif kind == "empty_chunks":
        k = (rs.random_sample(rows) < 0.7).astype(np.uint8)
        chunks = -(-rows // chunk_rows)
        for ch in rs.permutation(chunks)[:max(1, chunks // 3)]:
            k[ch * chunk_rows:(ch + 1) * chunk_rows] = 0
    elif kind == "late":  # real rows only in the last part: the merges start from empty partials
        k = np.zeros(rows, np.uint8)
        start = int(rs.randint(rows // 2, rows)) if rows > 1 else 0
        k[start:] = (rs.random_sample(rows - start) < 0.8)
        k[rows - 1] = 1
    elif kind == "one":
        k = np.zeros(rows, np.uint8)
        k[int(rs.randint(rows))] = 1
    else:
        k = np.zeros(rows, np.uint8)
    return kind, k


DATA = ["normal", "constant", "far_mean", "overflow", "nonfinite", "subnormal", "ties"]


def draw_data(rs, shape, fmt, kind=None):
    """float32 values of an fmt tensor of the given kind"""
    kind = kind or str(rs.choice(DATA, p=[.35, .1, .15, .08, .1, .07, .15]))
    c = shape[-1]
    if kind == "normal":
        x = rs.standard_normal(shape) * rs.uniform(0.1, 10) + rs.uniform(-3, 3)
    elif kind == "constant":  # constant columns: var 0, invstd rsqrt(eps)
        x = rs.standard_normal(shape)
        cols = rs.random_sample(c) < 0.6
        x[..., cols] = rs.standard_normal(int(cols.sum()))
    elif kind == "far_mean":  # |mean| 1e3 .. 1e4 against a small spread
        x = rs.uniform(1e3, 1e4, c) * rs.choice([-1, 1], c) + rs.standard_normal(shape) * rs.uniform(1e-2, 1)
    elif kind == "overflow":  # squares past float32's range: M2 becomes inf
        x = rs.standard_normal(shape) * (1e20 if fmt != "f16" else 6e4)
        if fmt != "f16":
            x[..., ::2] *= 1e17
    elif kind == "nonfinite":
        x = rs.standard_normal(shape)
        u = rs.random_sample(shape)
        x[u < 0.002] = np.nan
        x[(u >= 0.002) & (u < 0.004)] = np.inf
        x[(u >= 0.004) & (u < 0.006)] = -np.inf
    elif kind == "subnormal":
        x = rs.standard_normal(shape) * (1e-39 if fmt != "f16" else 1e-6)
    else:  # few distinct values: ties of the max within and across threads
        x = rs.randint(-2, 3, shape).astype(np.float64)
    x = x.astype(np.float32)
    return kind, NUM.quantize(x, fmt) if fmt != "f32" else x


def draw_affine(rs, c, fmt):
    kind = str(rs.choice(["none", "normal", "zero_gamma", "neg_gamma", "neg_zero_beta", "huge"],
                         p=[.25, .35, .1, .1, .1, .1]))
    if kind == "none":
        return kind, None, None
    gamma = rs.uniform(0.5, 2, c).astype(np.float32)
    beta = (rs.standard_normal(c) * 0.5).astype(np.float32)
    if kind == "zero_gamma":  # all-zero ReLU columns: every row ties
        gamma[rs.random_sample(c) < 0.7] = 0
        beta[:] = -np.abs(beta)
    elif kind == "neg_gamma":
        gamma = -gamma
    elif kind == "neg_zero_beta":
        beta[:] = -0.0
    elif kind == "huge":  # 16-bit outputs past 65504 (f16) and large bf16
        gamma *= np.float32(1e5 if fmt != "f32" else 1e30)
    return kind, gamma, beta


def draw_tracking(rs):
    kind = str(rs.choice(["momentum", "cma1", "cma_large", "none"], p=[.4, .2, .2, .2]))
    nbt = {"cma1": 0, "cma_large": int(rs.choice([12345, 2 ** 40 + 7]))}.get(kind, int(rs.randint(0, 50)))
    return kind, (-1.0 if kind.startswith("cma") else float(rs.choice([0.1, 0.01, 0.5, 1.0]))), nbt


def _common(rs, c, rows, fmt, keep_kind=None):
    dkind, x = draw_data(rs, (rows, c), fmt)
    akind, gamma, beta = draw_affine(rs, c, fmt)
    tkind, momentum, nbt = draw_tracking(rs)
    _, dy = draw_data(rs, (rows, c), fmt, "normal" if rs.rand() < 0.8 else "nonfinite")
    return dict(data=dkind, x=x, affine=akind, gamma=gamma, beta=beta, tracking=tkind, momentum=momentum, nbt=nbt,
                eps=float(rs.choice([1e-5, 1e-3, 0.1])), rm=(rs.standard_normal(c) * 3).astype(np.float32),
                rv=rs.uniform(0.1, 5, c).astype(np.float32), dy=dy, null_dgrads=bool(rs.rand() < 0.2))


def draw_misaligned(rs, g, names):
    """{name: element offset}: with vec 4, half the draws put one tensor alone one element off"""
    off = {k: 0 for k in names}
    if g["vec"] == 4 and rs.rand() < 0.5:
        off[str(rs.choice(names))] = 1
    return off


def draw_plain(rs):
    fmt = str(rs.choice(FMTS))
    c = int(rs.choice(WIDTHS))
    rkind, rows = draw_rows(rs, c)
    g = R.geom(rows, c)
    kkind, keep = draw_keep(rs, rows, g["chunk_rows"])
    p = dict(case="plain", fmt=fmt, c=c, rows=rows, rows_kind=rkind, keep_kind=kkind, keep=keep,
             off=draw_misaligned(rs, g, ["x", "y", "dy", "dx"]), pad_seed=int(rs.randint(1 << 30)))
    p.update(_common(rs, c, rows, fmt))
    return p


MAX_B = [1, 31, 32, 33, 70]


def draw_max(rs):
    fmt = str(rs.choice(FMTS))
    c = int(rs.choice(WIDTHS))
    g = R.geom(1, c)
    b = int(rs.choice(MAX_B)) if rs.rand() < 0.7 else int(rs.randint(2, 12))
    nkind = str(rs.choice(["lt_ty", "mid", "trips", "grid"], p=[.3, .3, .25, .15]))
    if nkind == "grid":  # b * n past one trip of the capped elementwise grid of the dx kernel
        per_trip = R.row_blocks(g, 1 << 30) * g["ty"] * R.UNROLL
        n = -(-per_trip // b) + int(rs.randint(1, 1 + per_trip // (2 * b) + 1))
    else:
        n = {"lt_ty": int(rs.randint(1, g["ty"])) if g["ty"] > 1 else 1, "mid": log_int(rs, g["ty"], 4 * g["ty"]),
             "trips": int(rs.randint(2 * R.UNROLL * g["ty"] + 1, 3 * R.UNROLL * g["ty"] + 2))}[nkind]
        if b * n * c > 3_000_000:  # keep a case small: the width decides n, the batch gives way
            b = max(1, 3_000_000 // (n * c))
    o = str(rs.choice(["none", "x", "dx"]))  # with vec 4: x or dx alone one element off
    lk = str(rs.choice(["full", "ragged", "empty_clouds"], p=[.3, .45, .25]))
    lengths = np.full(b, n) if lk == "full" else rs.randint(1, n + 1, b)
    if lk == "empty_clouds":
        lengths[rs.random_sample(b) < 0.4] = 0
    keep = (np.arange(n)[None, :] < lengths[:, None]).astype(np.uint8).reshape(-1)
    p = dict(case="max", fmt=fmt, b=b, n=n, c=c, n_kind=nkind, lengths_kind=lk, lengths=lengths, keep=keep,
             off={k: int(R.geom(b * n, c)["vec"] == 4 and k == o) for k in ("x", "dx")},
             pad_seed=int(rs.randint(1 << 30)))
    p.update(_common(rs, c, b * n, fmt))
    p["dout"] = draw_data(rs, (b, c), fmt, "normal")[1]
    return p


def tie_regimes(p):
    """ties of the max among a cloud's real rows, read off x where gamma > 0 (the ReLU output is then monotone in x):
    rows walked by one thread (equal j % ty), or by different threads.  Columns with gamma 0 and beta <= 0 are all
    zero after the ReLU, so all their real rows tie."""
    b, n, c = p["b"], p["n"], p["c"]
    ty = R.geom(b * n, c)["ty"]
    x = p["x"].reshape(b, n, c)
    keep = p["keep"].reshape(b, n) != 0
    gamma = p["gamma"] if p["gamma"] is not None else np.ones(c, np.float32)
    reg = set()
    for i in range(b):
        real = np.flatnonzero(keep[i])
        if len(real) < 2:
            continue
        xr = x[i, real]
        if np.isnan(xr).any():
            reg.add("max_nan_row")
        with np.errstate(invalid="ignore"):
            for k in range(c):
                if gamma[k] > 0:
                    col = xr[:, k]
                    if np.isnan(col).any():
                        continue
                    rows = real[col == col.max()]
                elif gamma[k] == 0 and p["beta"] is not None and p["beta"][k] <= 0 and np.isfinite(xr[:, k]).all():
                    rows = real
                else:
                    continue
                if len(rows) > 1:
                    th = rows % ty
                    if len(np.unique(th)) < len(th):
                        reg.add("max_tie_within_thread")
                    if len(np.unique(th)) > 1:
                        reg.add("max_tie_across_threads")
        if len(reg) >= 3:
            break
    return reg


REFUSALS = ["col_tiles", "ws_short", "ws_misaligned", "rm_without_rv", "cma_without_nbt", "bad_dtype", "null_x",
            "null_keep", "null_y", "null_save", "null_dx", "neg_rows", "max_rows_2_31", "max_n0", "max_null_argmax",
            "max_ws_short"]


def draw_refused(rs, k=0):
    """the k-th refusal of a seed takes REFUSALS[k % len(REFUSALS)]"""
    why = REFUSALS[k % len(REFUSALS)]
    return dict(case="refused", why=why, fmt=str(rs.choice(FMTS)), c=int(rs.choice([3, 8, 13])),
                backward=why == "null_dx" or bool(rs.rand() < 0.5) and why in ("ws_short", "ws_misaligned", "bad_dtype", "null_x",
                                                              "null_dx", "neg_rows", "col_tiles", "max_rows_2_31",
                                                              "max_ws_short"))


def draw_torch(rs):
    fmt = str(rs.choice(FMTS))
    form = str(rs.choice(["plain", "max"]))
    c = int(rs.choice([3, 8, 13, 64, 132]))
    momentum = None if rs.rand() < 0.3 else float(rs.choice([0.1, 0.5]))
    p = dict(case="torch", fmt=fmt, form=form, c=c, affine=bool(rs.rand() < 0.7), momentum=momentum,
             track=bool(rs.rand() < 0.8), nbt=int(rs.randint(0, 5)), eps=1e-5, functional=bool(rs.rand() < 0.5))
    if form == "plain":
        rows = log_int(rs, 1, 5000)
        keep = (rs.random_sample(rows) < 0.7).astype(np.uint8)
        keep[int(rs.randint(rows))] = 1
        p.update(rows=rows, keep=keep)
    else:
        b, n = int(rs.choice([1, 5, 33])), log_int(rs, 1, 300)
        lengths = rs.randint(0, n + 1, b)  # the layer clamps them to >= 1
        keep = (np.arange(n)[None, :] < np.clip(lengths, 1, n)[:, None]).astype(np.uint8).reshape(-1)
        p.update(b=b, n=n, rows=b * n, lengths=lengths, keep=keep)
    p["x"] = draw_data(rs, (p["rows"], c), fmt, "normal")[1]
    p["dy"] = draw_data(rs, (p["b"], c) if form == "max" else (p["rows"], c), fmt, "normal")[1]
    p["gamma"] = rs.uniform(0.5, 2, c).astype(np.float32)
    p["beta"] = rs.standard_normal(c).astype(np.float32)
    p["rm"] = rs.standard_normal(c).astype(np.float32)
    p["rv"] = rs.uniform(0.5, 2, c).astype(np.float32)
    return p


# --------------------------------------------------------------------------------------------------- helpers
def padded(p, a, rows_keep, mode):
    """a (rows, c) with its padding rows replaced: "poison" (NaN, ±inf, far values) or "copy" (real rows)"""
    a = np.array(a, np.float32, copy=True)
    pad = np.flatnonzero(rows_keep == 0)
    if not len(pad):
        return a
    rs = np.random.RandomState(p["pad_seed"] if "pad_seed" in p else 0)
    if mode == "poison":
        pool = np.array([np.nan, np.inf, -np.inf, 3e38, -3e38, 6e4], np.float32)
        a[pad] = pool[rs.randint(0, len(pool), (len(pad), a.shape[1]))]
    else:
        real = np.flatnonzero(rows_keep != 0)
        a[pad] = a[real[rs.randint(0, len(real), len(pad))]] if len(real) else rs.standard_normal((len(pad), a.shape[1]))
    return a


def to_dev(vals, off, fmt):
    """a device tensor of fmt holding vals from element off on, with a poisoned guard after"""
    return G.dev_buf(G.to_fmt_bits(np.asarray(vals, np.float32), fmt), off, fmt)


def F32(a):
    return G.F32(a) if a is not None else None


def f32_out(n):
    return G.out_buf(n, 0, "f32")


def bits(t, fmt):
    """the raw bits of a device tensor, flattened"""
    return G.host_bits(t, fmt).reshape(-1)


def same(got_bits, want_f32, fmt):
    return G.same_or_nan(got_bits, want_f32, fmt)


def invstd_ok(got, var_eps):
    """save_invstd within 2 ulp of 1 / sqrt(var + eps) (float64 of the float32 sum); NaN where that is NaN"""
    with np.errstate(all="ignore"):
        want = 1.0 / np.sqrt(var_eps.astype(np.float64))
    nan = np.isnan(want)
    if not np.array_equal(np.isnan(got), nan):
        return False
    g, w = got[~nan].astype(np.float64), want[~nan]
    return bool(np.all(np.abs(g - w) <= 2 * NUM.ulp(w, "f32")))


def lib():
    return _lib.load()


def _workspace(nbytes, misaligned=False):
    ws = torch.full((nbytes + 16,), 0x5A, dtype=torch.uint8, device=dev)
    G._LIVE.append(ws)
    return G.elem_ptr(ws, 8 if misaligned else 0)


def _stats_bufs(p):
    track = p["tracking"] != "none"
    rm = F32(p["rm"]) if track else None
    rv = F32(p["rv"]) if track else None
    nbt = None
    if track:
        nbt = torch.tensor([p["nbt"] + 1], dtype=torch.int64, device=dev)  # incremented, as the callers do
        G._LIVE.append(nbt)
    return rm, rv, nbt


def _want_stats(p, keep):
    track = p["tracking"] != "none"
    return O.oracle_mbn_stats(p["x"], keep, p["eps"], p["momentum"], p["nbt"] + 1, p["rm"] if track else None,
                              p["rv"] if track else None)


def abi_forward(p, mode):
    """pn2_masked_bn_relu_forward_typed: host results of one run"""
    fmt, rows, c, off = p["fmt"], p["rows"], p["c"], p["off"]
    x = to_dev(padded(p, p["x"], p["keep"], mode), off["x"], fmt)
    y = G.out_buf(rows * c, off["y"], fmt)
    sm, si = f32_out(c), f32_out(c)
    rm, rv, nbt = _stats_bufs(p)
    keep = torch.from_numpy(p["keep"]).to(dev)
    G._LIVE.append(keep)
    wsb = int(lib().pn2_masked_bn_workspace_bytes(rows, c))
    rc = lib().pn2_masked_bn_relu_forward_typed(
        CODE[fmt], rows, c, G.elem_ptr(x, off["x"]), ptr(keep), ptr(F32(p["gamma"])), ptr(F32(p["beta"])), p["eps"],
        p["momentum"], ptr(nbt), ptr(rm), ptr(rv), G.elem_ptr(y, off["y"]), ptr(sm), ptr(si), _workspace(wsb), wsb,
        stream_ptr(dev))
    return dict(rc=rc, wsb=wsb, x=x, y=y, y_bits=bits(y, fmt), sm=bits(sm, "f32"), si=bits(si, "f32"), keep=keep,
                rm=None if rm is None else bits(rm, "f32"), rv=None if rv is None else bits(rv, "f32"))


def abi_backward(p, fw, mode):
    fmt, rows, c, off = p["fmt"], p["rows"], p["c"], p["off"]
    dy = to_dev(padded(p, p["dy"], p["keep"], mode), off["dy"], fmt)
    dx = G.out_buf(rows * c, off["dx"], fmt)
    affine = p["gamma"] is not None and not p["null_dgrads"]
    dg, db = (f32_out(c), f32_out(c)) if affine else (None, None)
    sm = F32(fw["sm"].view(np.float32)[:c])
    si = F32(fw["si"].view(np.float32)[:c])
    wsb = fw["wsb"]
    y = fw["y"]
    rc = lib().pn2_masked_bn_relu_backward_typed(
        CODE[fmt], rows, c, G.elem_ptr(dy, off["dy"]), G.elem_ptr(fw["x"], off["x"]), G.elem_ptr(y, off["y"]),
        ptr(fw["keep"]), ptr(F32(p["gamma"])), ptr(sm), ptr(si), G.elem_ptr(dx, off["dx"]), ptr(dg), ptr(db),
        _workspace(wsb), wsb, stream_ptr(dev))
    return dict(rc=rc, dx_bits=bits(dx, fmt), dg=None if dg is None else bits(dg, "f32"),
                db=None if db is None else bits(db, "f32"))


def check_forward(p, fw, off_y, rows, c):
    """(ok, y values, mean, invstd) of a plain forward against the oracle"""
    fmt, keep = p["fmt"], p["keep"]
    if fw["rc"] != 0 or fw["wsb"] != R.workspace_bytes(rows, c):
        return False, None, None, None
    sm, si = fw["sm"][:c].view(np.float32), fw["si"][:c].view(np.float32)
    ok = np.array_equal(fw["sm"][c:], np.full(G.GUARD, POISON["f32"])) and np.array_equal(
        fw["si"][c:], np.full(G.GUARD, POISON["f32"]))
    mean, var_eps, _, rm, rv = _want_stats(p, keep)
    ok = ok and same(sm.view(np.uint32), mean, "f32") and invstd_ok(si, var_eps)
    if rm is not None:
        ok = ok and same(fw["rm"][:c], rm, "f32") and same(fw["rv"][:c], rv, "f32")
    body, clean = G.guarded(fw["y_bits"], off_y, rows * c, fmt)
    want = O.oracle_mbn_norm_relu(p["x"], keep, sm, si, p["gamma"], p["beta"])
    ok = ok and clean and same(body.reshape(rows, c), want, fmt)
    ok = ok and bool(np.all(body.reshape(rows, c)[keep == 0] == 0))
    return bool(ok), G.values(body, fmt).reshape(rows, c), sm, si


# ----------------------------------------------------------------------------------------------------- plain
def run_plain(p):
    fmt, rows, c, off, keep = p["fmt"], p["rows"], p["c"], p["off"], p["keep"]
    runs = []
    ok = True
    for mode in ("poison", "copy"):
        G._LIVE.clear()
        fw = abi_forward(p, mode)
        bw = abi_backward(p, fw, mode)
        runs.append((fw, bw))
        if mode == "copy":
            break
        okf, yv, sm, si = check_forward(p, fw, off["y"], rows, c)
        if not okf or bw["rc"] != 0:
            return False
        dx, dg, db = O.oracle_mbn_backward(p["dy"], p["x"], yv, keep, sm, si, p["gamma"])
        body, clean = G.guarded(bw["dx_bits"], off["dx"], rows * c, fmt)
        ok = clean and same(body.reshape(rows, c), dx, fmt) and bool(np.all(body.reshape(rows, c)[keep == 0] == 0))
        if bw["dg"] is not None:
            ok = ok and same(bw["dg"][:c], dg, "f32") and same(bw["db"][:c], db, "f32")
            ok = ok and bool(np.all(bw["dg"][c:] == POISON["f32"]) and np.all(bw["db"][c:] == POISON["f32"]))
        if not ok:
            return False
    (f1, b1), (f2, b2) = runs
    for k in ("y_bits", "sm", "si", "rm", "rv"):
        if f1[k] is not None and not np.array_equal(f1[k], f2[k]):
            return False
    for k in ("dx_bits", "dg", "db"):
        if b1[k] is not None and not np.array_equal(b1[k], b2[k]):
            return False
    return bool(f2["rc"] == 0 and b2["rc"] == 0)


# ------------------------------------------------------------------------------------------------------- max
def abi_max(p, mode):
    fmt, b, n, c, off = p["fmt"], p["b"], p["n"], p["c"], p["off"]
    rows = b * n
    x = to_dev(padded(p, p["x"], p["keep"], mode), off["x"], fmt)
    out = G.out_buf(b * c, 0, fmt)
    am = torch.full((b * c + G.GUARD,), -7, dtype=torch.int32, device=dev)
    sm, si = f32_out(c), f32_out(c)
    rm, rv, nbt = _stats_bufs(p)
    keep = torch.from_numpy(p["keep"]).to(dev)
    G._LIVE += [am, keep]
    wsb = int(lib().pn2_masked_bn_relu_max_workspace_bytes(b, n, c))
    rc = lib().pn2_masked_bn_relu_max_forward_typed(
        CODE[fmt], b, n, c, G.elem_ptr(x, off["x"]), ptr(keep), ptr(F32(p["gamma"])), ptr(F32(p["beta"])), p["eps"],
        p["momentum"], ptr(nbt), ptr(rm), ptr(rv), ptr(out), ptr(am), ptr(sm), ptr(si), _workspace(wsb), wsb,
        stream_ptr(dev))
    dout = to_dev(p["dout"], 0, fmt)
    dx = G.out_buf(rows * c, off["dx"], fmt)
    affine = p["gamma"] is not None and not p["null_dgrads"]
    dg, db = (f32_out(c), f32_out(c)) if affine else (None, None)
    rc2 = lib().pn2_masked_bn_relu_max_backward_typed(
        CODE[fmt], b, n, c, ptr(dout), G.elem_ptr(x, off["x"]), ptr(out), ptr(am), ptr(keep), ptr(F32(p["gamma"])),
        ptr(sm), ptr(si), G.elem_ptr(dx, off["dx"]), ptr(dg), ptr(db), _workspace(wsb), wsb, stream_ptr(dev))
    return dict(rc=rc, rc2=rc2, wsb=wsb, out=bits(out, fmt), am=am.cpu().numpy(), sm=bits(sm, "f32"),
                si=bits(si, "f32"), rm=None if rm is None else bits(rm, "f32"),
                rv=None if rv is None else bits(rv, "f32"), dx=bits(dx, fmt), dg=None if dg is None else bits(dg, "f32"),
                db=None if db is None else bits(db, "f32"))


def run_max(p):
    fmt, b, n, c, keep = p["fmt"], p["b"], p["n"], p["c"], p["keep"]
    rows = b * n
    G._LIVE.clear()
    r1 = abi_max(p, "poison")
    if r1["rc"] != 0 or r1["rc2"] != 0 or r1["wsb"] != R.max_workspace_bytes(b, n, c):
        return False
    sm, si = r1["sm"][:c].view(np.float32), r1["si"][:c].view(np.float32)
    mean, var_eps, _, rm, rv = _want_stats(p, keep)
    ok = same(sm.view(np.uint32), mean, "f32") and invstd_ok(si, var_eps)
    if rm is not None:
        ok = ok and same(r1["rm"][:c], rm, "f32") and same(r1["rv"][:c], rv, "f32")
    y = G.values(G.to_fmt_bits(O.oracle_mbn_norm_relu(p["x"], keep, sm, si, p["gamma"], p["beta"]), fmt), fmt)
    wout, warg = O.oracle_mbn_max_pool(y.reshape(b, n, c), keep)
    body, clean = G.guarded(r1["out"], 0, b * c, fmt)
    ok = ok and clean and same(body.reshape(b, c), wout, fmt)
    ok = ok and np.array_equal(r1["am"][:b * c].reshape(b, c), warg) and bool(np.all(r1["am"][b * c:] == -7))
    outv = G.values(body, fmt).reshape(b, c)
    dx, dg, db = O.oracle_mbn_max_backward(p["dout"], p["x"].reshape(b, n, c), outv, warg, keep, sm, si, p["gamma"])
    dbody, dclean = G.guarded(r1["dx"], p["off"]["dx"], rows * c, fmt)
    ok = ok and dclean and same(dbody.reshape(b, n, c), dx, fmt) and bool(np.all(dbody.reshape(rows, c)[keep == 0] == 0))
    if r1["dg"] is not None:
        ok = ok and same(r1["dg"][:c], dg, "f32") and same(r1["db"][:c], db, "f32")
    if not ok:
        return False
    # the plain entry's statistics on the same rows, bit for bit
    q = dict(p, rows=rows, off=dict(x=p["off"]["x"], y=0, dy=0, dx=0))
    G._LIVE.clear()
    fw = abi_forward(q, "poison")
    for k in ("sm", "si", "rm", "rv"):
        if r1[k] is not None and not np.array_equal(r1[k], fw[k]):
            return False
    G._LIVE.clear()
    r2 = abi_max(p, "copy")
    return all(r1[k] is None or np.array_equal(r1[k], r2[k]) for k in r1)


# --------------------------------------------------------------------------------------------------- refused
def run_refused(p):
    L = lib()
    fmt, c, why, bw = p["fmt"], p["c"], p["why"], p["backward"]
    code = 9 if why == "bad_dtype" else CODE[fmt]
    mx = why.startswith("max_")
    b, n = (65536, 32768) if why == "max_rows_2_31" else (2, 0 if why == "max_n0" else 5)
    rows = -1 if why == "neg_rows" else 10
    if why == "col_tiles":
        c = 32 * 65535 + 1  # vec 1: 65536 column tiles of 32 lanes
    small = 10 * c
    x = to_dev(np.zeros(small, np.float32), 0, fmt)
    keep = torch.ones(small, dtype=torch.uint8, device=dev)
    y = G.out_buf(small, 0, fmt)
    out = G.out_buf(2 * c, 0, fmt)
    am = torch.full((2 * c,), -7, dtype=torch.int32, device=dev)
    sm, si = f32_out(c), f32_out(c)
    rm, rv = F32(np.zeros(c)), F32(np.ones(c))
    nbt = torch.ones(1, dtype=torch.int64, device=dev)
    G._LIVE.extend([keep, am, nbt])
    if mx:
        wsb = int(L.pn2_masked_bn_relu_max_workspace_bytes(2, 5, c))
    else:
        wsb = int(L.pn2_masked_bn_workspace_bytes(max(rows, 1), c))
    ws = _workspace(wsb + 64, misaligned=why == "ws_misaligned")
    wsn = wsb - 1 if why.endswith("ws_short") else wsb
    P = lambda t: ptr(t)  # noqa: E731
    nul = lambda name, t: None if why == name else t  # noqa: E731
    torch.cuda.synchronize(dev)
    before = _lib.launch_count()
    mom = -1.0 if why == "cma_without_nbt" else 0.1
    if mx:
        if bw:
            rc = L.pn2_masked_bn_relu_max_backward_typed(code, b, n, c, P(out), P(x), P(out), P(am), P(keep), None, P(sm),
                                                        P(si), P(y), None, None, ws, wsn, stream_ptr(dev))
        else:
            rc = L.pn2_masked_bn_relu_max_forward_typed(code, b, n, c, P(x), P(keep), None, None, 1e-5, mom, None, P(rm),
                                                       P(rv), P(out), nul("max_null_argmax", P(am)), P(sm), P(si), ws,
                                                       wsn, stream_ptr(dev))
    elif bw:
        rc = L.pn2_masked_bn_relu_backward_typed(code, rows, c, P(y), nul("null_x", P(x)), P(y), P(keep), None, P(sm),
                                                 P(si), nul("null_dx", P(out)), None, None, ws, wsn, stream_ptr(dev))
    else:
        rc = L.pn2_masked_bn_relu_forward_typed(
            code, rows, c, nul("null_x", P(x)), nul("null_keep", P(keep)), None, None, 1e-5, mom,
            None if why == "cma_without_nbt" else P(nbt), P(rm), None if why == "rm_without_rv" else P(rv),
            nul("null_y", P(y)), nul("null_save", P(sm)), P(si), ws, wsn, stream_ptr(dev))
    launched = _lib.launch_count() - before
    torch.cuda.synchronize(dev)
    untouched = all(np.all(bits(t, f) == POISON[f]) for t, f in ((y, fmt), (out, fmt), (sm, "f32"), (si, "f32")))
    untouched = untouched and bool((am == -7).all().item())
    return rc == CUDA_ERROR_INVALID_VALUE and launched == 0 and untouched


# ----------------------------------------------------------------------------------------------------- torch
def run_torch(p):
    from pointnet2_b200 import layers
    fmt, c, rows = p["fmt"], p["c"], p["rows"]
    dt = G.TORCH[fmt]
    bn = torch.nn.BatchNorm1d(c, eps=p["eps"], momentum=p["momentum"], affine=p["affine"],
                              track_running_stats=p["track"]).to(dev).train()
    with torch.no_grad():
        if p["affine"]:
            bn.weight.copy_(torch.from_numpy(p["gamma"]))
            bn.bias.copy_(torch.from_numpy(p["beta"]))
        if p["track"]:
            bn.running_mean.copy_(torch.from_numpy(p["rm"]))
            bn.running_var.copy_(torch.from_numpy(p["rv"]))
            bn.num_batches_tracked.fill_(p["nbt"])
    x = torch.from_numpy(p["x"]).to(dev).to(dt).requires_grad_(True)
    dy = torch.from_numpy(p["dy"]).to(dev).to(dt)
    keep = torch.from_numpy(p["keep"]).to(dev).bool()
    w, bias = (bn.weight, bn.bias) if p["affine"] else (None, None)
    eps, mom, nbt, rm, rv = layers._bn_state(bn)
    if p["form"] == "plain":
        if p["functional"]:
            y, _, _, *st = torch.ops.pn2.masked_batch_norm_relu(x, w, bias, keep.view(torch.uint8), rm, rv, nbt, eps, mom)
            layers._write_back(st, nbt, rm, rv)
        else:
            y = layers.masked_batch_norm_relu(bn, x, keep)
        y.backward(dy)
        q = dict(case="plain", fmt=fmt, rows=rows, c=c, keep=p["keep"], off=dict(x=0, y=0, dy=0, dx=0), x=p["x"],
                 dy=p["dy"])
    else:
        b, n = p["b"], p["n"]
        if p["functional"]:
            out, am, _, _, *st = torch.ops.pn2.masked_bn_relu_max(x.view(b, n, c), w, bias, keep.view(torch.uint8), rm,
                                                                   rv, nbt, eps, mom)
            layers._write_back(st, nbt, rm, rv)
        else:
            out, am = layers.masked_bn_relu_max(bn, x.view(b, n, c), torch.from_numpy(p["lengths"]).to(dev),
                                                with_indices=True)
        out.backward(dy)
        y = out
        q = dict(case="max", fmt=fmt, b=b, n=n, c=c, keep=p["keep"], off=dict(x=0, dx=0), x=p["x"], dout=p["dy"])
    q.update(gamma=p["gamma"] if p["affine"] else None, beta=p["beta"] if p["affine"] else None, eps=p["eps"],
             momentum=-1.0 if p["momentum"] is None else p["momentum"], nbt=p["nbt"], rm=p["rm"], rv=p["rv"],
             tracking="momentum" if p["track"] else "none", null_dgrads=False)
    G._LIVE.clear()
    if p["form"] == "plain":
        fw = abi_forward(q, "poison")
        bw = abi_backward(q, fw, "poison")
        ok = np.array_equal(bits(y, fmt), fw["y_bits"][:rows * c]) and np.array_equal(bits(x.grad, fmt),
                                                                                     bw["dx_bits"][:rows * c])
        ref = dict(rm=fw["rm"], rv=fw["rv"], dg=bw["dg"], db=bw["db"])
    else:
        r = abi_max(q, "poison")
        ok = np.array_equal(bits(y, fmt), r["out"][:p["b"] * c]) and np.array_equal(am.cpu().numpy().reshape(-1),
                                                                                    r["am"][:p["b"] * c])
        ok = ok and np.array_equal(bits(x.grad, fmt), r["dx"][:rows * c])
        ref = r
    ok = ok and r_ok(ref, bn, p, c)
    return bool(ok)


def r_ok(ref, bn, p, c):
    ok = True
    if p["affine"]:
        ok = np.array_equal(bits(bn.weight.grad, "f32"), ref["dg"][:c]) and np.array_equal(bits(bn.bias.grad, "f32"),
                                                                                          ref["db"][:c])
    if p["track"]:
        ok = ok and np.array_equal(bits(bn.running_mean, "f32"), ref["rm"][:c])
        ok = ok and np.array_equal(bits(bn.running_var, "f32"), ref["rv"][:c])
        ok = ok and int(bn.num_batches_tracked.item()) == p["nbt"] + 1
    return bool(ok)


CASES = ["plain", "max", "refused", "torch"]
DRAW = {name: globals()["draw_" + name] for name in CASES}
RUN = {name: globals()["run_" + name] for name in CASES}


def draws(seed: int, iterations: int):
    """The parameters ``run(seed, iterations)`` uses, without a device (the run_* functions draw nothing)."""
    rs = np.random.RandomState(seed)
    return [_draw(rs, it) for it in range(iterations)]


def _draw(rs, it):
    name = SCHEDULE[it % len(SCHEDULE)]
    if name == "refused":
        return draw_refused(rs, sum(1 for i in range(it) if SCHEDULE[i % len(SCHEDULE)] == "refused"))
    return DRAW[name](rs)


def public(p):
    """the parameters of a case without its input arrays (they follow from the seed and the iteration)"""
    return {k: v for k, v in p.items() if not isinstance(v, np.ndarray)}


def _one(rs, seed, it, counts, fails, catch):
    name = SCHEDULE[it % len(SCHEDULE)]
    p = _draw(rs, it)
    G._LIVE.clear()
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
    return name, ok


def run(seed: int, iterations: int):
    """``iterations`` random cases in SCHEDULE order; returns (counts, failures)."""
    rs = np.random.RandomState(seed)
    counts, fails = {}, []
    for it in range(iterations):
        _one(rs, seed, it, counts, fails, catch=True)
    return counts, fails


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=float, default=120)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--iterations", type=int, default=None, help="stop after this many cases")
    ap.add_argument("--json", type=str, default=None)
    args = ap.parse_args()
    rs = np.random.RandomState(args.seed)
    counts, fails, secs = {}, [], {}
    t0 = time.time()
    it = 0
    while time.time() - t0 < args.seconds and (args.iterations is None or it < args.iterations):
        t1 = time.time()
        name, ok = _one(rs, args.seed, it, counts, fails, catch=True)
        secs[name] = secs.get(name, 0.0) + time.time() - t1
        if not ok:
            print("FAIL", json.dumps(fails[-1], default=str), flush=True)
        it += 1
    summary = dict(seed=args.seed, seconds=round(time.time() - t0, 1), cases=counts,
                   case_seconds={k: round(v, 1) for k, v in secs.items()}, failures=fails)
    print(json.dumps(summary, default=str))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(summary, f, indent=1, default=str)
    sys.exit(1 if fails else 0)


if __name__ == "__main__":
    main()
