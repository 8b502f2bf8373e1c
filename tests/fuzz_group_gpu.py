#!/usr/bin/env python
"""Randomised differential test of the grouping, interpolation and ordered-scatter kernels (group.cu,
interpolate.cu, scatter_det.cu) against the C oracle and tests/group_regimes.py (TEST TOOL, runs on a GPU box).

    python tests/fuzz_group_gpu.py [--seconds 120] [--seed 0] [--json out.json]

Each case is ``draw_<case>(rs)`` (parameters and inputs with numpy alone, no device) and ``run_<case>(p)``.  All but
``autograd`` call the C ABI with explicit pointers, so the buffer alignment, the workspace size and the dtype code
are exactly what was drawn.  Every output buffer is filled with a poison pattern before the call and has a guard
after its end; every element and the guard are compared, so a row that is never written (or one written past the
end) fails.

- ``group_point``: pn2_group_point_typed; copies are compared bit for bit with a numpy gather of the raw bits.
- ``group_concat``: pn2_group_concat_typed; features bit for bit, centred xyz bit for bit except that NaN equals
  NaN (the device's __fsub_rn returns the canonical NaN, numpy keeps the payload).
- ``ordered_grad``: pn2_three_interpolate_grad_det_ragged_typed (weighted) or pn2_group_point_grad_det_typed
  (unweighted) with target lists of exact lengths; the result must equal ``group_regimes.ordered_sum`` (NaN equals
  NaN), and a second call must give identical bits.
- ``atomic_grad``: group_point_grad (typed, vec4 or scalar, with the rounding pass), three_interpolate_grad and
  gather_point_grad.  Half the draws are exact-sum inputs (small integers times powers of two, on a normal or a
  subnormal grid, with NaN, ±inf and −0.0 mixed in: every partial sum is exact and NaN / inf absorb, so any atomic
  order gives the oracle's bits, on inputs whose subnormals are flushed as float atomics flush them, see ``ftz``);
  the rest are finite and held to ``numerics.within_bound``.
- ``interp``: pn2_three_interpolate_ragged_typed, vec4 or scalar, against oracle_three_interpolate.
- ``selection_sort``: pn2_selection_sort against oracle_selection_sort, the full (b, m, n) outputs, with NaN at the
  round's position and elsewhere, ±inf and ±0 ties.
- ``refused``: b > 65535 on the row paths, a workspace one byte short, a bad dtype code, null pointers: the call
  returns cudaErrorInvalidValue, launches nothing and leaves the poisoned output as it was.
- ``autograd``: group_and_concat and its gradient through torch and autograd.
- ``fp_front``: pn2_three_nn_interpolate_ragged_typed and pn2_fp_interpolate_concat_ragged_typed; each seed's k-th
  case takes one of the 24 (G, T, lengths) instantiations of fp_front_kernel in turn.  dist / idx must equal
  oracle_three_nn on the truncated clouds, the weights the float32 formula of ``fp_weights`` and the interpolated
  part oracle_three_interpolate with those weights, rounded once; padding rows hold the filler.

The data holds NaN (with payloads), ±inf, −0.0, subnormals and values past the 16-bit formats' range.
tests/test_fuzz_group_cpu.py replays the fixed slice through group_regimes and requires every instantiation and
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
import group_regimes as R  # noqa: E402
import numerics as NUM  # noqa: E402
from oracle import oracle as O  # noqa: E402
from pointnet2_b200 import _lib  # noqa: E402
from pointnet2_b200._tensor import ptr, stream_ptr  # noqa: E402

dev = torch.device("cuda:0")  # only dereferenced when a case runs

# the slice tests/test_fuzz_group_gpu.py runs, and tests/test_fuzz_group_cpu.py checks the coverage of
SLICE_SEEDS = (91, 92)
SCHEDULE = ["group_point", "ordered_grad", "group_concat", "selection_sort", "ordered_grad", "atomic_grad",
            "group_point", "interp", "ordered_grad", "group_concat", "refused", "atomic_grad", "interp", "autograd",
            "fp_front"]
SLICE_ITERATIONS = 32 * len(SCHEDULE)

FMTS = ["f32", "bf16", "f16"]
DTYPE_CODE = {"f32": 0, "bf16": 1, "f16": 2}
TORCH = {"f32": torch.float32, "bf16": torch.bfloat16, "f16": torch.float16}
RAW = {"f32": np.uint32, "bf16": np.uint16, "f16": np.uint16}
POISON = {"f32": np.uint32(0x7FA5A5A5), "bf16": np.uint16(0x7FA5), "f16": np.uint16(0x7DA5)}  # NaNs no kernel makes
GUARD = 8
CUDA_ERROR_INVALID_VALUE = 1
# exact list lengths: both sides of every bitonic bucket, of the sort cap, of the long-seq buffer and beyond 4096
LIST_LENGTHS = [0, 1, 32, 33, 64, 65, 128, 129, 256, 257, 2048, 2049, 4500, 9000]
TARGETS = [1023, 1024, 1025, 16000, 16001]


# ------------------------------------------------------------------------------------------------------ helpers
def log_int(rs, lo, hi):
    return int(np.clip(np.exp(rs.uniform(np.log(lo), np.log(hi + 1))), lo, hi))


def special_f32(rs, shape, scale=1.0):
    """float32 values with NaN (payloads), ±inf, −0, subnormals and magnitudes past the 16-bit ranges"""
    x = (rs.standard_normal(shape) * scale).astype(np.float32)
    u = rs.random_sample(shape)
    pool = np.array([np.nan, np.inf, -np.inf, -0.0, 0.0, 1e-40, -3e-42, 7e4, -1e5, 3e38, 2.0 ** -130, 6e-8],
                    np.float32)
    x = np.where(u < 0.08, pool[rs.randint(0, len(pool), shape)], x).astype(np.float32)
    pay = (u > 0.995)
    xb = x.view(np.uint32)
    xb[pay] = (0x7F800001 + rs.randint(0, 1 << 22, int(pay.sum()))).astype(np.uint32) | np.uint32(0x400000)
    return x


def raw_bits(rs, shape, fmt):
    """random raw bit patterns of a format (every class of value, NaN payloads included)"""
    if fmt == "f32":
        b = rs.randint(0, 1 << 32, shape, dtype=np.uint64).astype(np.uint32)
        sp = rs.random_sample(shape) < 0.5
        b[sp] = special_f32(rs, shape).view(np.uint32)[sp]
        return b
    return rs.randint(0, 1 << 16, shape).astype(np.uint16)


def to_fmt_bits(x, fmt):
    return NUM.round_once(x, fmt).view(RAW[fmt]) if fmt != "f32" else np.ascontiguousarray(x, np.float32).view(np.uint32)


def dev_buf(bits, offset, fmt):
    """a device tensor (of the format's torch dtype) holding ``bits`` from element ``offset`` on, poisoned guard after"""
    bits = np.ascontiguousarray(bits).reshape(-1)
    tot = np.full(offset + bits.size + GUARD, POISON[fmt], RAW[fmt])
    tot[offset:offset + bits.size] = bits
    t = torch.from_numpy(tot.view(np.int32 if fmt == "f32" else np.int16)).to(dev)
    return t.view(TORCH[fmt])


def out_buf(numel, offset, fmt):
    return dev_buf(np.full(numel, POISON[fmt], RAW[fmt]), offset, fmt)


def host_bits(t, fmt):
    a = t.detach().cpu()
    a = a.view(torch.int32) if fmt == "f32" else a.view(torch.int16)
    return a.numpy().view(RAW[fmt])


def elem_ptr(t, offset):
    return ctypes_ptr(t.data_ptr() + offset * t.element_size())


def ctypes_ptr(v):
    import ctypes
    return ctypes.c_void_p(v)


# The device inputs of the running case.  A tensor whose pointer goes to the C ABI must outlive the launch: were it
# freed when ptr() returns, the caching allocator could hand its block to the next input, whose copy is ordered
# before the kernel on the same stream.  _one clears the list when the next case starts.
_LIVE = []


def I32(a):
    t = torch.from_numpy(np.ascontiguousarray(a, np.int32)).to(dev)
    _LIVE.append(t)
    return t


def F32(a):
    t = torch.from_numpy(np.ascontiguousarray(a, np.float32)).to(dev)
    _LIVE.append(t)
    return t


def values(bits, fmt):
    return NUM.decode(bits, fmt) if fmt != "f32" else np.ascontiguousarray(bits).view(np.float32)


def same_or_nan(got_bits, want_f32, fmt):
    """got (raw bits of fmt) against float32 values rounded once to fmt: equal bits, or both NaN"""
    want = to_fmt_bits(want_f32, fmt)
    g, w = values(got_bits, fmt), values(want, fmt)
    return bool(np.all((got_bits == want) | (np.isnan(g) & np.isnan(w))))


def guarded(got, offset, numel, fmt):
    """(body, guard and leading pad untouched?)"""
    body = got[offset:offset + numel]
    rest = np.concatenate([got[:offset], got[offset + numel:]])
    return body, bool(np.all(rest == POISON[fmt]))


def lib():
    return _lib.load()


# --------------------------------------------------------------------------------------------------- group_point
def draw_group_point(rs):
    fmt = str(rs.choice(FMTS))
    e = R.ESIZE[fmt]
    kind = str(rs.choice(["vec4", "rows", "narrow", "misaligned", "flat_b", "cap"], p=[.3, .2, .15, .1, .1, .15]))
    per16 = 16 // e
    if kind == "vec4":  # every LPR: c4 in 1..4 / 5..8 / 9..16 / 17..40
        c4 = int(rs.choice([rs.randint(1, 5), rs.randint(5, 9), rs.randint(9, 17), rs.randint(17, 41)]))
        c = c4 * per16
    elif kind == "misaligned":
        c = per16 * int(rs.randint(1, 20))
    elif kind == "narrow":
        c = int(rs.randint(1, 5))
    else:
        c = int(rs.choice([3, 5, 7, 9, 11, 13, 14, 17, 29, 33, 70, 131, 259]))
        if c * e % 16 == 0:
            c += 1
    if kind == "flat_b":
        b, n, m, s = 65536, int(rs.randint(1, 3)), 1, 1
        c = per16 * int(rs.randint(1, 3))
    elif kind == "cap":  # past the grid cap: more rows per cloud than the capped grid covers in one trip
        b = int(rs.choice([2112, 4300, 9000]))
        n, m, s = int(rs.randint(1, 4)), int(rs.randint(17, 40)), int(rs.choice([16, 32]))
        c = int(rs.choice([per16, 2 * per16, 3, 5, 9, 17, 40]))
    else:
        b, n = int(rs.randint(1, 5)), log_int(rs, 1, 3000)
        m, s = log_int(rs, 1, 400), int(rs.choice([1, 3, 8, 16, 32, 64]))
        if kind == "vec4" and rs.rand() < 0.5:  # a last batch of 1, 2 or 3 rows (R = 4)
            m, s = 4 * int(rs.randint(0, 100)) + int(rs.randint(1, 4)), 1
    off = (1, 0) if kind == "misaligned" and rs.rand() < 0.5 else (0, 1) if kind == "misaligned" else (0, 0)
    idx = rs.randint(0, n, (b, m, s)).astype(np.int32)
    return dict(case="group_point", kind=kind, fmt=fmt, b=b, n=n, c=c, m=m, s=s, points_off=off[0], out_off=off[1],
                pts=raw_bits(rs, (b, n, c), fmt), idx=idx)


def run_group_point(p):
    fmt, b, n, c, m, s = p["fmt"], p["b"], p["n"], p["c"], p["m"], p["s"]
    pts = dev_buf(p["pts"], p["points_off"], fmt)
    numel = b * m * s * c
    out = out_buf(numel, p["out_off"], fmt)
    rc = lib().pn2_group_point_typed(DTYPE_CODE[fmt], b, n, c, m, s, elem_ptr(pts, p["points_off"]), ptr(I32(p["idx"])),
                                     elem_ptr(out, p["out_off"]), stream_ptr(dev))
    got = host_bits(out, fmt)
    body, clean = guarded(got, p["out_off"], numel, fmt)
    want = p["pts"][np.arange(b)[:, None, None], p["idx"]]
    return rc == 0 and clean and np.array_equal(body, want.reshape(-1))


# -------------------------------------------------------------------------------------------------- group_concat
def draw_group_concat(rs):
    fmt = "f32" if rs.rand() < 0.5 else str(rs.choice(["bf16", "f16"]))
    kind = str(rs.choice(["vec", "rows", "c0", "cap"], p=[.45, .35, .1, .1]))
    if kind == "vec" and fmt == "f32":
        c = 4 * int(rs.randint(2, 17))
    elif kind == "c0":
        c = 0
    else:
        c = int(rs.choice([1, 2, 3, 4, 5, 8, 10, 11, 13, 29, 61, 64, 128, 131, 259, 320]))
    if kind == "cap":
        fmt = "f32" if rs.rand() < 0.7 else fmt
        b, n, m, s = int(rs.choice([4300, 9000])), int(rs.randint(1, 4)), int(rs.randint(5, 12)), 32
        c = int(rs.choice([0, 1, 8, 16, 40]))
    else:
        b, n, m, s = int(rs.randint(1, 4)), log_int(rs, 1, 2000), log_int(rs, 1, 200), int(rs.choice([1, 3, 8, 16, 32]))
    scale = float(rs.choice([1.0, 1e-5, 1e5, 1e-39]))
    xyz = special_f32(rs, (b, n, 3), scale)
    new_xyz = special_f32(rs, (b, m, 3), scale)
    misal = kind == "rows" and fmt == "f32" and c % 4 == 0 and rs.rand() < 0.5
    return dict(case="group_concat", kind=kind, fmt=fmt, b=b, n=n, c=c, m=m, s=s, xyz_first=int(rs.randint(0, 2)),
                with_gx=bool(rs.rand() < 0.6), points_off=1 if misal else 0, out_off=0, scale=scale,
                pts=raw_bits(rs, (b, n, c), fmt), idx=rs.randint(0, n, (b, m, s)).astype(np.int32), xyz=xyz,
                new_xyz=new_xyz)


def run_group_concat(p):
    fmt, b, n, c, m, s = p["fmt"], p["b"], p["n"], p["c"], p["m"], p["s"]
    w = c + 3
    pts = dev_buf(p["pts"], p["points_off"], fmt) if c else None
    out = out_buf(b * m * s * w, 0, fmt)
    gx = out_buf(b * m * s * 3, 0, "f32") if p["with_gx"] else None
    rc = lib().pn2_group_concat_typed(DTYPE_CODE[fmt], b, n, c, m, s, ptr(F32(p["xyz"])), ptr(F32(p["new_xyz"])),
                                      elem_ptr(pts, p["points_off"]) if c else None, ptr(I32(p["idx"])),
                                      p["xyz_first"], ptr(out), ptr(gx) if gx is not None else None, stream_ptr(dev))
    body, clean = guarded(host_bits(out, fmt), 0, b * m * s * w, fmt)
    body = body.reshape(b, m, s, w)
    bi = np.arange(b)[:, None, None]
    with np.errstate(all="ignore"):
        diff = (p["xyz"][bi, p["idx"]] - p["new_xyz"][:, :, None, :]).astype(np.float32)
    lo = 0 if p["xyz_first"] else c
    fx = body[..., lo:lo + 3]
    fp = np.concatenate([body[..., :lo], body[..., lo + 3:]], -1)
    ok = rc == 0 and clean and np.array_equal(fp, p["pts"][bi, p["idx"]]) and same_or_nan(fx, diff, fmt)
    if gx is not None:
        gb, gclean = guarded(host_bits(gx, "f32"), 0, b * m * s * 3, "f32")
        ok = ok and gclean and same_or_nan(gb.reshape(b, m, s, 3), diff, "f32")
    return bool(ok)


# ------------------------------------------------------------------------------------------- ordered gradients
def exact_lists(rs, nt, lengths, total):
    """a target per entry: the first len(lengths) targets (a random subset) get exactly those many entries, the
    rest of the ``total`` entries go to the other targets at random, shuffled"""
    chosen = rs.permutation(nt)[:len(lengths)]
    fixed = np.repeat(chosen, lengths)
    others = np.setdiff1d(np.arange(nt), chosen)
    rest = others[rs.randint(0, len(others), max(total - len(fixed), 0))] if len(others) else np.zeros(0, np.int64)
    t = np.concatenate([fixed, rest])[:max(total, len(fixed))]
    return rs.permutation(t).astype(np.int32)


def draw_ordered_grad(rs):
    fmt = str(rs.choice(FMTS))
    weighted = bool(rs.rand() < 0.5)
    kind = str(rs.choice(["targets", "lists", "wide"], p=[.35, .45, .2]))
    nt = int(rs.choice(TARGETS)) if kind == "targets" else log_int(rs, 5, 3000)
    lens = sorted(set(int(rs.choice(LIST_LENGTHS)) for _ in range(4 if kind != "targets" else 2)))
    if kind == "wide":  # two or more channel passes in every list kernel
        c = int(rs.choice([259, 260, 1028, 1031])) if fmt == "f32" or rs.rand() < 0.5 else int(rs.choice([264, 1032]))
        lens = [int(rs.choice([257, 300, 2049, 2500]))] + [int(rs.choice([1, 40, 129]))]
    else:
        c = int(rs.choice([1, 3, 4, 8, 16, 33, 64, 128, 131]))
    b = int(rs.randint(1, 3))
    # finite data half the time: a NaN or inf among a long list's entries would hide how the list is associated
    finite = bool(rs.rand() < 0.5)
    base = sum(lens) + int(rs.randint(0, 3 * nt + 2))
    vec_off = int(rs.rand() < 0.25)
    if weighted:
        l0 = max(1, -(-base // 3))
        ragged = bool(rs.rand() < 0.5)
        # a ragged draw puts the exact lists in cloud 0 with at least 3 padding rows behind them, so its pieces are
        # cut from 3 * len, which gives another piece length than 3 * n (3 * (n - len) >= 9 > 8)
        n = l0 + int(rs.randint(3, l0 // 3 + 5)) if ragged else l0
        ls = [int(rs.randint(max(1, n - n // 3), n + 1)) if ragged else n for _ in range(b)]
        ls[0] = l0
        idx = np.stack([np.concatenate([exact_lists(rs, nt, lens, 3 * l0), np.full(3 * (n - l0), nt - 1, np.int32)])
                        if k == 0 else exact_lists(rs, nt, [], 3 * n) for k in range(b)]).reshape(b, n, 3)
        for k, l in enumerate(ls):
            idx[k, l:] = nt - 1  # padding: an in-range index that must never be counted
        wt = special_f32(rs, (b, n, 3)) if not finite else rs.random_sample((b, n, 3)).astype(np.float32)
        wt[rs.random_sample(wt.shape) < (0.6 if not finite else 0.1)] = np.float32(0.25)
        for k, l in enumerate(ls):
            wt[k, l:] = np.nan
        rows = n
    else:
        ragged, ls = False, None
        s = int(rs.choice([1, 4, 16]))
        m = max(1, -(-base // s))
        idx = np.stack([exact_lists(rs, nt, lens if k == 0 else [], m * s) for k in range(b)]).reshape(b, m, s)
        wt = None
        rows = m * s
        n = m
    go = special_f32(rs, (b, rows, c)) if not finite else rs.standard_normal((b, rows, c)).astype(np.float32)
    if fmt != "f32":
        go = NUM.quantize(go, fmt)
    return dict(case="ordered_grad", kind=kind, fmt=fmt, weighted=weighted, ragged=ragged, finite=finite, b=b, nt=nt, c=c, n=n,
                s=None if weighted else idx.shape[2], lens_exact=lens, lengths=ls, off=vec_off, idx=idx, w=wt, go=go)


def ordered_counts(p):
    """(b, nt) list lengths of the real entries"""
    b, nt = p["b"], p["nt"]
    out = np.zeros((b, nt), np.int64)
    for k in range(b):
        real = p["idx"][k][:p["lengths"][k]] if p["weighted"] else p["idx"][k]
        out[k] = np.bincount(real.reshape(-1), minlength=nt)
    return out


def ordered_want(p):
    b, nt = p["b"], p["nt"]
    res = []
    for k in range(b):
        if p["weighted"]:
            l = p["lengths"][k]
            res.append(R.ordered_sum(p["go"][k, :l], p["idx"][k, :l], nt, weight=p["w"][k, :l]))
        else:
            res.append(R.ordered_sum(p["go"][k], p["idx"][k].reshape(-1), nt))
    return np.stack(res)


def run_ordered_grad(p):
    fmt, b, nt, c, n = p["fmt"], p["b"], p["nt"], p["c"], p["n"]
    L = lib()
    off = p["off"]
    go = dev_buf(to_fmt_bits(p["go"], fmt), off, fmt)
    idx = I32(p["idx"])
    if p["weighted"]:
        wsb = int(L.pn2_three_interpolate_grad_det_workspace_bytes(b, n, nt))
    else:
        wsb = int(L.pn2_group_point_grad_det_workspace_bytes(b, nt, n, p["s"]))
    runs = []
    for _ in range(2):
        ws = torch.full((wsb,), 0x5A, dtype=torch.uint8, device=dev)
        gp = out_buf(b * nt * c, off, fmt)
        if p["weighted"]:
            lens = I32(p["lengths"]) if p["ragged"] else None
            rc = L.pn2_three_interpolate_grad_det_ragged_typed(DTYPE_CODE[fmt], b, n, c, nt, elem_ptr(go, off), ptr(idx),
                                                              ptr(F32(p["w"])), ptr(lens), elem_ptr(gp, off), ptr(ws), wsb,
                                                              stream_ptr(dev))
        else:
            rc = L.pn2_group_point_grad_det_typed(DTYPE_CODE[fmt], b, nt, c, n, p["s"], elem_ptr(go, off), ptr(idx),
                                                  elem_ptr(gp, off), ptr(ws), wsb, stream_ptr(dev))
        runs.append((rc, host_bits(gp, fmt)))
    (rc, got), (rc2, got2) = runs
    body, clean = guarded(got, off, b * nt * c, fmt)
    ok = rc == 0 and rc2 == 0 and clean and np.array_equal(got, got2)
    return bool(ok and same_or_nan(body.reshape(b, nt, c), ordered_want(p), fmt))


# -------------------------------------------------------------------------------------------- atomic gradients
def exact_values(rs, shape, lo=-8, hi=9):
    """small integers times a power of two: sums of a few thousand of them are exact in float32"""
    return (rs.randint(lo, hi, shape) * np.float32(2.0 ** int(rs.randint(-6, 3)))).astype(np.float32)


def ftz(x):
    """x with its subnormals flushed to zero: what a float atomic add sees.  PTX's atom / red .add.f32 on global memory
    flushes subnormal inputs and results to sign-preserving zero (the reference's atomicAdd kernels do the same); the
    products of three_interpolate's gradient stay subnormal for subnormal rows (weights are at most 1), so flushing
    the rows flushes the terms.  Only the ordered (deterministic) sums keep subnormals."""
    x = np.asarray(x, np.float32)
    return np.where(np.abs(x) < np.float32(2.0 ** -126), np.float32(0), x).astype(np.float32)


def exact_specials(rs, shape, fmt="f32"):
    """exact_values on a grid of normal or subnormal numbers (2^-140 in float32 and bfloat16, 2^-22 in float16), with
    a few NaN, ±inf and −0.0 mixed in: NaN and inf are absorbing and every finite partial sum is exact, so any order of
    addition gives the same bits"""
    x = exact_values(rs, shape)
    if rs.rand() < 0.3:
        x = (x * np.float32(2.0 ** (-140 if fmt != "f16" else -22))).astype(np.float32)
    u = rs.random_sample(shape)
    x[u < 0.004] = np.array([np.nan, np.inf, -np.inf, -0.0], np.float32)[rs.randint(0, 4, int((u < 0.004).sum()))]
    return x


def draw_atomic_grad(rs):
    which = str(rs.choice(["group_point", "three_interp", "gather"]))
    exact = bool(rs.rand() < 0.5)
    fmt = str(rs.choice(FMTS)) if which == "group_point" else "f32"
    c = int(rs.choice([1, 4, 8, 13, 64, 128, 131])) if which != "gather" else 3
    ragged = which == "three_interp" and bool(rs.rand() < 0.5)
    b = int(rs.randint(1, 4))
    big = rs.rand() < 0.25  # past grid_for's cap (SMS * 64 CTAs)
    if which == "group_point":
        n, m, s = log_int(rs, 1, 2000), log_int(rs, 1, 200), int(rs.choice([1, 8, 32]))
        if big:
            b, c, m, s = 4, 4, 8500, 64
        idx = rs.randint(0, n, (b, m, s)).astype(np.int32)
        gshape = (b, m, s, c)
    elif which == "three_interp":
        n, m = log_int(rs, 1, 4000), log_int(rs, 1, 500)
        if big:  # m = 64: ~28 000 entries per target, exact-sum inputs stay below 2^24 units
            b, c, n, m = 4, 4, 600000, 64
        idx = rs.randint(0, m, (b, n, 3)).astype(np.int32)
        gshape = (b, n, c)
    else:
        n, m = log_int(rs, 1, 3000), log_int(rs, 1, 3000)
        if big:
            b, m = 9, 250000
        idx = rs.randint(0, n, (b, m)).astype(np.int32)
        gshape = (b, m, 3)
    go = exact_specials(rs, gshape, fmt) if exact else rs.standard_normal(gshape).astype(np.float32)
    if fmt != "f32":
        go = NUM.quantize(go, fmt)
    w = None
    if which == "three_interp":
        w = (rs.randint(0, 5, (b, n, 3)) * 0.25).astype(np.float32) if exact else rs.random_sample((b, n, 3)).astype(np.float32)
    ls = [int(rs.randint(1, n + 1)) if ragged else n for _ in range(b)]
    return dict(case="atomic_grad", which=which, exact=exact, fmt=fmt, b=b, n=n, m=m, c=c, big=bool(big),
                ragged=ragged, lengths=ls, off=int(rs.rand() < 0.25), idx=idx, go=go, w=w,
                pts=special_f32(rs, (b, n, 3)) if which == "gather" else None)


def run_atomic_grad(p):
    L = lib()
    fmt, b, n, m, c, off = p["fmt"], p["b"], p["n"], p["m"], p["c"], p["off"]
    idx = I32(p["idx"])
    if p["which"] == "group_point":
        s = p["idx"].shape[2]
        go = dev_buf(to_fmt_bits(p["go"], fmt), off, fmt)
        acc = torch.zeros(b * n * c + off, dtype=torch.float32, device=dev)
        gp = out_buf(b * n * c, 0, fmt) if fmt != "f32" else acc
        rc = L.pn2_group_point_grad_typed(DTYPE_CODE[fmt], b, n, c, m, s, elem_ptr(go, off), ptr(idx),
                                          elem_ptr(gp, off if fmt == "f32" else 0),
                                          elem_ptr(acc, off) if fmt != "f32" else None, stream_ptr(dev))
        if fmt == "f32":
            got = acc.cpu().numpy()[off:]
            got_bits = got.view(np.uint32)
        else:
            got_bits, clean = guarded(host_bits(gp, fmt), 0, b * n * c, fmt)
            if not clean:
                return False
        want = O.oracle_group_point_grad((b, n, c), p["idx"], ftz(p["go"]))
        targets = [p["idx"][k].reshape(-1) for k in range(b)]
        terms = [p["go"][k].reshape(-1, c) for k in range(b)]
        nt = n
    elif p["which"] == "three_interp":
        go = F32(np.concatenate([np.zeros(off, np.float32), p["go"].reshape(-1)]))
        acc = torch.zeros(b * m * c + off, dtype=torch.float32, device=dev)
        ls = p["lengths"]
        lens = I32(ls) if p["ragged"] else None
        w = p["w"].copy()
        for k, l in enumerate(ls):
            w[k, l:] = np.nan  # padding rows: never read
        rc = L.pn2_three_interpolate_grad_ragged(b, n, c, m, elem_ptr(go, off), ptr(idx), ptr(F32(w)), ptr(lens),
                                                 elem_ptr(acc, off), stream_ptr(dev))
        got_bits = acc.cpu().numpy()[off:].view(np.uint32)
        want = np.stack([O.oracle_three_interpolate_grad((1, m, c), p["idx"][k:k + 1, :l], p["w"][k:k + 1, :l],
                                                         ftz(p["go"][k:k + 1, :l]))[0] for k, l in enumerate(ls)])
        targets = [p["idx"][k, :l].reshape(-1) for k, l in enumerate(ls)]
        terms = [(np.repeat(p["go"][k, :l].astype(np.float64), 3, axis=0) * p["w"][k, :l].reshape(-1, 1))
                 for k, l in enumerate(ls)]
        nt = m
    else:
        out = out_buf(b * m * 3, 0, "f32")
        rc0 = L.pn2_gather_point(b, n, m, ptr(F32(p["pts"])), ptr(idx), ptr(out), stream_ptr(dev))
        body, clean = guarded(host_bits(out, "f32"), 0, b * m * 3, "f32")
        bi = np.arange(b)[:, None]
        if rc0 != 0 or not clean or not np.array_equal(body, p["pts"][bi, p["idx"]].reshape(-1).view(np.uint32)):
            return False
        acc = torch.zeros(b * n * 3, dtype=torch.float32, device=dev)
        rc = L.pn2_gather_point_grad(b, n, m, ptr(F32(p["go"])), ptr(idx), ptr(acc), stream_ptr(dev))
        got_bits = acc.cpu().numpy().view(np.uint32)
        want = O.oracle_gather_point_grad((b, n, 3), p["idx"], ftz(p["go"]))
        targets = [p["idx"][k] for k in range(b)]
        terms = [p["go"][k] for k in range(b)]
        nt, c = n, 3
    if rc != 0:
        return False
    if p["exact"]:
        return same_or_nan(got_bits.reshape(want.shape), want, fmt)
    got = values(got_bits, fmt).reshape(b, nt, c)
    ok = True
    for k in range(b):
        ref, mass, count = NUM.scatter64(nt, targets[k], terms[k])
        ok = ok and bool(np.all(NUM.within_bound(got[k], ref, mass, np.maximum(count, 1)[:, None], fmt)))
    return ok


# ------------------------------------------------------------------------------------------- three_interpolate
def draw_interp(rs):
    fmt = str(rs.choice(FMTS))
    c = int(rs.choice([1, 3, 4, 8, 12, 13, 64, 131, 256]))
    b, n, m = int(rs.randint(1, 4)), log_int(rs, 1, 5000), log_int(rs, 1, 600)
    if rs.rand() < 0.15:  # past grid_for's cap, vec4 (c = 4, aligned) or scalar
        b, c, n, m = 4, int(rs.choice([4, 5])), 600000, 64
    ragged = bool(rs.rand() < 0.5)
    ls = [int(rs.randint(1, n + 1)) if ragged else n for _ in range(b)]
    pts = special_f32(rs, (b, m, c))
    if fmt != "f32":
        pts = NUM.quantize(pts, fmt)
    return dict(case="interp", fmt=fmt, b=b, n=n, m=m, c=c, ragged=ragged, lengths=ls, off=int(rs.rand() < 0.25),
                pts=pts, idx=rs.randint(0, m, (b, n, 3)).astype(np.int32), w=special_f32(rs, (b, n, 3)))


def run_interp(p):
    fmt, b, n, m, c, off = p["fmt"], p["b"], p["n"], p["m"], p["c"], p["off"]
    pts = dev_buf(to_fmt_bits(p["pts"], fmt), off, fmt)
    out = out_buf(b * n * c, off, fmt)
    lens = I32(p["lengths"]) if p["ragged"] else None
    rc = lib().pn2_three_interpolate_ragged_typed(DTYPE_CODE[fmt], b, m, c, n, elem_ptr(pts, off), ptr(I32(p["idx"])),
                                                 ptr(F32(p["w"])), ptr(lens), elem_ptr(out, off), stream_ptr(dev))
    body, clean = guarded(host_bits(out, fmt), off, b * n * c, fmt)
    body = body.reshape(b, n, c)
    want = O.oracle_three_interpolate(p["pts"], p["idx"], p["w"])
    real = np.arange(n)[None, :] < np.asarray(p["lengths"])[:, None]
    return bool(rc == 0 and clean and same_or_nan(body[real], want[real], fmt) and np.all(body[~real] == 0))


# ---------------------------------------------------------------------------------------------- selection_sort
def draw_selection_sort(rs):
    n = int(rs.choice([rs.randint(1, 32), 32, rs.randint(33, 100), rs.randint(100, 700)]))
    k = int(rs.choice([1, 2, max(1, n // 3), n, n + 5]))
    b, m = int(rs.randint(1, 3)), int(rs.randint(1, 40))
    kind = str(rs.choice(["nan_at_s", "nan", "ties", "mixed"]))
    d = rs.randint(0, 6, (b, m, n)).astype(np.float32) if kind == "ties" else rs.random_sample((b, m, n)).astype(np.float32)
    u = rs.random_sample((b, m, n))
    frac = float(rs.choice([0.02, 0.1, 0.4]))
    if kind in ("nan", "mixed"):
        d[u < frac] = np.nan
    if kind == "nan_at_s":  # NaN at the first positions, where the early rounds start
        d[..., :int(rs.randint(1, 4))] = np.nan
        d[u < frac / 4] = np.nan
    if kind in ("ties", "mixed"):
        d[u > 0.9] = -0.0
        d[(u > 0.8) & (u <= 0.9)] = 0.0
        d[(u > 0.75) & (u <= 0.8)] = np.inf
        d[(u > 0.7) & (u <= 0.75)] = -np.inf
    return dict(case="selection_sort", kind=kind, b=b, m=m, n=n, k=k, nan_rows=int(np.isnan(d).any(-1).sum()), d=d)


def run_selection_sort(p):
    b, m, n, k = p["b"], p["m"], p["n"], p["k"]
    outi = torch.full((b * m * n,), -7, dtype=torch.int32, device=dev)
    out = out_buf(b * m * n, 0, "f32")
    rc = lib().pn2_selection_sort(b, n, m, k, ptr(F32(p["d"])), ptr(outi), ptr(out), stream_ptr(dev))
    wi, wv = O.oracle_selection_sort(k, p["d"])
    body, clean = guarded(host_bits(out, "f32"), 0, b * m * n, "f32")
    return bool(rc == 0 and clean and np.array_equal(outi.cpu().numpy(), wi.reshape(-1))
                and np.array_equal(body, wv.reshape(-1).view(np.uint32)))


# ----------------------------------------------------------------------------------------------------- refusals
REFUSALS = ["group_point_b", "group_concat_b", "grad_det_ws", "interp_grad_det_ws", "bad_dtype", "null_idx",
            "null_out", "null_points"]


def draw_refused(rs):
    return dict(case="refused", why=str(REFUSALS[rs.randint(len(REFUSALS))]), fmt=str(rs.choice(FMTS)),
                c=int(rs.choice([3, 5, 13])))


def run_refused(p):
    L = lib()
    fmt, c, why = p["fmt"], p["c"], p["why"]
    code = DTYPE_CODE[fmt]
    b, n, m, s = 65536 if why in ("group_point_b", "group_concat_b") else 2, 4, 2, 2
    pts = dev_buf(np.zeros(b * n * c, RAW[fmt]), 0, fmt)
    idx = I32(np.zeros((b, m, s)))
    numel = b * m * s * (c + 3)
    out = out_buf(numel, 0, fmt)
    xyz, nx = F32(np.zeros((b, n, 3))), F32(np.zeros((b, m, 3)))
    torch.cuda.synchronize(dev)
    before = _lib.launch_count()
    if why == "group_point_b":
        rc = L.pn2_group_point_typed(code, b, n, c, m, s, ptr(pts), ptr(idx), ptr(out), stream_ptr(dev))
    elif why == "group_concat_b":
        rc = L.pn2_group_concat_typed(code, b, n, c, m, s, ptr(xyz), ptr(nx), ptr(pts), ptr(idx), 1, ptr(out), None,
                                      stream_ptr(dev))
    elif why == "grad_det_ws":
        wsb = int(L.pn2_group_point_grad_det_workspace_bytes(b, n, m, s))
        ws = torch.empty(wsb, dtype=torch.uint8, device=dev)
        rc = L.pn2_group_point_grad_det_typed(code, b, n, c, m, s, ptr(pts), ptr(idx), ptr(out), ptr(ws), wsb - 1,
                                              stream_ptr(dev))
    elif why == "interp_grad_det_ws":
        wsb = int(L.pn2_three_interpolate_grad_det_workspace_bytes(b, n, m))
        ws = torch.empty(wsb, dtype=torch.uint8, device=dev)
        i3 = I32(np.zeros((b, n, 3)))
        rc = L.pn2_three_interpolate_grad_det_typed(code, b, n, c, m, ptr(pts), ptr(i3), ptr(F32(np.zeros((b, n, 3)))),
                                                    ptr(out), ptr(ws), wsb - 1, stream_ptr(dev))
    elif why == "bad_dtype":
        rc = L.pn2_group_point_typed(7, b, n, c, m, s, ptr(pts), ptr(idx), ptr(out), stream_ptr(dev))
    elif why == "null_idx":
        rc = L.pn2_group_point_typed(code, b, n, c, m, s, ptr(pts), None, ptr(out), stream_ptr(dev))
    elif why == "null_out":
        rc = L.pn2_group_concat_typed(code, b, n, c, m, s, ptr(xyz), ptr(nx), ptr(pts), ptr(idx), 0, None, None,
                                      stream_ptr(dev))
    else:
        rc = L.pn2_group_concat_typed(code, b, n, c, m, s, ptr(xyz), ptr(nx), None, ptr(idx), 0, ptr(out), None,
                                      stream_ptr(dev))
    launched = _lib.launch_count() - before
    torch.cuda.synchronize(dev)
    untouched = bool(np.all(host_bits(out, fmt) == POISON[fmt]))
    return rc == CUDA_ERROR_INVALID_VALUE and launched == 0 and untouched


# ------------------------------------------------------------------------------------------- torch + autograd
def draw_autograd(rs):
    fmt = str(rs.choice(FMTS))
    b, n, m, s = int(rs.randint(1, 3)), log_int(rs, 4, 500), log_int(rs, 1, 64), int(rs.choice([4, 16]))
    c = int(rs.choice([8, 13, 64]))
    return dict(case="autograd", fmt=fmt, b=b, n=n, m=m, s=s, c=c, det=bool(rs.rand() < 0.5),
                pts=exact_specials(rs, (b, n, c), fmt), xyz=special_f32(rs, (b, n, 3)),
                new_xyz=rs.random_sample((b, m, 3)).astype(np.float32),
                idx=rs.randint(0, n, (b, m, s)).astype(np.int32), go=exact_specials(rs, (b, m, s, c + 3), fmt))


def run_autograd(p):
    from pointnet2_b200.pointnet_util import group_and_concat
    fmt, c = p["fmt"], p["c"]
    prev = torch.are_deterministic_algorithms_enabled()
    try:
        torch.use_deterministic_algorithms(p["det"])
        pt = F32(p["pts"]).to(TORCH[fmt]).requires_grad_(True)
        cat, _ = group_and_concat(F32(p["xyz"]), F32(p["new_xyz"]), pt, I32(p["idx"]), xyz_first=True)
        cat.backward(F32(p["go"]).to(TORCH[fmt]))
    finally:
        torch.use_deterministic_algorithms(prev)
    bi = np.arange(p["b"])[:, None, None]
    want_f = p["pts"][bi, p["idx"]]
    with np.errstate(all="ignore"):
        diff = (p["xyz"][bi, p["idx"]] - p["new_xyz"][:, :, None, :]).astype(np.float32)
    got = host_bits(cat, fmt)
    ok = same_or_nan(got[..., 3:], want_f, fmt) and same_or_nan(got[..., :3], diff, fmt)
    gq = NUM.quantize(p["go"][..., 3:], fmt)
    gw = O.oracle_group_point_grad((p["b"], p["n"], c), p["idx"], gq if p["det"] else ftz(gq))
    return bool(ok and same_or_nan(host_bits(pt.grad, fmt), gw, fmt))


# ------------------------------------------------------------------------------------------------ FP front end
FP_COMBOS = [(g, t, rg) for g in (1, 2, 4, 8, 16, 32) for t in ("float", "u16") for rg in (False, True)]
FRONT_BUDGET = 2 * R.SMS * R.NN_THREADS  # fp_front_dispatch: lanes per point grow while b * n * G stays below this


def draw_fp_front(rs, k):
    """the k-th case of a seed takes FP_COMBOS[k % 24]: b, n and m are drawn so that fp_front_dispatch picks its G,
    either because 2G lanes would exceed the known pairs (m) or because b * n * G fills the machine"""
    g, t, ragged = FP_COMBOS[k % len(FP_COMBOS)]
    fmt = "f32" if t == "float" else str(rs.choice(["bf16", "f16"]))
    by_m = bool(rs.rand() < 0.5)
    b = int(rs.randint(1, 4))
    if g == 32 or (by_m and g > 1):
        # G reached: b * n * G / 2 below the budget and G <= (m + 1) // 2; stopped there: 2G > (m + 1) // 2
        n = int(rs.randint(1, (FRONT_BUDGET // 16 - 1) // b + 1 if g == 32 else (FRONT_BUDGET // g) // b + 1))
        m = int(rs.randint(2 * g - 1, 4 * g - 1)) if g < 32 else log_int(rs, 63, 700)
    elif g == 1 and by_m:
        n, m = log_int(rs, 1, 3000), int(rs.randint(1, 3))
    else:  # b * n * G >= the budget, b * n * G / 2 below it
        lo, hi = -(-FRONT_BUDGET // g), -(-2 * FRONT_BUDGET // g) - 1 if g > 1 else 2 * FRONT_BUDGET
        b = 1
        n, m = int(rs.randint(lo, hi + 1)), int(rs.randint(8 * g - 1, 8 * g + 200))
    c2, c1 = int(rs.choice([1, 3, 4, 8, 64, 131])), int(rs.choice([0, 3, 4, 64]))
    xyz1 = rs.random_sample((b, n, 3)).astype(np.float32)
    xyz2 = rs.random_sample((b, m, 3)).astype(np.float32)
    if m <= n and rs.rand() < 0.4:
        xyz2 = xyz1[:, :m].copy()  # nested sets as in feature propagation: exact zero distances
    if rs.rand() < 0.3:
        xyz2[:, rs.randint(0, m, max(1, m // 4))] = xyz2[:, :1]  # coincident known points: distance ties
    ls = [int(rs.randint(1, n + 1)) if ragged else n for _ in range(b)]
    p2 = special_f32(rs, (b, m, c2))
    if fmt != "f32":
        p2 = NUM.quantize(p2, fmt)
    return dict(case="fp_front", g=g, fmt=fmt, ragged=ragged, b=b, n=n, m=m, c2=c2, c1=c1, lengths=ls,
                xyz1=NUM.pad_rows(xyz1, ls, "poison"), xyz2=xyz2, p2=p2, p1=raw_bits(rs, (b, n, c1), fmt))


def fp_weights(d):
    """the FP front end's weights from its float32 distances: r = 1 / max(d, 1e-10), w = r / ((r1 + r2) + r3)"""
    with np.errstate(all="ignore"):
        r = (np.float32(1) / np.fmax(d, np.float32(1e-10))).astype(np.float32)
        norm = ((r[..., 0] + r[..., 1]).astype(np.float32) + r[..., 2]).astype(np.float32)
        return (r / norm[..., None]).astype(np.float32)


def run_fp_front(p):
    L = lib()
    fmt, b, n, m, c2, c1 = p["fmt"], p["b"], p["n"], p["m"], p["c2"], p["c1"]
    code = DTYPE_CODE[fmt]
    x1, x2 = F32(p["xyz1"]), F32(p["xyz2"])
    lens = I32(p["lengths"]) if p["ragged"] else None
    p2 = dev_buf(to_fmt_bits(p["p2"], fmt), 0, fmt)
    p1 = dev_buf(p["p1"], 0, fmt) if c1 else None
    out = out_buf(b * n * c2, 0, fmt)
    cat = out_buf(b * n * (c2 + c1), 0, fmt)
    dist, wgt = out_buf(b * n * 3, 0, "f32"), out_buf(b * n * 3, 0, "f32")
    idx = torch.full((b * n * 3,), -7, dtype=torch.int32, device=dev)
    rc = L.pn2_three_nn_interpolate_ragged_typed(code, b, n, m, c2, ptr(x1), ptr(lens), ptr(x2), ptr(p2), ptr(out),
                                                 ptr(dist), ptr(idx), ptr(wgt), stream_ptr(dev))
    rc2 = L.pn2_fp_interpolate_concat_ragged_typed(code, b, n, m, c2, c1, ptr(x1), ptr(lens), ptr(x2), ptr(p1),
                                                   ptr(p2), ptr(cat), stream_ptr(dev))
    ob, ok1 = guarded(host_bits(out, fmt), 0, b * n * c2, fmt)
    cb, ok2 = guarded(host_bits(cat, fmt), 0, b * n * (c2 + c1), fmt)
    db, ok3 = guarded(host_bits(dist, "f32"), 0, b * n * 3, "f32")
    wb, ok4 = guarded(host_bits(wgt, "f32"), 0, b * n * 3, "f32")
    ok = rc == 0 and rc2 == 0 and ok1 and ok2 and ok3 and ok4
    ob, cb = ob.reshape(b, n, c2), cb.reshape(b, n, c2 + c1)
    db, wb, ib = db.reshape(b, n, 3), wb.reshape(b, n, 3), idx.cpu().numpy().reshape(b, n, 3)
    for k, l in enumerate(p["lengths"]):
        od, oi = O.oracle_three_nn(p["xyz1"][k:k + 1, :l], p["xyz2"][k:k + 1])
        w = fp_weights(od)
        want = O.oracle_three_interpolate(p["p2"][k:k + 1], oi, w)[0]
        ok = ok and np.array_equal(ib[k, :l], oi[0]) and same_or_nan(db[k, :l], od[0], "f32")
        ok = ok and same_or_nan(wb[k, :l], w[0], "f32") and same_or_nan(ob[k, :l], want, fmt)
        ok = ok and same_or_nan(cb[k, :l, :c2], want, fmt) and np.array_equal(cb[k, :l, c2:], p["p1"][k, :l])
        pad = slice(l, n)  # padding rows: idx 0, dist +inf, weight 0, features 0
        ok = ok and (ib[k, pad] == 0).all() and (db[k, pad] == np.float32(np.inf).view(np.uint32)).all()
        ok = ok and (wb[k, pad] == 0).all() and (ob[k, pad] == 0).all() and (cb[k, pad] == 0).all()
    return bool(ok)


CASES = ["group_point", "group_concat", "ordered_grad", "atomic_grad", "interp", "selection_sort", "refused",
         "autograd", "fp_front"]
DRAW = {name: globals()["draw_" + name] for name in CASES}
RUN = {name: globals()["run_" + name] for name in CASES}


def draws(seed: int, iterations: int):
    """The parameters ``run(seed, iterations)`` uses, without a device (the run_* functions draw nothing)."""
    rs = np.random.RandomState(seed)
    return [_draw(rs, seed, it) for it in range(iterations)]


def _draw(rs, seed, it):
    """case `it` of a seed; the FP front end draws from its own stream, so adding it left the other cases' draws
    as they were"""
    name = SCHEDULE[it % len(SCHEDULE)]
    if name == "fp_front":
        return draw_fp_front(np.random.RandomState([seed, it]), it // len(SCHEDULE))
    return DRAW[name](rs)


def public(p):
    """the parameters of a case without its input arrays (they follow from the seed and the iteration)"""
    return {k: v for k, v in p.items() if not isinstance(v, np.ndarray)}


def _one(rs, seed, it, counts, fails, catch):
    name = SCHEDULE[it % len(SCHEDULE)]
    p = _draw(rs, seed, it)
    _LIVE.clear()
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
        _one(rs, seed, it, counts, fails, catch=False)
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
