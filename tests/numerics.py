"""Reference arithmetic for the tests: one float32 -> 16-bit rounding, and the float64 error bound of a float32 sum.

Numpy only (no torch, no device), so CPU tests can check it against hand-computed values.  Formats are named by
string: "f32", "bf16", "f16".

* ``round_once(x, fmt)``: the bits of float32 ``x`` rounded once, to nearest even, into ``fmt`` (uint16 for the 16-bit
  formats, float32 unchanged for "f32"): what ``__float2bfloat16_rn`` / ``__float2half_rn`` and torch's ``.to(D)`` do.
* ``scatter64``: the exact (float64) per-target sums of a scatter-add and their absolute mass Σ|term|.
* ``within_bound``: |got − ref64| ≤ γ·mass (+ ½ ulp of the 16-bit result), the bound any float32 summation order
  satisfies.  It replaces fixed atols where a result is not bit-exact by contract (float atomics, the eight-piece sums
  of long lists).
"""
from __future__ import annotations

import numpy as np

U32 = 2.0 ** -24  # unit roundoff of float32 (round to nearest)

# mantissa bits and smallest normal exponent of each format
_FORMATS = {"f32": (23, -126), "bf16": (7, -126), "f16": (10, -14)}


def round_once(x, fmt: str) -> np.ndarray:
    """float32 array -> its round-to-nearest-even image in ``fmt``: uint16 bit patterns for "bf16" / "f16", the float32
    values themselves for "f32".  Overflow goes to ±inf; a NaN becomes torch's canonical NaN (bf16 0x7fc0)."""
    x = np.ascontiguousarray(x, dtype=np.float32)
    if fmt == "f32":
        return x
    if fmt == "f16":
        with np.errstate(over="ignore"):
            return x.astype(np.float16).view(np.uint16)  # numpy converts float32 -> float16 with one RNE rounding
    if fmt != "bf16":
        raise ValueError(fmt)
    u = x.view(np.uint32).astype(np.uint64)
    r = ((u + 0x7FFF + ((u >> 16) & 1)) >> 16).astype(np.uint16)
    r[np.isnan(x)] = 0x7FC0
    return r


def decode(bits, fmt: str) -> np.ndarray:
    """The float32 values of ``fmt`` data (uint16 bit patterns for the 16-bit formats): an exact upcast."""
    if fmt == "f32":
        return np.asarray(bits, dtype=np.float32)
    b = np.ascontiguousarray(bits).view(np.uint16)
    if fmt == "f16":
        return b.view(np.float16).astype(np.float32)
    return (b.astype(np.uint32) << 16).view(np.float32)


def quantize(x, fmt: str) -> np.ndarray:
    """float32 ``x`` rounded once to ``fmt`` and upcast again: the float32 values a ``fmt`` tensor made from x holds."""
    return decode(round_once(x, fmt), fmt)


def ulp(x, fmt: str) -> np.ndarray:
    """Spacing of ``fmt`` numbers at |x| (float64): 2^(max(e, emin) − p) for 2^e ≤ |x| < 2^(e+1), the subnormal
    spacing at and below the smallest normal."""
    p, emin = _FORMATS[fmt]
    a = np.abs(np.asarray(x, dtype=np.float64))
    _, e2 = np.frexp(a)  # a = f·2^e2 with 0.5 ≤ f < 1, so e = e2 − 1 (frexp(0) gives 0)
    e = np.where(a > 0, e2 - 1, emin)
    return np.ldexp(1.0, np.maximum(e, emin) - p)


def scatter64(n_targets: int, targets, terms):
    """Exact sums of a scatter-add in float64: ``ref[t] = Σ terms[e]`` and ``mass[t] = Σ |terms[e]|`` over the entries e
    with targets[e] = t.  ``targets`` (E,) ints in [0, n_targets), ``terms`` (E,) or (E, c) (float32 products are exact
    in float64).  Returns (ref, mass, count) with count[t] the list length of target t."""
    targets = np.asarray(targets, dtype=np.int64).ravel()
    terms = np.asarray(terms, dtype=np.float64)
    terms = terms.reshape(len(targets), -1)
    ref = np.zeros((n_targets, terms.shape[1]), np.float64)
    mass = np.zeros_like(ref)
    np.add.at(ref, targets, terms)
    np.add.at(mass, targets, np.abs(terms))
    return ref, mass, np.bincount(targets, minlength=n_targets)


def gamma(length):
    """γ = (L+1)·u / (1 − (L+1)·u): a float32 sum of L rounded products, in any order, is within γ·Σ|terms| of the
    exact sum (Higham, Accuracy and Stability of Numerical Algorithms, §3.1), u = 2^-24."""
    k = (np.asarray(length, dtype=np.float64) + 1.0) * U32
    return k / (1.0 - k)


def within_bound(got, ref64, mass, length, fmt: str) -> np.ndarray:
    """Elementwise |got − ref64| ≤ γ(L)·mass, plus, for a 16-bit result, ½ ulp of that format at |ref64| + γ(L)·mass
    (the float32 sum lies within γ·mass of ref64 and is rounded once; the ulp is taken at the largest magnitude it can
    have, so a binade boundary between ref64 and the float32 sum cannot break the bound).  ``length`` is the longest
    list L (a scalar, or per element).  For finite results; NaN in ``got`` fails."""
    ref64 = np.asarray(ref64, dtype=np.float64)
    err = gamma(length) * np.asarray(mass, dtype=np.float64)
    tol = err if fmt == "f32" else err + 0.5 * ulp(np.abs(ref64) + err, fmt)
    return np.abs(np.asarray(got, dtype=np.float64) - ref64) <= tol


FAR = np.float32(50.0)


def pad_rows(x, lengths, kind: str) -> np.ndarray:
    """A copy of ``x`` (b, n, ...) whose rows from lengths[i] on are overwritten: "poison" cycles NaN, +inf, −inf and a
    far point (FAR, −FAR, FAR, ...); "copy" repeats the real rows (row r holds row r mod lengths[i]).  Real rows are
    never touched."""
    x = np.array(x, copy=True)
    for i, l in enumerate(lengths):
        rows = np.arange(int(l), x.shape[1])
        if not len(rows):
            continue
        if kind == "poison":
            x[i, rows[0::4]] = np.nan
            x[i, rows[1::4]] = np.inf
            x[i, rows[2::4]] = -np.inf
            far = np.full(x.shape[2:], FAR, x.dtype)
            if far.ndim:
                far.reshape(-1)[1::2] = -FAR
            x[i, rows[3::4]] = far
        elif kind == "copy":
            x[i, rows] = x[i, rows % int(l)]
        else:
            raise ValueError(kind)
    return x


def pad_index_rows(idx, weight, lengths, kind: str, m: int):
    """Padding rows of an interpolation's idx / weight (b, n, 3): "poison" = the in-range index m − 1 and NaN weights,
    "copy" = the real rows repeated.  Real rows are never touched."""
    idx, weight = np.array(idx, copy=True), np.array(weight, copy=True)
    for k, l in enumerate(lengths):
        l = int(l)
        if kind == "poison":
            idx[k, l:] = m - 1
            weight[k, l:] = np.nan
        else:
            rows = np.arange(l, idx.shape[1]) % l
            idx[k, l:] = idx[k, rows]
            weight[k, l:] = weight[k, rows]
    return idx, weight
