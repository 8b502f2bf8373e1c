"""Reference side of the fused inference MLP kernels (csrc/mlp_tile.cuh, sa_mlp.cu, fp_mlp.cu), numpy only.

* ``sa_plan`` / ``row_plan``: the tile planners ``sa_mlp_plan_launch`` / ``row_mlp_plan_launch`` restated (row strides,
  weight slabs, the shared-memory formula, the slot loop), and ``branches``: the planner branches a shape takes.
* ``sa_rows`` / ``max_pool``: the set-abstraction gather (float32 ``xyz[idx] - new_xyz``, what ``__fsub_rn`` computes,
  then one rounding to the arithmetic format) and a NaN-propagating max over each group.
* ``bound16``: the float64 reference of the 16-bit path and an elementwise bound on the kernel's distance from it.
* ``simulate16``: a CPU model of the 16-bit kernel (float32 accumulation in a random order, one rounding per layer),
  on which the bound is checked without a GPU.

Layers are dicts as ``oracle.oracle_mlp_rows_f32`` takes them: "w" (cout, cin) and optional "b", "gamma", "beta",
"mean", "var", "eps", "relu".  The float32 (scale, shift) of a layer come from ``oracle.oracle_mlp_affine_f32``.
"""
from __future__ import annotations

import numpy as np

import numerics as NUM

SMEM_LIMIT = 227 * 1024   # kMlpSmemLimit
TN, KS = 64, 32           # output channels per pass, input channels per weight slab
MAX_LAYERS, MAX_WIDTH = 4, 1024
SA_MAX_IN, ROW_MAX_IN = MAX_WIDTH + 3, 1536
TILES = (64, 32, 16)
ESIZE = {"f32": 4, "bf16": 2, "f16": 2}

# Unit roundoff assumed for the float32 accumulation inside mma.sync (4 x the float32 unit roundoff): the tensor cores
# are documented to truncate rather than round in accumulation on earlier generations, and no measurement for Hopper is
# known to us.  The observed worst err / bound is recorded in DESIGN.md §6.13.
U_MMA = 2.0 ** -22
# smallest magnitude that rounds to inf in each 16-bit format
OVERFLOW = {"f16": 65520.0, "bf16": float(np.float32(3.3961514e38))}


# ------------------------------------------------------------------------------------------------------ planners
def act_stride(esize: int, c: int) -> int:
    return (c + 31) // 32 * 32 + 4 if esize == 4 else (c + 63) // 64 * 64 + 8


def slab_elems(esize: int) -> int:
    return 2 * TN * (KS + 4 if esize == 4 else KS + 8)


def _strides(esize, cin, widths, stored):
    """row strides of the two activation buffers: buffer 0 holds the input and the outputs of layers 1, 3, buffer 1
    those of layers 0, 2; ``stored`` layers' outputs take a buffer"""
    w0, w1 = cin, 1
    for l in range(stored):
        if l & 1:
            w0 = max(w0, widths[l])
        else:
            w1 = max(w1, widths[l])
    return act_stride(esize, w0), act_stride(esize, w1)


def sa_smem(esize, cin, widths, tm, slots):
    s0, s1 = _strides(esize, cin, widths, len(widths) - 1)
    return esize * (tm * (s0 + s1) + slab_elems(esize)) + 4 * 2 * max(widths) + 4 * tm + 4 * slots * widths[-1]


def sa_plan(esize, cin, widths, k, groups=1):
    """sa_mlp_plan_launch: {"tm", "slots" (groups per tile), "trimmed", "pieces", "grid", "smem"}, or None when no tile
    fits"""
    for tm in TILES:
        if sa_smem(esize, cin, widths, tm, 1) > SMEM_LIMIT:
            continue
        want = tm // k if k <= tm else 1
        slots = want
        while slots > 1 and sa_smem(esize, cin, widths, tm, slots) > SMEM_LIMIT:
            slots -= 1
        return dict(tm=tm, slots=slots, trimmed=slots < want, pieces=-(-k // tm) if k > tm else 1,
                    grid=-(-groups // slots), smem=sa_smem(esize, cin, widths, tm, slots))
    return None


def row_smem(esize, cin, widths, tm):
    s0, s1 = _strides(esize, cin, widths, len(widths))
    return esize * (tm * (s0 + s1) + slab_elems(esize)) + 4 * 2 * max(widths) + 4 * tm


def row_plan(esize, cin, widths, rows=1):
    """row_mlp_plan_launch: {"tm", "grid", "smem"}, or None"""
    for tm in TILES:
        smem = row_smem(esize, cin, widths, tm)
        if smem <= SMEM_LIMIT:
            return dict(tm=tm, grid=-(-rows // tm), smem=smem)
    return None


def branches(kind, esize, cin, widths, plan, k=None, rows=None):
    """the planner and tile branches one launch takes (kind "sa" or "rows")"""
    tm = plan["tm"]
    tags = {f"{kind}_e{esize}_tm{tm}"}
    if cin % KS:
        tags.add(f"{kind}_cin_off_slab")
    if any(w % TN for w in widths):
        tags.add(f"{kind}_partial_pass")
    if len(widths) == MAX_LAYERS:
        tags.add(f"{kind}_four_layers")
    if kind == "sa":
        if plan["pieces"] > 1:
            tags.add(f"sa_pieces_tm{tm}")
            if k % tm:
                tags.add("sa_partial_piece")
        if plan["slots"] > 1:
            tags.add(f"sa_groups_tm{tm}")
            if tm % k:
                tags.add("sa_k_ndiv_tm")
        if plan["trimmed"]:
            tags.add(f"sa_trimmed_e{esize}")
    elif rows % tm:
        tags.add("rows_partial_tile")
    return tags


# ---------------------------------------------------------------------------------------------- gather and pool
def sa_rows(xyz, new_xyz, points, idx, xyz_first, use_xyz, fmt):
    """The (B, S, K, cin) float32 rows the kernel's first layer reads: the centred xyz as float32 differences rounded
    once to fmt, then the features (already fmt values), in the kernel's channel order.  idx None: one group of every
    point in order; new_xyz None: zeros."""
    xyz = np.asarray(xyz, np.float32)
    b, n = xyz.shape[:2]
    if idx is None:
        idx = np.broadcast_to(np.arange(n, dtype=np.int64), (b, 1, n))
    idx = np.asarray(idx, np.int64)
    bi = np.arange(b)[:, None, None]
    ctr = np.zeros((b, idx.shape[1], 3), np.float32) if new_xyz is None else np.asarray(new_xyz, np.float32)
    gx = NUM.quantize((xyz[bi, idx] - ctr[:, :, None, :]).astype(np.float32), fmt)
    if points is None:
        return gx
    gp = np.asarray(points, np.float32)[bi, idx]
    if not use_xyz:
        return gp
    return np.concatenate([gx, gp] if xyz_first else [gp, gx], axis=-1)


def max_pool(y, k):
    """(G * k, c) -> (G, c): the maximum of each group's k rows, NaN if any row holds NaN"""
    return np.max(np.asarray(y).reshape(-1, k, y.shape[-1]), axis=1)


# ----------------------------------------------------------------------------------------------- 16-bit bound
def gamma_mma(k):
    t = float(k) * U_MMA
    return t / (1.0 - t)


def bound16(x, layers, affine, fmt, pool_k=None):
    """float64 reference and elementwise bound of the 16-bit kernels.  ``x`` (R, cin): the inputs exactly as the kernel
    reads them (fmt values).  ``affine``: per layer the float32 (scale, shift).  Weights are rounded once to fmt,
    activations are not rounded.  Per layer, with r the reference input and e its bound:

        δacc = |Wq|·e + γ'(K)·|Wq|·(|r| + e)                 (float32 accumulation, unit roundoff U_MMA)
        δy   = |scale|·δacc + u32·(|y| + |scale|·δacc)         (the fmaf epilogue)
        ReLU is 1-Lipschitz; each stored activation adds ½ ulp_fmt at |y| + δy.

    ``pool_k``: the set-abstraction kernel, whose last layer stays float32 until the max over each group of pool_k
    rows, rounded once.  A value that may round past the format's largest finite number gets an infinite bound (the
    kernel may write inf there, and what follows is unconstrained).  Returns (ref, bound) float64."""
    r = np.asarray(x, np.float64)
    e = np.zeros_like(r)
    nl = len(layers)

    def rounding(y, d):
        d = d + 0.5 * NUM.ulp(np.abs(y) + d, fmt)
        return np.where(np.abs(y) + d >= OVERFLOW[fmt], np.inf, d)

    for l, (L, (sc, sh)) in enumerate(zip(layers, affine)):
        wq = NUM.quantize(np.asarray(L["w"], np.float32), fmt).astype(np.float64)
        aw = np.abs(wq).T
        sc, sh = np.asarray(sc, np.float64), np.asarray(sh, np.float64)
        with np.errstate(invalid="ignore", over="ignore"):
            dacc = e @ aw + gamma_mma(wq.shape[1]) * ((np.abs(r) + e) @ aw)
            dacc = np.where(np.isnan(dacc), np.inf, dacc)
            y = (r @ wq.T) * sc + sh
            d = np.abs(sc) * dacc
            d = d + NUM.U32 * (np.abs(y) + d)
        if L.get("relu"):
            y = np.maximum(y, 0.0)  # np.maximum keeps NaN, as the kernel's ReLU does
        if l + 1 < nl or pool_k is None:
            d = rounding(y, d)
        r, e = y, d
    if pool_k is not None:
        r, e = max_pool(r, pool_k), max_pool(e, pool_k)
        e = rounding(r, e)
    return r, e


def check16(got, ref, bound):
    """(every element within its bound, worst |got − ref| / bound over the finite bounds).  NaN in ref must be NaN in
    got; an infinite bound admits anything."""
    got = np.asarray(got, np.float64)
    with np.errstate(invalid="ignore"):
        err = np.abs(got - ref)
        ok = np.isinf(bound) | (err <= bound) | (np.isnan(ref) & np.isnan(got))
        fin = np.isfinite(bound) & np.isfinite(ref)
        ratio = err[fin] / np.maximum(bound[fin], 1e-300)
    return bool(ok.all()), float(ratio.max()) if ratio.size else 0.0


# -------------------------------------------------------------------------------------------------- mutations
MUTATIONS = ("eps", "bias", "swap", "relu")


def mutate(layers, kind):
    """A copy of ``layers`` with one defect a kernel could have, for checking that a comparison catches it:
    "eps" every batch norm with eps 1e-5 instead of its own, "bias" the last layer's largest bias dropped, "relu" the
    first ReLU removed; "swap" leaves the layers alone (see swap_partial_pass)."""
    out = [dict(L) for L in layers]
    if kind == "eps":
        for L in out:
            if "mean" in L:
                L["eps"] = 1e-5
    elif kind == "bias":
        b = np.array(out[-1]["b"], np.float32)
        b[int(np.argmax(np.abs(b)))] = 0
        out[-1]["b"] = b
    elif kind == "relu":
        first = next(l for l, L in enumerate(out) if L.get("relu"))
        out[first]["relu"] = False
    elif kind != "swap":
        raise ValueError(kind)
    return out


def swap_partial_pass(a):
    """``a`` (..., cout) with the first two columns of its last, partial 64-column pass swapped"""
    cout = a.shape[-1]
    lo = cout // TN * TN
    if cout - lo < 2:
        raise ValueError(f"{cout} channels leave no two columns in a partial last pass")
    a = np.array(a, copy=True)
    a[..., [lo, lo + 1]] = a[..., [lo + 1, lo]]
    return a


# ------------------------------------------------------------------------------------- the 16-bit kernel on a CPU
def simulate16(x, layers, affine, fmt, rs, pool_k=None):
    """The 16-bit kernels' arithmetic with a random summation order: products of fmt values (exact in float32) summed
    in float32 in a random order of k, the epilogue y = acc·scale + shift rounded once to float32, ReLU, each stored
    activation rounded to fmt (round to nearest even); with ``pool_k`` the last layer's float32 maxima rounded once.
    Returns float32 values."""
    a = NUM.quantize(np.asarray(x, np.float32), fmt)
    nl = len(layers)
    for l, (L, (sc, sh)) in enumerate(zip(layers, affine)):
        wq = NUM.quantize(np.asarray(L["w"], np.float32), fmt)
        acc = np.zeros((a.shape[0], wq.shape[0]), np.float32)
        for k in rs.permutation(wq.shape[1]):
            acc = (acc + a[:, k:k + 1] * wq[:, k][None, :]).astype(np.float32)
        y = (acc.astype(np.float64) * np.asarray(sc, np.float64) + np.asarray(sh, np.float64)).astype(np.float32)
        if L.get("relu"):
            y = np.where(y < 0, np.float32(0), y)
        a = y if (l + 1 == nl and pool_k is not None) else NUM.quantize(y, fmt)
    if pool_k is not None:
        a = NUM.quantize(max_pool(a, pool_k), fmt)
    return a
