"""A numpy restatement of the seeded row selection shared by the samplers (pn2_common.cuh cta_select_sorted) and of
the host side of csrc/voxel.cu, shapes.cu, crops.cu and vscan.cu: launch plans, workspace sizes and refusals (TEST
TOOL, no device).

* ``select_trace(keys, m)``: cta_select_sorted over distinct 64-bit orders, step by step: whether a radix select ran,
  the digits and the prefix, the pass at which the boundary bucket was taken whole, the gathered keys, the bitonic
  sort of pow2_at_least(m) of them (padded with ~0) and its first m.
* ``boundary_pass(keys, m)``: the pass the select finishes at, from the m-th and (m+1)-th smallest orders alone.
* ``voxel_plan`` / ``shapes_plan``: per cell or entry the path, key width, m and whether a select runs; the grids and
  dynamic shared memory of the select launches.  ``edge_regimes``: the c / m edges of one select call.
* ``*_refusal``: the host checks of each entry point, as the reason a call is refused (None when it is accepted).
* ``collisions`` / ``PLANTED``: rows whose rng_row_key high halves collide, for the select's passes 3 to 5.

tests/fuzz_samplers_gpu.py plans its cases with it; tests/test_fuzz_samplers_cpu.py replays the fixed slice through
it and checks that its constants are those of the .cu sources."""
from __future__ import annotations

import numpy as np

from crop_oracle import draw
from fps_regimes import SMS  # the H100's SM count (132): voxel_cta_kernel's grid is capped at 2 per SM

SELECT_THREADS = 1024  # every select CTA: crops / vscan kSelectThreads, shapes kShapeThreads, voxel kCtaThreads
RADIX_BINS = 2048      # kSelectRadixBins
MAX_ROWS = 16384       # kSelectMaxRows
WARP_KEYS = 4          # voxel.cu kWarpKeys
WARP_CELL = 32 * WARP_KEYS
ROW_THREADS = WARP_THREADS = 256
SCAN_MAX_BATCH = 4096  # vscan.cu kScanMaxBatch
CROP_MAX_BATCH = 65535
# the rng_row_key stream of each sampler
STREAM = {"crops": 2, "shapes": 1, "vscan": 4, "voxel": 9}
# digit widths of the six passes: 11, 11, 10 bits over the high half of an order, then over the low half
WIDTHS = (11, 11, 10, 11, 11, 10)
M64 = (1 << 64) - 1
I31 = 1 << 31
U64 = np.uint64


def pow2_at_least(n: int) -> int:
    p = 1
    while p < n:
        p <<= 1
    return p


def row_keys(seed: int, stream: int, e: int, rows) -> np.ndarray:
    """rng_row_key: (draw(seed, stream, e, j) >> 32 << 32) | j as uint64"""
    rows = np.asarray(rows, np.int64).astype(U64)
    return (draw(seed & M64, stream, e, rows) >> U64(32) << U64(32)) | rows


def _bitonic(a: np.ndarray) -> np.ndarray:
    """the CTA's bitonic network over a power-of-two buffer, stage by stage"""
    a = a.copy()
    n = len(a)
    i = np.arange(n)
    k = 2
    while k <= n:
        h = k >> 1
        while h > 0:
            p = i ^ h
            lo = i[p > i]
            hi = lo ^ h
            x, y = a[lo], a[hi]
            swap = (x > y) == ((lo & k) == 0)
            a[lo[swap]], a[hi[swap]] = y[swap], x[swap]
            h >>= 1
        k <<= 1
    return a


def select_trace(keys, m: int) -> dict:
    """cta_select_sorted over the member orders ``keys`` (distinct uint64, any order; c = len(keys) >= m) for m rows.
    ``select``: a radix select ran (c > m); ``pass``: the pass (0..5) at which the boundary bucket was taken whole,
    None without a select; ``digits``; ``prefix`` and ``bits``; ``gathered``: how many orders the gather kept (m
    unless the select is wrong); ``sort_n``; ``out``: the first m of the sorted buffer."""
    keys = np.asarray(keys, U64)
    c = len(keys)
    assert c >= m >= 0 and len(np.unique(keys)) == c
    prefix, bits, fin, digits = M64, 0, None, []
    if c > m:
        prefix, need = 0, m
        for ps in range(6):
            wd = WIDTHS[ps]
            shift = 64 - bits - wd
            sel = keys if not bits else keys[(keys >> U64(64 - bits)) == U64(prefix)]
            d = ((sel >> U64(shift)) & U64((1 << wd) - 1)).astype(np.int64)
            hist = np.bincount(d, minlength=RADIX_BINS)
            cum = np.cumsum(hist)
            digit = int(np.searchsorted(cum, need))  # the first bin whose inclusive sum reaches need
            before, cnt = int(cum[digit] - hist[digit]), int(hist[digit])
            need -= before
            prefix = (prefix << wd) | digit
            bits += wd
            digits.append(digit)
            if cnt == need:
                fin = ps
                break
    kept = keys if not bits else keys[(keys >> U64(64 - bits)) <= U64(prefix)]
    sort_n = pow2_at_least(m)
    buf = np.full(max(sort_n, len(kept)), M64, U64)
    buf[:len(kept)] = kept
    srt = _bitonic(buf[:sort_n]) if len(kept) <= sort_n else np.sort(kept)
    return {"select": c > m, "pass": fin, "digits": digits, "prefix": prefix if bits else None, "bits": bits,
            "gathered": len(kept), "sort_n": sort_n, "out": srt[:m]}


def boundary_pass(keys, m: int):
    """the pass cta_select_sorted finishes at: the one holding the highest bit in which the m-th and (m+1)-th smallest
    orders differ (None when no select runs)"""
    keys = np.sort(np.asarray(keys, U64))
    if len(keys) <= m:
        return None
    top = (int(keys[m - 1]) ^ int(keys[m])).bit_length() - 1  # m >= 1 here
    used = 0
    for ps, wd in enumerate(WIDTHS):
        used += wd
        if top >= 64 - used:
            return ps
    raise AssertionError("distinct orders differ somewhere")


def collisions(seed: int, stream: int, e: int, lo: int, count: int):
    """(j1 < j2) pairs among rows lo .. lo + count - 1 whose rng_row_key high halves are equal: a birthday search"""
    j = np.arange(lo, lo + count, dtype=np.int64).astype(U64)
    h = draw(seed & M64, stream, e, j) >> U64(32)
    o = np.argsort(h, kind="stable")
    hs = h[o]
    d = np.nonzero(hs[1:] == hs[:-1])[0]
    return [(int(min(j[o[k]], j[o[k + 1]])), int(max(j[o[k]], j[o[k + 1]]))) for k in d]


def pair_pass(j1: int, j2: int) -> int:
    """the pass at which a select whose boundary splits two rows with equal high halves finishes"""
    return boundary_pass(np.array([(1 << 32) | j1, (1 << 32) | j2], U64), 1)


# Rows whose rng_row_key high halves collide, found by collisions(): (seed, entry, j1, j2) per finishing pass.
# voxel (stream 9): rows around 2^21 (lo = 2^21 - 2^19, 2^20 rows), entries of a 3^3 grid's cloud 0;
# shapes (stream 1): rows below 16384, entry e of a batch.
VOXEL_WINDOW = ((1 << 21) - (1 << 19), 1 << 20)
PLANTED = {
    ("voxel", 3): (7, 0, 2019872, 2283615),
    ("voxel", 4): (7, 0, 1711416, 1846551),
    ("voxel", 5): (7, 11, 2289351, 2289488),
    ("shapes", 4): (0, 8, 1174, 2154),
    ("shapes", 5): (4, 15, 14608, 15333),
}


# ----------------------------------------------------------------------------------------------------- voxel.cu
def voxel_cells(b: int, n: int, dim: int, dims: int) -> int:
    if b < 1 or n < 1 or dim < 1 or dims not in (2, 3) or b * n >= I31:
        return 0
    if dim > (46340 if dims == 2 else 1290):
        return 0
    cells = dim ** dims
    return cells if cells * b < I31 else 0


def _a256(v: int) -> int:
    return -(-v // 256) * 256


def voxel_layout(b: int, n: int, cells: int) -> dict:
    big_cap = b * min(cells, n // (WARP_CELL + 1))
    off = 0
    out = {}
    for name, size in (("cursor", 4 * b * cells), ("member", 4 * b * n), ("big", 4 * big_cap), ("nbig", 4)):
        out[name] = off
        off = _a256(off + size)
    out.update(total=off, big_cap=big_cap)
    return out


def voxel_workspace_bytes(b: int, n: int, dim: int, dims: int) -> int:
    cells = voxel_cells(b, n, dim, dims)
    return voxel_layout(b, n, cells)["total"] if cells else 0


def voxel_refusal(b, n, dim, dims, radius, nsample, ws_bytes, ws_aligned=True):
    cells = voxel_cells(b, n, dim, dims)
    if not cells:
        return "shape"
    if not 1 <= nsample <= MAX_ROWS:
        return "nsample"
    rf, vf = np.float32(radius), np.float32(2.0 * radius / dim)
    if not (radius > 0 and rf > 0 and vf > 0 and np.isfinite(rf) and np.isfinite(2.0 * radius / dim)):
        return "radius"
    if ws_bytes < voxel_layout(b, n, cells)["total"] or not ws_aligned:
        return "workspace"
    return None


def voxel_plan(count: np.ndarray, n: int, nsample: int, sms: int = SMS) -> dict:
    """the launches of pn2_voxel_group for the per-cell counts (B, C) of a call; per cell: path (empty / warp / cta),
    warp key width, CTA key type and whether the CTA cell runs a select"""
    count = np.asarray(count, np.int64)
    b, cells = count.shape
    L = voxel_layout(b, n, cells)
    c = count.reshape(-1)
    big = np.nonzero(c > WARP_CELL)[0]
    width = np.where(c <= 32, 1, np.where(c <= 64, 2, 4))
    cta_grid = min(L["big_cap"], 2 * sms)
    reg = set()
    for w in (1, 2, 4):
        if ((c > 0) & (c <= WARP_CELL) & (width == w)).any():
            reg.add(f"voxel_warp_w{w}")
    warp = c[(c > 0) & (c <= WARP_CELL)]
    if (warp > nsample).any():
        reg.add("voxel_warp_seeded")
    if (warp <= nsample).any():
        reg.add("voxel_warp_rows")
    if (c == 0).any():
        reg.add("voxel_empty_cell")
    for v in (1, 31, 32, 33, 64, 65, 127, 128):
        if (c == v).any():
            reg.add(f"voxel_c{v}")
    if len(big):
        reg.add("voxel_cta")
        if (c[big] > nsample).any():
            reg.add("voxel_cta_seeded")
        if (c[big] <= nsample).any():
            reg.add("voxel_cta_rows")
        if len(big) > cta_grid:
            reg.add("voxel_cta_reuse")  # a CTA serves several listed cells
    if L["big_cap"] == 0:
        reg.add("voxel_no_cta_launch")
    if nsample % 32:
        reg.add("voxel_s_not_x32")
    return {"cells": cells, "big_cap": L["big_cap"], "cta_grid": cta_grid, "nbig": len(big), "width": width,
            "path": np.where(c == 0, "empty", np.where(c <= WARP_CELL, "warp", "cta")),
            "smem": 8 * pow2_at_least(nsample), "launches": 4 + (L["big_cap"] > 0), "regimes": reg,
            "selects": [(int(e), int(c[e]), nsample) for e in big if c[e] > nsample]}


# ---------------------------------------------------------------------------------------------------- shapes.cu
def shapes_refusal(max_shape, b, votes, npoints, with_normals, subset_random=0):
    if max_shape < 1 or max_shape > MAX_ROWS or b < 1 or votes < 0 or not 1 <= npoints <= MAX_ROWS:
        return "shape"
    ent = votes * b if votes else b
    if ent > 0x7FFFFFFF or ent * npoints * (6 if with_normals else 3) >= I31:
        return "entries"
    if votes and subset_random:
        return "vote_options"
    return None


def shapes_plan(sizes, shape_idx, npoints: int, subset_random: bool, votes: int) -> dict:
    """per entry (pool q, m, select); the kernel's dynamic shared memory"""
    sizes = np.asarray(sizes, np.int64)
    idx = np.asarray(shape_idx, np.int64)
    max_shape = int(sizes.max())
    pool = max_shape if subset_random else min(max_shape, npoints)
    ent = []
    for e in range(len(idx) * votes if votes else len(idx)):
        s = int(idx[e % len(idx)])
        ps = int(sizes[s]) if 0 <= s < len(sizes) else 0
        q = ps if (subset_random and not votes) else min(ps, npoints)
        ent.append((q, min(q, npoints), q > min(q, npoints)))
    return {"entries": ent, "pool": pool, "smem": 8 * pow2_at_least(min(pool, npoints))}


# ------------------------------------------------------------------------------------------- crops.cu, vscan.cu
KEY_WORDS, ATTEMPTS = 1986, 10


def crops_workspace_bytes(b: int, npoints: int) -> int:
    if not (1 <= b <= CROP_MAX_BATCH and 1 <= npoints <= MAX_ROWS and b * npoints * 3 < I31):
        return 0
    return _a256(b * (ATTEMPTS * 2 + ATTEMPTS * KEY_WORDS) * 4)


def crops_refusal(b, npoints, ws_bytes, ws_aligned=True, max_dropout=0.0):
    if not (1 <= b <= CROP_MAX_BATCH and 1 <= npoints <= MAX_ROWS and b * npoints * 3 < I31):
        return "shape"
    if not 0.0 <= max_dropout <= 1.0:
        return "dropout"
    if ws_bytes < crops_workspace_bytes(b, npoints) or not ws_aligned:
        return "workspace"
    return None


RAYS, CELLS = 200 * 150, 634 * 159


def vscan_workspace_bytes(b: int, max_scene: int, npoints: int) -> int:
    if not (1 <= b <= SCAN_MAX_BATCH and 1 <= max_scene < 0x7FFFFFFF and 1 <= npoints <= MAX_ROWS
            and b * npoints * 3 < I31):
        return 0
    words = (max_scene + 31) // 32
    zero = _a256(4 * (b * 4 + b * CELLS + b * words))
    return zero + 4 * _a256(8 * b * RAYS) + _a256(4 * b * RAYS) + _a256(8 * b * RAYS)


def vscan_refusal(b, max_scene, npoints, ws_bytes, ws_aligned=True, min_points=0):
    if vscan_workspace_bytes(b, max_scene, npoints) == 0 or min_points < 0:
        return "shape"
    if ws_bytes < vscan_workspace_bytes(b, max_scene, npoints) or not ws_aligned:
        return "workspace"
    return None


def edge_regimes(c: int, m: int, prefix: str) -> set:
    """the c / m edges of one select call"""
    reg = set()
    if c == m:
        reg.add(prefix + "_c_eq_m")
    if c == m + 1:
        reg.add(prefix + "_c_eq_m_plus_1")
    if m == 1 and c > 1:
        reg.add(prefix + "_m1")
    if m == MAX_ROWS:
        reg.add(prefix + "_m_max")
    if m > 1 and m & (m - 1) == 0:
        reg.add(prefix + "_m_pow2")
    if m > 2 and (m - 1) & (m - 2) == 0:
        reg.add(prefix + "_m_pow2_plus_1")
    if m > 1024:
        reg.add(prefix + "_compact_over_1024")
    return reg
