"""A numpy restatement of the host side of csrc/masked_bn.cu: the thread geometry, the workspace layouts, the grids and
the <T, V, VEC> choice of every launch, with the named regimes a call reaches (TEST TOOL, no device).

* ``geom(rows, c)``: mbn_geom.  vec = 4 when c % 4 == 0 else 1; tx = the power of two >= ceil(c / vec), at most 32;
  ty = 256 / tx; col_tiles = ceil(lanes / tx); chunk_rows = 32 * ty; chunks = ceil(rows / chunk_rows).
* ``workspace_bytes`` / ``max_workspace_bytes``: pn2_masked_bn_workspace_bytes / pn2_masked_bn_relu_max_workspace_bytes.
* ``row_blocks(g, rows, sms)``: elementwise_row_blocks, the grid of the normalise and dx kernels.
* ``plain_call`` / ``max_call``: the launches of one forward + backward with their instantiations, grids and
  grid-stride trips, and the regimes the call's geometry and mask reach.

tests/fuzz_masked_bn_gpu.py plans its cases with it; tests/test_fuzz_masked_bn_cpu.py replays the fixed slice
through it and checks that its constants are those of masked_bn.cu."""
from __future__ import annotations

import numpy as np

from fps_regimes import SMS  # the H100's SM count (132), the elementwise grids' cap is planned with it

THREADS = 256      # kMbnThreads
ROWS = 8           # kMbnRows: rows of one register group
GROUPS = 4         # kMbnGroups: groups per thread in a chunk
MERGE_WARPS = 32   # kMbnMergeWarps: warps of a finalize CTA
UNROLL = 4         # kMbnUnroll: rows per thread per step of the elementwise kernels
COL_TILE_LIMIT = 65535
TYPES = {"f32": "float", "bf16": "__nv_bfloat16", "f16": "__half"}
ESIZE = {"f32": 4, "bf16": 2, "f16": 2}


def _cdiv(a, b):
    return -(-a // b)


def geom(rows: int, c: int) -> dict:
    vec = 4 if c % 4 == 0 else 1
    lanes = _cdiv(c, vec)
    tx = 1
    while tx < lanes and tx < 32:
        tx <<= 1
    ty = THREADS // tx
    chunk_rows = ty * ROWS * GROUPS
    return dict(vec=vec, tx=tx, ty=ty, lanes=lanes, col_tiles=_cdiv(lanes, tx), chunk_rows=chunk_rows,
                chunks=_cdiv(rows, chunk_rows) if rows > 0 else 0)


def _a256(v):
    return _cdiv(v, 256) * 256


def layout_bytes(g: dict, c: int) -> int:
    """mbn_layout(g, c).total: two float partials per (chunk, column), an int per chunk, three floats per column"""
    part = _a256(4 * g["chunks"] * c)
    return 2 * part + _a256(4 * g["chunks"]) + _a256(4 * 3 * c)


def max_bwd_bytes(b: int, c: int) -> int:
    return _a256(4 * 3 * c) + _a256(4 * b * c)


def workspace_bytes(rows: int, c: int) -> int:
    if rows <= 0 or c <= 0:
        return 0
    return layout_bytes(geom(rows, c), c)


def max_workspace_bytes(b: int, n: int, c: int) -> int:
    if b <= 0 or n <= 0 or c <= 0 or b * n > 0x7FFFFFFF:
        return 0
    return max(layout_bytes(geom(b * n, c), c), max_bwd_bytes(b, c))


def row_blocks(g: dict, rows: int, sms: int = SMS) -> int:
    """elementwise_row_blocks: CTAs along the rows, at most ~8 per SM over all column tiles"""
    need = _cdiv(rows, g["ty"] * UNROLL)
    cap = sms * 8 // g["col_tiles"] + 1
    return min(need, cap)


def dispatch(g: dict, aligned: bool):
    """dispatch_vec: (V, VEC)"""
    if g["vec"] == 4:
        return 4, bool(aligned)
    return 1, False


def _inst(kernel, fmt, v, vec):
    return f"{kernel}<{TYPES[fmt]},{v},{'true' if vec else 'false'}>"


def _elementwise(kernel, fmt, v, vec, g, rows, sms):
    blocks = row_blocks(g, rows, sms)
    return dict(kernel=_inst(kernel, fmt, v, vec), grid=(blocks, g["col_tiles"]),
                trips=_cdiv(rows, blocks * g["ty"] * UNROLL))


def _geometry_regimes(g: dict, c: int) -> set:
    reg = {f"vec{g['vec']}_tx{g['tx']}"}
    if g["col_tiles"] * g["tx"] > g["lanes"]:
        reg.add("idle_lanes")
    if g["col_tiles"] > 1:
        reg.add("col_tiles_many")
        if g["lanes"] % g["tx"]:
            reg.add("partial_last_tile")
    return reg


def keep_regimes(keep, g: dict) -> set:
    """the merge paths the mask reaches: chunk counts, chunks without a real row, real rows only in late chunks"""
    keep = np.asarray(keep).reshape(-1) != 0
    rows, cr, chunks = keep.size, g["chunk_rows"], g["chunks"]
    reg = set()
    if chunks == 1:
        reg.add("chunks_1")
    if rows == cr:
        reg.add("rows_eq_chunk_rows")
    if chunks in (32, 33):
        reg.add(f"chunks_{chunks}")
    if chunks >= 64 and rows % cr:
        reg.add("chunks_ge_64_remainder")
    real = int(keep.sum())
    if real == rows:
        reg.add("keep_all")
    if real == 0:
        reg.add("keep_none")
    elif real == 1:
        reg.add("keep_one")
    if real and chunks > 1:
        per_chunk = np.add.reduceat(keep, np.arange(0, rows, cr)) if rows else np.zeros(0)
        if (per_chunk == 0).any():
            reg.add("empty_chunk")
        if per_chunk[0] == 0:
            reg.add("late_rows_only")  # the merges start from an empty partial (na == 0)
    return reg


def plain_call(fmt: str, rows: int, c: int, keep, aligned_fwd: bool, aligned_bwd: bool, sms: int = SMS) -> dict:
    """forward + backward of pn2_masked_bn_relu_{forward,backward}_typed"""
    g = geom(rows, c)
    vf, vecf = dispatch(g, aligned_fwd)
    vb, vecb = dispatch(g, aligned_bwd)
    launches = [
        dict(kernel=_inst("mbn_stats_kernel", fmt, vf, vecf), grid=(g["chunks"], g["col_tiles"]), trips=1),
        dict(kernel="mbn_finalize_kernel", grid=(_cdiv(c, 32), 1), trips=1),
        _elementwise("mbn_norm_relu_kernel", fmt, vf, vecf, g, rows, sms),
        dict(kernel=_inst("mbn_bwd_sums_kernel", fmt, vb, vecb), grid=(g["chunks"], g["col_tiles"]), trips=1),
        dict(kernel="mbn_bwd_finalize_kernel", grid=(_cdiv(c, 32), 1), trips=1),
        _elementwise("mbn_bwd_dx_kernel", fmt, vb, vecb, g, rows, sms),
    ]
    return dict(geom=g, launches=launches, regimes=_geometry_regimes(g, c) | keep_regimes(keep, g))


def max_call(fmt: str, b: int, n: int, c: int, keep, aligned_fwd: bool, aligned_bwd: bool, sms: int = SMS) -> dict:
    """forward + backward of pn2_masked_bn_relu_max_{forward,backward}_typed"""
    rows = b * n
    g = geom(rows, c)
    vf, vecf = dispatch(g, aligned_fwd)
    vb, vecb = dispatch(g, aligned_bwd)
    launches = [
        dict(kernel=_inst("mbn_stats_kernel", fmt, vf, vecf), grid=(g["chunks"], g["col_tiles"]), trips=1),
        dict(kernel="mbn_finalize_kernel", grid=(_cdiv(c, 32), 1), trips=1),
        dict(kernel=_inst("mbn_norm_relu_max_kernel", fmt, vf, vecf), grid=(b, g["col_tiles"]),
             trips=_cdiv(n, g["ty"] * UNROLL)),
        dict(kernel=f"mbn_max_bwd_finalize_kernel<{TYPES[fmt]}>", grid=(_cdiv(c, 32), 1),
             trips=_cdiv(b, MERGE_WARPS)),
        _elementwise("mbn_max_bwd_dx_kernel", fmt, vb, vecb, g, rows, sms),
    ]
    reg = _geometry_regimes(g, c) | keep_regimes(keep, g)
    k = np.asarray(keep).reshape(b, n) != 0
    if b in (1, 31, 32, 33, 70):
        reg.add(f"max_b{b}")
    if b > MERGE_WARPS and b % MERGE_WARPS:
        reg.add("max_ragged_last_pass")
    if n < g["ty"]:
        reg.add("max_n_lt_ty")
    if n > 2 * UNROLL * g["ty"]:
        reg.add("max_row_trips_3_plus")
    if (~k.any(1)).any():
        reg.add("max_empty_cloud")
    return dict(geom=g, launches=launches, regimes=reg)


def thread_of_row(j: int, g: dict) -> int:
    """the thread row (threadIdx.y) of mbn_norm_relu_max_kernel that walks row j of a cloud"""
    return j % g["ty"]


def instances() -> list:
    """every <T, V, VEC> instantiation the entry points can launch"""
    out = []
    for fmt in TYPES:
        for v, vec in ((1, False), (4, False), (4, True)):
            for k in ("mbn_stats_kernel", "mbn_norm_relu_kernel", "mbn_norm_relu_max_kernel", "mbn_bwd_sums_kernel",
                      "mbn_bwd_dx_kernel", "mbn_max_bwd_dx_kernel"):
                out.append(_inst(k, fmt, v, vec))
        out.append(f"mbn_max_bwd_finalize_kernel<{TYPES[fmt]}>")
    return out + ["mbn_finalize_kernel", "mbn_bwd_finalize_kernel"]
