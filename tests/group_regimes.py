"""The host side of group.cu, interpolate.cu and scatter_det.cu restated in numpy (no device): which kernel
instantiation each entry launches, with what grid, how many grid-stride trips it takes and which tail state it
reaches; and the exact float32 association of the ordered (atomic-free) gradient sums.

tests/fuzz_group_gpu.py runs the kernels against the C oracle and these sums; tests/test_fuzz_group_cpu.py replays
its fixed slice through this module, requires every instantiation and regime below, and checks the lists here
against the launch sites of the three .cu files.

Names: an instantiation is written ``kernel<args>`` with the template arguments as in the source, ``u16`` for the
2-byte features moved as unsigned short, ``bf16`` / ``f16`` for __nv_bfloat16 / __half, ``u32`` / ``u64`` for the
index types.  A plan is a list of launches, each a dict with ``kernel``, ``grid`` (x, y) and ``trips`` (the most
grid-stride trips any thread takes) and the regimes (strings) the call reaches.
"""
from __future__ import annotations

import numpy as np

from fps_regimes import SMS  # the H100's SM count (132)

COPY_THREADS = 256   # kCopyThreads (group.cu)
IT_THREADS = 256     # kItThreads (interpolate.cu)
NN_THREADS = 128     # kNnThreads
INV_THREADS = 256    # kInvThreads (scatter_det.cu)
SORT_CAP = 256       # kInvSortCap: lists up to this length are sorted in registers by one warp
BUILD_MAX_M = 16000  # kInvBuildMaxM: the one-CTA build keeps nt + 1 counters in shared memory
SEQ_SCAN = 8         # kSeqScan
SEQ_BUF = 2 * SEQ_SCAN * INV_THREADS  # kSeqBuf: 4096 buffered entries
PIECES = INV_THREADS // 32            # inv_long_kernel: one piece per warp
ESIZE = {"f32": 4, "bf16": 2, "f16": 2}
TNAME = {"f32": "float", "bf16": "u16", "f16": "u16"}          # group.cu / scatter_det.cu: 2-byte formats share a T
TNAME3 = {"f32": "float", "bf16": "bf16", "f16": "f16"}        # interpolate.cu / atomic gradients: one T per format
LARGE = "reached only by test_large_index_gpu.py / the beyond-2^31 tests in test_half_features_gpu.py"
UNUSED = "compiled, never launched: the narrow kernel takes every row of at most 4 elements"


def _cdiv(a, b):
    return -(-int(a) // int(b))


def grid_for(work, per_block):
    """pn2_common.cuh grid_for: ceil(work / per_block), at most SMS * 64, at least 1"""
    return max(1, min(_cdiv(work, per_block), SMS * 64))


def _trips(work, per_trip):
    return max(1, _cdiv(work, per_trip))


# ---------------------------------------------------------------------------------------------- instantiations
def _instances():
    """{name: note} of every kernel instantiation in the three files (note None: reachable by the fuzz)"""
    inst = {"gather_point_kernel": None, "gather_point_grad_kernel": None, "selection_sort_kernel": None,
            "group_point_vec4_kernel<u32>": None, "group_point_vec4_kernel<u64>": LARGE}
    for lpr in (4, 8, 16, 32):
        inst[f"group_rows_vec4_kernel<{lpr},4>"] = None
        for t in ("float", "u16"):
            inst[f"group_rows_kernel<{lpr},true,{t}>"] = None
            inst[f"group_rows_kernel<{lpr},false,{t}>"] = UNUSED if lpr == 4 else None
    for lpr in (8, 16):
        inst[f"group_concat_vec_kernel<{lpr},2>"] = None
    for h in ("true", "false"):
        for t in ("float", "u16"):
            inst[f"group_narrow_kernel<{h},{t}>"] = None
    for t in ("float", "bf16", "f16"):
        for ix in ("u32", "u64"):
            note = LARGE if ix == "u64" else None
            inst[f"group_point_grad_vec4_kernel<{ix},{t}>"] = note
            inst[f"group_point_grad_scalar_kernel<{ix},{t}>"] = note
            for lv in ("false", "true"):
                inst[f"three_interp_vec4_kernel<{ix},{t},{lv}>"] = note
                inst[f"three_interp_scalar_kernel<{ix},{t},{lv}>"] = note
    for t in ("bf16", "f16"):
        inst[f"round_to_kernel<{t}>"] = None
    for ix in ("u32", "u64"):
        for lv in ("false", "true"):
            inst[f"three_interp_grad_vec4_kernel<{ix},{lv}>"] = LARGE if ix == "u64" else None
            inst[f"three_interp_grad_scalar_kernel<{ix},{lv}>"] = LARGE if ix == "u64" else None
    for g in (1, 2, 4, 8, 16, 32):
        for t in ("float", "u16"):
            for lv in ("false", "true"):
                inst[f"fp_front_kernel<{g},{t},{lv}>"] = None
    inst["inv_scan_kernel"] = None
    for lv in ("false", "true"):
        inst[f"inv_count_kernel<{lv}>"] = None
        inst[f"inv_fill_kernel<{lv}>"] = None
        inst[f"inv_build_kernel<{lv}>"] = None
    for v in ("true", "false"):
        for t in ("float", "u16"):
            for wtd in ("true", "false"):
                inst[f"inv_gather_kernel<{v},{wtd},{t}>"] = None
            inst[f"inv_long_seq_kernel<{v},{t}>"] = None
            for lv in ("false", "true"):
                inst[f"inv_long_kernel<{v},{t},{lv}>"] = None
    return inst


INSTANCES = _instances()
REACHABLE = sorted(k for k, v in INSTANCES.items() if v is None)


def _aligned(offset_elems, esize, bytes_):
    """a buffer whose data starts ``offset_elems`` elements past a 256-byte aligned allocation"""
    return (offset_elems * esize) % bytes_ == 0


# --------------------------------------------------------------------------------------------------- group_point
def launch_group_rows(has_xyz, b, c, m, s, fmt, aligned16):
    """launch_group_rows<HAS_XYZ, T>: the narrow kernel, the vectorised concat kernel or the LPR row kernel"""
    rpc = m * s
    w = c + (3 if has_xyz else 0)
    t = TNAME[fmt]
    hx = "true" if has_xyz else "false"
    if w <= 4 and (not has_xyz or c == 0):
        cap = _cdiv(SMS * 16, b)
        gx = min(_cdiv(rpc, COPY_THREADS), cap)
        return dict(kernel=f"group_narrow_kernel<{hx},{t}>", grid=(gx, b), trips=_trips(rpc, gx * COPY_THREADS),
                    regimes=[f"narrow_c{c}"])
    if fmt == "f32" and has_xyz and 8 <= c <= 64 and c % 4 == 0 and aligned16:
        c4 = c // 4
        lpr = 8 if c4 <= 8 else 16
        per_trip_rows = (COPY_THREADS // 32) * (32 // lpr) * 2
        cap = _cdiv(SMS * 32, b)
        gx = max(1, min(_cdiv(rpc, per_trip_rows), cap))
        return dict(kernel=f"group_concat_vec_kernel<{lpr},2>", grid=(gx, b), trips=_trips(rpc, gx * per_trip_rows),
                    lpr=lpr, c4=c4, regimes=[])
    lpr = 4 if w <= 4 else 8 if w <= 8 else 16 if w <= 16 else 32
    per_trip_rows = (COPY_THREADS // 32) * (32 // lpr) * 2
    cap = _cdiv(SMS * 32, b)
    gx = max(1, min(_cdiv(rpc, per_trip_rows), cap))
    u = 16 // ESIZE[fmt]
    return dict(kernel=f"group_rows_kernel<{lpr},{hx},{t}>", grid=(gx, b), trips=_trips(rpc, gx * per_trip_rows),
                regimes=[f"rows_channel_steps_{min(_cdiv(c, lpr * u), 2)}" if c else "rows_no_features"])


def group_point_impl(b, n, c, m, s, fmt, points_off=0, out_off=0, mode=0, ctas=16):
    """group_point_impl<T>: (launch or None, refusal) for the typed entry with buffers offset by whole elements"""
    e = ESIZE[fmt]
    rpc, rows = m * s, b * m * s
    if b * m * s * c == 0:
        return None, False
    if (c * e) % 16 == 0 and _aligned(points_off, e, 16) and _aligned(out_off, e, 16):
        c4 = c * e // 16
        tv = rows * c4
        if mode == 0 and rpc < 2 ** 32 and b <= 65535:
            lpr = 4 if c4 <= 4 else 8 if c4 <= 8 else 16 if c4 <= 16 else 32
            per_trip_rows = (COPY_THREADS // 32) * (32 // lpr) * 4
            cap = _cdiv(SMS * ctas, b)
            gx = max(1, min(_cdiv(rpc, per_trip_rows), cap))
            return dict(kernel=f"group_rows_vec4_kernel<{lpr},4>", grid=(gx, b),
                        trips=_trips(rpc, gx * per_trip_rows), lpr=lpr, c4=c4,
                        regimes=[f"vec4_channel_steps_{min(_cdiv(c4, lpr), 2)}", f"vec4_rows_mod4_{rpc % 4}"]), False
        grid = max(1, min(_cdiv(tv, COPY_THREADS), SMS * ctas))
        ix = "u32" if tv < 2 ** 31 else "u64"
        return dict(kernel=f"group_point_vec4_kernel<{ix}>", grid=(grid, 1), trips=_trips(tv, grid * COPY_THREADS),
                    regimes=["flat_b_over_65535" if b > 65535 else "flat_mode1"]), False
    if rpc >= 2 ** 32 or b > 65535:
        return None, True
    return launch_group_rows(False, b, c, m, s, fmt, False), False


def group_concat_impl(b, n, c, m, s, fmt, points_off=0, out_off=0):
    """group_concat_impl<T>: (launch or None, refusal)"""
    if b * m * s == 0:
        return None, False
    if b > 65535:
        return None, True
    e = ESIZE[fmt]
    al = c == 0 or (_aligned(points_off, e, 16) and _aligned(out_off, e, 16))
    return launch_group_rows(True, b, c, m, s, fmt, al), False


def concat_heads(c, m, s, b, xyz_first, out_off=0):
    """the `head` values (0..3) group_concat_vec_kernel's rows take: 4 - ((row * (c + 3) + feat_lo) mod 4) mod 4"""
    rows = np.arange(b * m * s, dtype=np.int64)
    feat_lo = 3 if xyz_first else 0
    return sorted(set(((4 - ((rows * (c + 3) + feat_lo + out_off) & 3)) & 3).tolist()))


# ------------------------------------------------------------------------------------------- atomic gradients
def group_point_grad_impl(b, n, c, m, s, fmt, go_off=0, acc_off=0):
    """group_point_grad_impl<T> (+ the rounding pass over the (b, n, c) accumulator for the 2-byte formats)"""
    total = b * m * s * c
    t = TNAME3[fmt]
    e = ESIZE[fmt]
    if c % 4 == 0 and _aligned(go_off, e, 4 * e) and _aligned(acc_off, 4, 16):
        tv = total // 4
        g = grid_for(tv, COPY_THREADS)
        out = [dict(kernel=f"group_point_grad_vec4_kernel<u32,{t}>", grid=(g, 1), trips=_trips(tv, g * COPY_THREADS))]
    else:
        g = grid_for(total, COPY_THREADS)
        out = [dict(kernel=f"group_point_grad_scalar_kernel<u32,{t}>", grid=(g, 1),
                    trips=_trips(total, g * COPY_THREADS))]
    if fmt != "f32":
        g = grid_for(b * n * c, COPY_THREADS)
        out.append(dict(kernel=f"round_to_kernel<{t}>", grid=(g, 1), trips=_trips(b * n * c, g * COPY_THREADS)))
    return out


def gather_point(b, m, grad=False):
    g = grid_for(b * m, COPY_THREADS)
    k = "gather_point_grad_kernel" if grad else "gather_point_kernel"
    return dict(kernel=k, grid=(g, 1), trips=_trips(b * m, g * COPY_THREADS))


def three_interpolate_launch(b, m, c, n, fmt, ragged, points_off=0, out_off=0):
    """three_interpolate_launch<T, L>"""
    e = ESIZE[fmt]
    total = b * n * c
    lv = "true" if ragged else "false"
    t = TNAME3[fmt]
    if c % 4 == 0 and _aligned(points_off, e, 4 * e) and _aligned(out_off, e, 4 * e):
        tv = total // 4
        g = grid_for(tv, IT_THREADS)
        return dict(kernel=f"three_interp_vec4_kernel<u32,{t},{lv}>", grid=(g, 1), trips=_trips(tv, g * IT_THREADS))
    g = grid_for(total, IT_THREADS)
    return dict(kernel=f"three_interp_scalar_kernel<u32,{t},{lv}>", grid=(g, 1), trips=_trips(total, g * IT_THREADS))


def three_interpolate_grad_atomic(b, n, c, ragged, go_off=0, acc_off=0):
    total = b * n * c
    lv = "true" if ragged else "false"
    if c % 4 == 0 and _aligned(go_off, 4, 16) and _aligned(acc_off, 4, 16):
        g = grid_for(total // 4, IT_THREADS)
        return dict(kernel=f"three_interp_grad_vec4_kernel<u32,{lv}>", grid=(g, 1), trips=_trips(total // 4, g * IT_THREADS))
    g = grid_for(total, IT_THREADS)
    return dict(kernel=f"three_interp_grad_scalar_kernel<u32,{lv}>", grid=(g, 1), trips=_trips(total, g * IT_THREADS))


def fp_front_launch(b, n, m, fmt, ragged):
    """fp_front_dispatch<T>: fp_front_kernel<G, T, L>, one CTA per 128 / G unknown points of each cloud"""
    g = fp_front_g(b, n, m)
    ppb = NN_THREADS // g
    return dict(kernel=f"fp_front_kernel<{g},{TNAME[fmt]},{'true' if ragged else 'false'}>",
                grid=(_cdiv(n, ppb), b), trips=1, g=g)


def fp_front_g(b, n, m):
    """fp_front_dispatch's lanes per unknown point"""
    g = 1
    while g < 32 and b * n * g < 2 * SMS * NN_THREADS and 2 * g <= (m + 1) // 2:
        g *= 2
    return g


# ------------------------------------------------------------------------------------------- ordered gradients
def inv_workspace_bytes(b, ne, nt):
    longs = b * (ne // (SORT_CAP + 1) + 1)
    return 4 * (b * (nt + 1) + b * nt + b * ne + 1 + longs)


def bucket(length):
    """inv_gather_kernel's bitonic register bucket for a list of `length` <= 256 entries"""
    nreg = _cdiv(length, 32)
    return 1 if nreg <= 1 else 2 if nreg == 2 else 4 if nreg <= 4 else 8


def inv_scatter_det(weighted, b, nt, c, fmt, counts, ragged=False, go_off=0, gp_off=0, idx=None):
    """inv_scatter_det<WEIGHTED, T>: the launches and regimes of one call.  counts (b, nt): each target's list length
    (the real entries only); idx (b, ne): the entries' targets, for the buffer flushes of the unweighted long lists."""
    e = ESIZE[fmt]
    t = TNAME[fmt]
    lv = "true" if ragged else "false"
    counts = np.asarray(counts).reshape(b, nt)
    regimes, launches = set(), []
    if nt <= BUILD_MAX_M:
        launches.append(f"inv_build_kernel<{lv}>")
        regimes.add("build_one_cta")
    else:
        launches += [f"inv_count_kernel<{lv}>", "inv_scan_kernel", f"inv_fill_kernel<{lv}>"]
        regimes.add("build_count_scan_fill")
    # both builds scan the nt + 1 offsets in chunks of 1024: one chunk, a boundary crossed, or many
    regimes.add(f"offsets_chunks_{min(_cdiv(nt + 1, 1024), 3)}")
    vec = c % 4 == 0 and _aligned(go_off, e, 4 * e) and _aligned(gp_off, e, 4 * e)
    v = "true" if vec else "false"
    launches.append(f"inv_gather_kernel<{v},{'true' if weighted else 'false'},{t}>")
    W = 4 if vec else 1
    short = counts[counts <= SORT_CAP]
    for L in np.unique(short):
        regimes.add(f"bucket_{bucket(int(L))}" if L > 0 else "empty_list")
    regimes.add(f"gather_channel_passes_{min(_cdiv(c, 32 * W), 3)}")
    longs = counts[counts > SORT_CAP]
    if weighted:
        launches.append(f"inv_long_kernel<{v},{t},{lv}>")
        if len(longs):
            regimes.add("long_weighted")
            regimes.add(f"long_channel_passes_{min(_cdiv(c, 32 * W), 3)}")
    else:
        launches.append(f"inv_long_seq_kernel<{v},{t}>")
        if len(longs):
            regimes.add("long_seq")
            regimes.add(f"seq_channel_passes_{min(_cdiv(c, INV_THREADS * W), 2)}")
            # a flush when the buffer cannot take another step: cnt > SEQ_BUF - SEQ_SCAN * INV_THREADS = 2048
            for k, i in zip(*np.nonzero(counts > SORT_CAP)):
                f = seq_flushes(np.flatnonzero(idx[k] == i), idx.shape[1])
                regimes.add(f"seq_flushes_{min(f, 3)}")
    return dict(launches=launches, vec=vec, regimes=sorted(regimes), long_lists=int(len(longs)))


def seq_flushes(positions, ne):
    """buffer flushes of inv_long_seq_kernel for a list whose entries sit at `positions` of the cloud's `ne`: the fill
    loop takes steps of SEQ_SCAN * INV_THREADS entries while at most SEQ_BUF - SEQ_SCAN * INV_THREADS are buffered"""
    step = SEQ_SCAN * INV_THREADS
    per_step = np.bincount(np.asarray(positions) // step, minlength=_cdiv(ne, step))
    flushes, cnt = 0, 0
    for k in per_step:
        cnt += int(k)
        if cnt > SEQ_BUF - step:
            flushes, cnt = flushes + 1, 0
    return flushes + (1 if cnt or not flushes else 0)


# --------------------------------------------------------------------------------------- exact ordered sums
def ordered_sum(src, idx, nt, weight=None, long_pieces=True, cut=None):
    """The float32 result of inv_scatter_det, exactly: (nt, c).

    unweighted: src (ne, c) float32, idx (ne,); target i sums src[e] over idx[e] == i in ascending e.
    weighted:   src (n, c) float32 (the gradient rows), idx (n, 3), weight (n, 3); entry e = 3j + t adds
                src[j] * weight[j, t] (each product rounded).  Lists of at most 256 entries are one ascending sum from
                +0; a longer list is cut into PIECES pieces of the n3 = 3n entries, piece p = [p * ceil(n3/8), ...),
                each an ascending sum from +0, and the piece sums are added in piece order starting from piece 0.
                (For a ragged cloud pass the truncated rows: the pieces are cut from 3 * len.  ``cut`` overrides the
                entry count the pieces are cut from: cut = 3n on a truncated cloud is the cut that ignores its length.)
    Every operation is one float32 rounding, as __fadd_rn / __fmul_rn."""
    src = np.ascontiguousarray(src, dtype=np.float32)
    c = src.shape[1]
    if weight is not None:
        n3 = idx.size
        tgt = np.asarray(idx, np.int64).reshape(-1)
        with np.errstate(all="ignore"):
            terms = (np.repeat(src, 3, axis=0) * np.asarray(weight, np.float32).reshape(-1, 1)).astype(np.float32)
    else:
        n3 = idx.size
        tgt = np.asarray(idx, np.int64).reshape(-1)
        terms = src
    counts = np.bincount(tgt, minlength=nt) if n3 else np.zeros(nt, np.int64)
    e = np.arange(n3)
    piece_len = _cdiv(cut if cut is not None else n3, PIECES) if n3 else 1
    piece = np.where((counts[tgt] > SORT_CAP) & (weight is not None) & long_pieces, e // piece_len, 0)
    group = tgt * PIECES + piece
    order = np.lexsort((e, group))
    g_sorted = group[order]
    first = np.r_[0, np.flatnonzero(np.diff(g_sorted)) + 1] if n3 else np.zeros(0, np.int64)
    rank = np.arange(n3) - np.repeat(first, np.diff(np.r_[first, n3])) if n3 else np.zeros(0, np.int64)
    parts = np.zeros((nt * PIECES, c), np.float32)
    with np.errstate(all="ignore"):
        for r in range(int(rank.max()) + 1 if n3 else 0):
            sel = order[rank == r]
            parts[group[sel]] = (parts[group[sel]] + terms[sel]).astype(np.float32)
        parts = parts.reshape(nt, PIECES, c)
        out = parts[:, 0].copy()
        if weight is not None and long_pieces:
            lng = counts > SORT_CAP
            for p in range(1, PIECES):
                out[lng] = (out[lng] + parts[lng, p]).astype(np.float32)
    return out
