#!/usr/bin/env python
"""Randomised differential test of the fused inference MLP kernels (TEST TOOL, runs on a GPU box): sa_mlp_max
(csrc/sa_mlp.cu), fp_mlp and mlp_rows (csrc/fp_mlp.cu).

    python tests/fuzz_mlp_gpu.py [--seconds 120] [--seed 0] [--json out.json]

Each case is ``draw_<case>(rs, it)`` (parameters and inputs with numpy alone; ``it`` picks the planner branch the
draw aims at, round-robin) and ``run_<case>(p)`` (the CUDA op and the comparison).  float32 outputs must equal
``oracle.oracle_mlp_rows_f32`` as values (±0 equal, NaN in the same places); 16-bit outputs must lie within
``mlp_oracle.bound16`` of the float64 reference, element by element.  Outputs written into a channel slice of a
NaN-filled wider tensor must leave the other columns NaN, and padding rows (ragged lengths, masked rows) must be 0.
A failure is printed with the seed, the iteration and its parameters; ``run(seed, iteration + 1)`` reproduces it.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import mlp_oracle as MO  # noqa: E402
import numerics as NUM  # noqa: E402

# the slice tests/test_fuzz_mlp_gpu.py runs, and tests/test_fuzz_mlp_cpu.py checks the coverage of
SLICE_SEEDS = (51, 52, 53)
SLICE_ITERATIONS = 72  # 24 of each case per seed: every SA target twice

CASES = ["sa", "fp", "rows"]
FORMATS = ["f32", "bf16", "f16"]
EDGE_WIDTHS = [1, 7, 8, 31, 32, 33, 63, 64, 65, 127, 129, 255, 257, 513, 1023, 1024]
WIDE = [513, 1023, 1024]
KS = [1, 2, 3, 5, 15, 16, 17, 31, 32, 33, 63, 64, 65, 129, 200]
FEATURES = [0, 1, 2, 5, 8, 29, 32, 61, 64, 125, 128, 253, 320, 509, 640, 1021, 1024]
MAC_CAP = 30_000_000  # rows x multiply-adds per row: the C oracle stays under about 0.1 s

# the branch each draw aims at, in turn (tests/test_fuzz_mlp_cpu.py checks that the slice reaches them all)
SA_TARGETS = ["sa_e4_tm64", "sa_e4_tm32", "sa_e4_tm16", "sa_e2_tm64", "sa_e2_tm32", "sa_groups_tm32",
              "sa_pieces_tm32", "sa_trimmed_e4", "sa_trimmed_e2", "sa_k_ndiv_tm", "sa_pieces_tm64+sa_partial_piece", "sa_pieces_tm16"]
ROW_TARGETS = ["rows_e4_tm64", "rows_e4_tm32", "rows_e4_tm16", "rows_e2_tm64", "rows_e2_tm32"]


# ----------------------------------------------------------------------------------------------------- drawing
def _fmt(rs):
    fmt = str(rs.choice(FORMATS))
    return fmt, bool(fmt != "f32" and rs.rand() < 0.3)


def _widths(rs, wide):
    nl = int(rs.randint(1, MO.MAX_LAYERS + 1))
    pool = WIDE if wide else EDGE_WIDTHS
    return [int(rs.choice(pool)) if rs.rand() < 0.8 else int(rs.choice(EDGE_WIDTHS)) for _ in range(nl)]


def _macs(cin, widths):
    return sum(a * b for a, b in zip([cin] + widths[:-1], widths))


def draw_layers(rs, cin, widths, fmt):
    """Linear (xavier-uniform weights, biases of a few tenths) [+ batch norm: affine, plain or none] [+ ReLU] per layer;
    running variances from 1e-4 to 10 (the small ones on one layer at most, so that float16 stays mostly finite),
    negative γ, eps 1e-3 or 1e-5; the last layer without ReLU now and then."""
    layers, prev = [], cin
    sharp = int(rs.randint(len(widths))) if rs.rand() < 0.5 else -1
    for l, w in enumerate(widths):
        lim = np.sqrt(6.0 / (prev + w))
        L = dict(w=rs.uniform(-lim, lim, (w, prev)).astype(np.float32),
                 b=(rs.standard_normal(w) * 0.3).astype(np.float32),
                 relu=bool(l + 1 < len(widths) or rs.rand() < 0.7))
        bn = str(rs.choice(["affine", "plain", "none"], p=[0.6, 0.15, 0.25]))
        if bn != "none":
            lo = 1e-4 if l == sharp else 0.3
            L.update(mean=(rs.standard_normal(w) * 0.3).astype(np.float32),
                     var=np.exp(rs.uniform(np.log(lo), np.log(10.0), w)).astype(np.float32),
                     eps=float(rs.choice([1e-3, 1e-3, 1e-5])))
            if bn == "affine":
                g = rs.uniform(0.3, 1.5, w) * np.where(rs.rand(w) < 0.25, -1, 1)
                L.update(gamma=g.astype(np.float32), beta=(rs.standard_normal(w) * 0.2).astype(np.float32))
        L["bn"] = bn
        layers.append(L)
        prev = w
    return layers


def _scaled(rs, shape, fmt):
    """standard normal features with per-channel scales from 1e-3 to 1e3 (1e2 for float16) half of the time"""
    x = rs.standard_normal(shape).astype(np.float32)
    if rs.rand() < 0.5 and shape[-1]:
        top = 1e2 if fmt == "f16" else 1e3
        x *= np.exp(rs.uniform(np.log(1e-3), np.log(top), shape[-1])).astype(np.float32)
    return x


def _poison(rs, x, frac=0.002):
    """NaN, +inf and -inf at a few places of a float32 array (float32 draws only)"""
    x = x.copy()
    flat = x.reshape(-1)
    if flat.size:
        at = rs.randint(0, flat.size, max(1, int(flat.size * frac)))
        flat[at] = rs.choice([np.nan, np.inf, -np.inf], len(at))
    return x


def _slice(rs):
    """(lo, hi): sentinel columns before and after the output's slice, or None for a tensor of its own"""
    return (int(rs.randint(0, 9)), int(rs.randint(0, 9))) if rs.rand() < 0.4 else None


def _reached(target, tags, attempt):
    """whether a draw's branches reach the target (tags joined by "+": all of them); after 300 attempts, any draw"""
    return attempt >= 300 or set(target.split("+")) <= tags


def draw_sa(rs, it=0):
    target = SA_TARGETS[(it // len(CASES)) % len(SA_TARGETS)]
    fmt, autocast = _fmt(rs)
    # TM = 16 is float32 only (16-bit stacks always fit TM = 32, see tests/test_fuzz_mlp_cpu.py)
    if "_e4_" in target or target.endswith("_e4") or "tm16" in target or target == "sa_pieces_tm32":
        fmt, autocast = "f32", False
    elif "_e2" in target and fmt == "f32":
        fmt = str(rs.choice(["bf16", "f16"]))
    esize = MO.ESIZE[fmt]
    wide = "tm16" in target or "tm32" in target
    for attempt in range(400):
        c = 0 if (autocast and rs.rand() < 0.5) else int(rs.choice(FEATURES))
        if wide and rs.rand() < 0.6:
            c = int(rs.choice([509, 640, 1021, 1024]))
        use_xyz = bool(c == 0 or rs.rand() < 0.75)
        cin = c + 3 if use_xyz else c
        widths = _widths(rs, wide and rs.rand() < 0.7)
        if "trimmed" in target and rs.rand() < 0.7:
            widths[-1] = int(rs.choice([1023, 1024]))
        group_all = bool(rs.rand() < 0.15)
        k = int(rs.randint(65, 301)) if group_all else int(rs.choice(KS))
        if "trimmed" in target and rs.rand() < 0.7:
            k = 1
        if "piece" in target and rs.rand() < 0.7:
            group_all, k = False, int(rs.choice([17, 31, 33, 63, 65, 129]))
        if target == "sa_pieces_tm16" and rs.rand() < 0.5:  # float32 TM = 16 needs wide buffers: few MACs to spare
            c, use_xyz, cin = 1024, True, 1027
            widths, k = [int(rs.choice([513, 1023, 1024])), int(rs.choice([1023, 1024]))], int(rs.choice([17, 31]))
        if cin < 1 or cin > MO.SA_MAX_IN:
            continue
        per_group = k * _macs(cin, widths)
        if per_group > MAC_CAP:
            continue
        b = int(rs.randint(1, 4))
        s = 1 if group_all else int(rs.choice([1, 2, 3, 7, 20, 64, 150]))
        while b * s * per_group > MAC_CAP and s > 1:
            s = max(1, s // 2)
        while b * s * per_group > MAC_CAP and b > 1:
            b -= 1
        plan = MO.sa_plan(esize, cin, widths, k, b * s)
        tags = MO.branches("sa", esize, cin, widths, plan, k=k)
        if _reached(target, tags, attempt):
            break
    autocast = autocast or (c == 0 and fmt != "f32")  # without features only autocast picks a 16-bit type
    n = k if group_all else int(rs.choice([k, k + 1, 40, 300, 2000]))
    xs = float(rs.choice([1.0, 1e-2, 30.0]))
    xyz = (rs.random_sample((b, n, 3)) * xs).astype(np.float32)
    if group_all:
        idx, new_xyz = None, (None if rs.rand() < 0.5 else (rs.random_sample((b, 1, 3)) * xs).astype(np.float32))
    else:
        idx = rs.randint(0, n, (b, s, k)).astype(np.int32)
        new_xyz = xyz[:, rs.randint(0, n, s)].copy() if rs.rand() < 0.8 else None
    points = _scaled(rs, (b, n, c), fmt) if c else None
    nonfinite = bool(fmt == "f32" and rs.rand() < 0.25)
    if nonfinite:
        if points is not None and rs.rand() < 0.7:
            points = _poison(rs, points)
        else:
            xyz = _poison(rs, xyz)
    return dict(case="sa", fmt=fmt, autocast=autocast, target=target, b=b, n=n, s=s, k=k, c=c, cin=cin,
                widths=widths, group_all=group_all, xyz_first=bool(rs.rand() < 0.5), use_xyz=use_xyz,
                nonfinite=nonfinite, slice=_slice(rs), plan=plan, tags=sorted(tags),
                xyz=xyz, new_xyz=new_xyz, points=points, idx=idx) | _layers(rs, cin, widths, fmt)


def _layers(rs, cin, widths, fmt):
    layers = draw_layers(rs, cin, widths, fmt)
    return dict(layers=layers, bn=[L["bn"] for L in layers], relu=[L["relu"] for L in layers])


def _row_shape(rs, target):
    fmt, autocast = _fmt(rs)
    if "_e4_" in target:
        fmt, autocast = "f32", False
    elif "_e2_" in target and fmt == "f32":
        fmt = str(rs.choice(["bf16", "f16"]))
    return fmt, autocast, "tm16" in target or "tm32" in target


def draw_fp(rs, it=0):
    target = ROW_TARGETS[(it // len(CASES)) % len(ROW_TARGETS)]
    fmt, autocast, wide = _row_shape(rs, target)
    esize = MO.ESIZE[fmt]
    for attempt in range(400):
        c2 = int(rs.choice([1, 3, 8, 33, 64, 128, 255, 512, 1024]))
        c1 = 0 if rs.rand() < 0.3 else int(rs.choice([1, 3, 7, 22, 64, 128, 256, 512]))
        if wide and rs.rand() < 0.6:
            c2, c1 = int(rs.choice([512, 1024])), int(rs.choice([0, 256, 512]))
        cin = c2 + c1
        widths = _widths(rs, wide and rs.rand() < 0.7)
        if cin > MO.ROW_MAX_IN:
            continue
        b = int(rs.randint(1, 4))
        n = int(rs.choice([1, 2, 17, 63, 64, 65, 200, 1000, 3000]))
        while b * n * _macs(cin, widths) > MAC_CAP and n > 1:
            n = max(1, n // 3)
        if b * n * _macs(cin, widths) > MAC_CAP:
            continue
        plan = MO.row_plan(esize, cin, widths, b * n)
        tags = MO.branches("rows", esize, cin, widths, plan, rows=b * n)
        if _reached(target, tags, attempt):
            break
    m = int(rs.choice([1, 2, 3, 16, 100, 700]))
    xyz1 = rs.random_sample((b, n, 3)).astype(np.float32)
    xyz2 = rs.random_sample((b, m, 3)).astype(np.float32)
    if rs.rand() < 0.3 and m <= n:
        xyz2 = xyz1[:, :m].copy()  # nested sets, as in feature propagation: exact zero distances
    ragged = bool(rs.rand() < 0.5)
    lengths = [int(rs.choice([1, n, max(1, n - 1), int(rs.randint(1, n + 1))])) for _ in range(b)] if ragged else None
    return dict(case="fp", fmt=fmt, autocast=autocast, target=target, b=b, n=n, m=m, c2=c2, c1=c1, cin=cin,
                widths=widths, lengths=lengths, slice=_slice(rs), plan=plan, tags=sorted(tags),
                xyz1=xyz1, xyz2=xyz2, p2=_scaled(rs, (b, m, c2), fmt),
                p1=_scaled(rs, (b, n, c1), fmt) if c1 else None) | _layers(rs, cin, widths, fmt)


def draw_rows(rs, it=0):
    target = ROW_TARGETS[(it // len(CASES)) % len(ROW_TARGETS)]
    fmt, autocast, wide = _row_shape(rs, target)
    esize = MO.ESIZE[fmt]
    for attempt in range(400):
        c = int(rs.choice([1, 2, 7, 31, 32, 33, 64, 65, 129, 259, 513, 1024, 1027, 1535, 1536]))
        if wide and rs.rand() < 0.6:
            c = int(rs.choice([1027, 1280, 1535, 1536]))
        widths = _widths(rs, wide and rs.rand() < 0.7)
        rows = int(rs.choice([1, 15, 16, 17, 64, 65, 500, 4000]))
        while rows * _macs(c, widths) > MAC_CAP and rows > 1:
            rows = max(1, rows // 3)
        if rows * _macs(c, widths) > MAC_CAP:
            continue
        plan = MO.row_plan(esize, c, widths, rows)
        tags = MO.branches("rows", esize, c, widths, plan, rows=rows)
        if _reached(target, tags, attempt):
            break
    lead = (rows,) if rs.rand() < 0.5 or rows % 2 else (2, rows // 2)
    x = _scaled(rs, (rows, c), fmt)
    mask = (rs.rand(rows) < 0.7) if rs.rand() < 0.4 else None
    nonfinite = bool(fmt == "f32" and rs.rand() < 0.25)
    if nonfinite:
        x = _poison(rs, x)
    return dict(case="rows", fmt=fmt, autocast=autocast, target=target, rows=rows, lead=lead, c=c, cin=c,
                widths=widths, nonfinite=nonfinite, slice=_slice(rs), plan=plan, tags=sorted(tags),
                x=x, mask=mask) | _layers(rs, c, widths, fmt)


# ----------------------------------------------------------------------------------------------------- running
# torch and the package are imported when a case runs, so that the draws (and tests/test_fuzz_mlp_cpu.py) need neither
# a device nor the built library
def _torch():
    import torch
    return torch


DTYPES = {"f32": "float32", "bf16": "bfloat16", "f16": "float16"}


def torch_dtype(fmt):
    return getattr(_torch(), DTYPES[fmt])


def dev():
    return _torch().device("cuda:0")


def build_mlp(cin, layers):
    """an eval-mode SharedMLP on cuda:0 holding exactly these layers (batch norms with or without affine, ReLU or not)"""
    torch = _torch()
    from torch import nn
    from pointnet2_b200.layers import SharedMLP
    mlp = SharedMLP(cin, [int(L["w"].shape[0]) for L in layers])
    mods = []
    for L in layers:
        cout, prev = L["w"].shape
        lin = nn.Linear(prev, cout)
        with torch.no_grad():
            lin.weight.copy_(torch.from_numpy(L["w"]))
            lin.bias.copy_(torch.from_numpy(L["b"]))
        mods.append(lin)
        if "mean" in L:
            bn = nn.BatchNorm1d(cout, eps=L["eps"], affine="gamma" in L)
            with torch.no_grad():
                bn.running_mean.copy_(torch.from_numpy(L["mean"]))
                bn.running_var.copy_(torch.from_numpy(L["var"]))
                if "gamma" in L:
                    bn.weight.copy_(torch.from_numpy(L["gamma"]))
                    bn.bias.copy_(torch.from_numpy(L["beta"]))
            mods.append(bn)
        if L["relu"]:
            mods.append(nn.ReLU())
    mlp.body = nn.Sequential(*mods)
    return mlp.to(dev()).eval()


def oracle_layers(layers):
    """the layer dicts the C oracle takes (bias always present, as nn.Linear has one)"""
    keys = ("w", "b", "gamma", "beta", "mean", "var", "eps", "relu")
    return [{k: L[k] for k in keys if k in L} for L in layers]


def affine(layers):
    from oracle import oracle as O
    return [O.oracle_mlp_affine_f32(L) for L in oracle_layers(layers)]


def values(t):
    """a device tensor as float32 numpy values (an exact upcast)"""
    return t.detach().float().cpu().numpy()


def same_values(got, want):
    """equal as values: ±0 equal, NaN in the same places"""
    return bool(got.shape == want.shape and np.array_equal(got, want, equal_nan=True))


def compare(got, rows, layers, fmt, pool_k=None, stats=None):
    """got (R', cout) float32 values against the reference of rows (R, cin) (R' = R / pool_k with pooling)"""
    from oracle import oracle as O
    if fmt == "f32":
        want = O.oracle_mlp_rows_f32(rows, oracle_layers(layers))
        if pool_k is not None:
            want = MO.max_pool(want, pool_k)
        return same_values(got, want)
    ref, bound = MO.bound16(rows, layers, affine(layers), fmt, pool_k)
    ok, ratio = MO.check16(got, ref, bound)
    if stats is not None:
        stats["worst_ratio"] = max(stats.get("worst_ratio", 0.0), ratio)
        stats["unbounded"] = stats.get("unbounded", 0) + int(np.isinf(bound).sum())
        stats["elements"] = stats.get("elements", 0) + int(bound.size)
    return ok


def _out(lead, cout, sl, dtype):
    """(tensor passed as out, full tensor): a slice of a NaN-filled wider tensor, or (None, None)"""
    torch = _torch()
    if sl is None:
        return None, None
    lo, hi = sl
    full = torch.full((*lead, lo + cout + hi), float("nan"), dtype=dtype, device=dev())
    return full[..., lo:lo + cout], full


def _sentinels_hold(full, sl, cout):
    if full is None:
        return True
    f = values(full)
    lo, hi = sl
    return bool(np.isnan(f[..., :lo]).all() and np.isnan(f[..., lo + cout:]).all())


def _autocast(p):
    torch = _torch()
    return torch.autocast("cuda", dtype=torch_dtype(p["fmt"]), enabled=p["autocast"])


def _feat(a, p):
    """float32 numpy features on the device, in the arithmetic type (float32 under autocast: the op casts them)"""
    torch = _torch()
    t = torch.from_numpy(np.ascontiguousarray(a)).to(dev())
    return t if p["autocast"] else t.to(torch_dtype(p["fmt"]))


def sa_output(p):
    """sa_mlp_max on case p: (output tensor, the NaN-filled tensor it is a slice of or None, the (B, S, K, cin) rows)"""
    torch = _torch()
    from pointnet2_b200.layers import sa_mlp_max
    fmt, cout = p["fmt"], p["widths"][-1]
    mlp = build_mlp(p["cin"], p["layers"])
    T = lambda a: None if a is None else torch.from_numpy(np.ascontiguousarray(a)).to(dev())
    points = None if p["points"] is None else _feat(p["points"], p)
    s = 1 if p["group_all"] else p["s"]
    out, full = _out((p["b"], s), cout, p["slice"], torch_dtype(fmt))
    with torch.no_grad(), _autocast(p):
        got = sa_mlp_max(T(p["xyz"]), T(p["new_xyz"]), points, T(p["idx"]), mlp, p["xyz_first"], p["use_xyz"], out=out)
    pq = None if p["points"] is None else NUM.quantize(p["points"], fmt)
    return got, full, MO.sa_rows(p["xyz"], p["new_xyz"], pq, p["idx"], p["xyz_first"], p["use_xyz"], fmt)


def run_sa(p, stats=None):
    got, full, rows = sa_output(p)
    fmt, cout = p["fmt"], p["widths"][-1]
    ok = got.dtype == torch_dtype(fmt) and tuple(got.shape) == (p["b"], rows.shape[1], cout)
    k = rows.shape[2]
    ok = ok and compare(values(got).reshape(-1, cout), rows.reshape(-1, rows.shape[-1]), p["layers"], fmt, k, stats)
    return bool(ok and _sentinels_hold(full, p["slice"], cout))


def run_fp(p, stats=None):
    torch = _torch()
    from pointnet2_b200.layers import fp_mlp
    from pointnet2_b200.tf_interpolate import fp_interpolate_concat
    fmt, cout, b, n = p["fmt"], p["widths"][-1], p["b"], p["n"]
    mlp = build_mlp(p["cin"], p["layers"])
    ls = p["lengths"]
    x1, p1 = p["xyz1"], p["p1"]
    if ls is not None:  # the padding is never read: poison it
        x1 = NUM.pad_rows(x1, ls, "poison")
        p1 = None if p1 is None else NUM.pad_rows(p1, ls, "poison")
    T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev())
    lengths = None if ls is None else torch.tensor(ls, dtype=torch.int32, device=dev())
    out, full = _out((b, n), cout, p["slice"], torch_dtype(fmt))
    p1d = None if p1 is None else _feat(p1, p)
    with torch.no_grad(), _autocast(p):
        got = fp_mlp(T(x1), T(p["xyz2"]), p1d, _feat(p["p2"], p), mlp, lengths=lengths, out=out)
    ok = got.dtype == torch_dtype(fmt) and tuple(got.shape) == (b, n, cout)
    # the first layer's rows: what fp_interpolate_concat writes (pinned bit for bit to the oracle elsewhere)
    D = torch_dtype(fmt)
    cat = fp_interpolate_concat(T(x1), T(p["xyz2"]), None if p1 is None else T(p1).to(D), T(p["p2"]).to(D),
                                lengths=lengths)
    real = np.ones((b, n), bool) if ls is None else np.arange(n)[None, :] < np.asarray(ls)[:, None]
    g = values(got)
    ok = ok and compare(g[real], values(cat)[real], p["layers"], fmt, None, stats)
    ok = ok and bool((g[~real] == 0).all())
    return bool(ok and _sentinels_hold(full, p["slice"], cout))


def rows_output(p):
    """mlp_rows (or, for an output slice, its C entry) on case p: (output tensor, the NaN-filled tensor it is a slice of
    or None, the float32 inputs with the masked rows poisoned)"""
    torch = _torch()
    from pointnet2_b200 import _lib
    from pointnet2_b200._tensor import ptr, stream_ptr
    from pointnet2_b200.layers import DTYPE_CODES, _layer_args, _mlp_stack, mlp_rows
    fmt, cout, lead = p["fmt"], p["widths"][-1], p["lead"]
    mlp = build_mlp(p["cin"], p["layers"])
    x, mask = p["x"], p["mask"]
    if mask is not None:  # masked rows are never read: poison them
        x = x.copy()
        x[~mask] = np.array([np.nan, np.inf, -np.inf, NUM.FAR], np.float32)[np.arange((~mask).sum()) % 4, None]
    t = _feat(x, p).reshape(*lead, p["c"])
    md = None if mask is None else torch.from_numpy(mask).to(dev()).reshape(lead)
    D = torch_dtype(fmt)
    with torch.no_grad(), _autocast(p):
        if p["slice"] is None:
            return mlp_rows(t, mlp, md), None, x
        # a channel slice of a wider tensor: the C entry's row stride (mlp_rows itself always allocates)
        got, full = _out(lead, cout, p["slice"], D)
        keep = None if md is None else md.reshape(-1).contiguous().view(torch.uint8)
        td = t.to(D)
        rc = _lib.load().pn2_mlp_rows_typed(DTYPE_CODES[D], p["rows"], p["c"], ptr(td), ptr(keep),
                                            *_layer_args(_mlp_stack(mlp)), ptr(got), full.shape[-1], stream_ptr(dev()))
        _lib.check(rc, "pn2_mlp_rows_typed")
    return got, full, x


def run_rows(p, stats=None):
    got, full, x = rows_output(p)
    fmt, cout, lead, mask = p["fmt"], p["widths"][-1], p["lead"], p["mask"]
    ok = got.dtype == torch_dtype(fmt) and tuple(got.shape) == (*lead, cout)
    g = values(got).reshape(-1, cout)
    real = np.ones(p["rows"], bool) if mask is None else mask
    ok = ok and compare(g[real], NUM.quantize(x, fmt)[real], p["layers"], fmt, None, stats)
    ok = ok and bool((g[~real] == 0).all())
    return bool(ok and _sentinels_hold(full, p["slice"], cout))


def mutation_layers(rs, cin=37):
    """the stack the mutation checks run on: two layers, the last with a partial second pass (80 channels), batch
    norms with eps 1e-3 and running variances from 1e-4 to 1e-3, ReLU throughout"""
    layers = draw_layers(rs, cin, [96, 80], "bf16")
    for L in layers:
        cout = L["w"].shape[0]
        L.update(mean=(rs.standard_normal(cout) * 0.1).astype(np.float32),
                 var=rs.uniform(1e-4, 1e-3, cout).astype(np.float32), eps=1e-3,
                 gamma=rs.uniform(0.3, 1.0, cout).astype(np.float32),
                 beta=(rs.standard_normal(cout) * 0.1).astype(np.float32), relu=True, bn="affine")
    return layers


DRAW = {name: globals()["draw_" + name] for name in CASES}
RUN = {name: globals()["run_" + name] for name in CASES}


def draws(seed: int, iterations: int):
    """The parameters ``run(seed, iterations)`` uses, without a device (the run_* functions draw nothing)."""
    rs = np.random.RandomState(seed)
    return [DRAW[CASES[it % len(CASES)]](rs, it) for it in range(iterations)]


def public(p):
    """the parameters of a case without its arrays (they follow from the seed and the iteration)"""
    return {k: v for k, v in p.items() if not isinstance(v, np.ndarray) and k != "layers"}


def _one(rs, it, seed, counts, branches, fails, stats, catch):
    name = CASES[it % len(CASES)]
    p = DRAW[name](rs, it)
    try:
        ok = RUN[name](p, stats)
    except Exception as e:  # noqa: BLE001 — report the exception as a failure of that case
        if not catch:
            raise
        ok = False
        p = dict(p, error=f"{type(e).__name__}: {e}")
    counts[name] = counts.get(name, 0) + 1
    for t in p["tags"]:
        branches[t] = branches.get(t, 0) + 1
    if not ok:
        fails.append(dict(public(p), seed=seed, iteration=it))
    return ok, fails[-1] if not ok else None


def run(seed: int, iterations: int, stats: dict | None = None):
    """``iterations`` random cases (round-robin over CASES); returns (counts, failures).  ``stats``, if given, receives
    the planner branches taken and the worst 16-bit err / bound."""
    rs = np.random.RandomState(seed)
    counts, fails, branches = {}, [], {}
    stats = {} if stats is None else stats
    for it in range(iterations):
        _one(rs, it, seed, counts, branches, fails, stats, catch=False)
    stats["branches"] = branches
    return counts, fails


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=float, default=120)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--json", type=str, default=None)
    args = ap.parse_args()
    rs = np.random.RandomState(args.seed)
    counts, branches, fails, stats, secs = {}, {}, [], {}, {}
    t0 = last = time.time()
    it = 0
    while time.time() - t0 < args.seconds:
        if time.time() - last >= 60:  # a progress line a minute
            last = time.time()
            print(json.dumps(dict(seconds=round(last - t0), cases=it, failures=len(fails))), flush=True)
        t1 = time.time()
        ok, fail = _one(rs, it, args.seed, counts, branches, fails, stats, catch=True)
        name = CASES[it % len(CASES)]
        secs[name] = secs.get(name, 0.0) + time.time() - t1
        if not ok:
            print("FAIL", json.dumps(fail, default=str), flush=True)
        it += 1
    summary = dict(seed=args.seed, seconds=round(time.time() - t0, 1), cases=counts,
                   branches=dict(sorted(branches.items())), worst_err_over_bound_16bit=stats.get("worst_ratio"),
                   elements_16bit=stats.get("elements", 0), unbounded_16bit=stats.get("unbounded", 0),
                   case_seconds={k: round(v, 1) for k, v in secs.items()}, failures=fails)
    print(json.dumps(summary, default=str))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(summary, f, indent=1, default=str)
    sys.exit(1 if fails else 0)


if __name__ == "__main__":
    main()
