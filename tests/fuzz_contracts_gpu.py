#!/usr/bin/env python
"""Randomised differential test of the per-cloud lengths, 16-bit features and deterministic gradients (TEST TOOL, runs
on a GPU box).

    python tests/fuzz_contracts_gpu.py [--seconds 120] [--seed 0] [--json out.json]

Each case is two functions: ``draw_<case>(rs)`` makes its parameters and inputs with numpy alone (no device), and
``run_<case>(p)`` runs the CUDA ops and compares them with the C oracle on the truncated clouds.  Outputs must be
bit-exact wherever the contract says so (DESIGN.md §6.4 "16-bit features", §6.8); float atomics and the eight-piece
sums of lists longer than 256 entries are held to the float64 bound of ``numerics.within_bound`` instead of a fixed
atol.  Every ragged case runs once with poisoned padding (NaN, ±inf, a far point) and once with padding that copies
real rows, and the two runs must agree bit for bit.  A failure is printed with the seed, the iteration and its
parameters; the inputs come from numpy's RandomState, so ``run(seed, iteration + 1)`` reproduces it on any machine.
"""
from __future__ import annotations

import argparse
import ctypes
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numerics as NUM  # noqa: E402
from fuzz_gpu import cloud, log_n  # noqa: E402  (the U/S/D/G/L cloud distributions)
from oracle import oracle as _oracle  # noqa: E402
from pointnet2_b200 import _lib, tf_interpolate, workloads as W  # noqa: E402
from pointnet2_b200._tensor import ptr, stream_ptr  # noqa: E402
from pointnet2_b200.pointnet_util import group_and_concat  # noqa: E402
from pointnet2_b200.sa_layer import sample_group, sample_group_msg  # noqa: E402
from pointnet2_b200.tf_grouping import group_point, query_ball_point  # noqa: E402
from pointnet2_b200.tf_interpolate import fp_interpolate_concat, three_interpolate, three_nn, three_nn_interpolate  # noqa: E402
from pointnet2_b200.tf_sampling import farthest_point_sample_and_gather, gather_point  # noqa: E402

dev = torch.device("cuda:0")  # only dereferenced when a case runs

# the slice tests/test_fuzz_contracts_gpu.py runs, and tests/test_fuzz_contracts_cpu.py checks the coverage of
SLICE_SEEDS = (31, 32, 33)
SLICE_ITERATIONS = 180  # twenty of each case per seed

DTYPES = {"f32": torch.float32, "bf16": torch.bfloat16, "f16": torch.float16}
WIDTHS = [1, 3, 4, 5, 7, 8, 16, 64, 67, 128, 131, 259, 320]  # the channel counts the feature kernels branch on
CUDA_ERROR_INVALID_VALUE = 1


class _Counted:
    """The oracle module with a call counter (the cost of each case is reported in oracle calls)."""

    def __init__(self, mod):
        self._mod, self.calls = mod, 0

    def __getattr__(self, name):
        fn = getattr(self._mod, name)

        def counted(*a, **k):
            self.calls += 1
            return fn(*a, **k)
        return counted


O = _Counted(_oracle)


# ------------------------------------------------------------------------------------------------------ helpers
def T(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


def N(t):
    return t.detach().cpu().numpy()


def bits(t):
    """a tensor's raw bits as numpy (uint16 for 2-byte floats, int32 view for float32, ints as they are)"""
    t = t.detach()
    if t.dtype in (torch.bfloat16, torch.float16):
        return t.view(torch.int16).cpu().numpy().view(np.uint16)
    if t.dtype == torch.float32:
        return t.cpu().numpy().view(np.int32)
    return t.cpu().numpy()


def want_bits(x_f32, fmt):
    """the bits a fmt result must have: float32 values rounded once"""
    r = NUM.round_once(x_f32, fmt)
    return r if fmt != "f32" else r.view(np.int32)


def feat(a, fmt, offset=0):
    """float32 numpy features as a device tensor of format fmt whose data starts ``offset`` elements into its buffer
    (offset 1: a base that is 2- or 4-byte but not 16-byte aligned)"""
    t = T(a).to(DTYPES[fmt])
    buf = torch.empty(t.numel() + offset, dtype=t.dtype, device=dev)
    buf[offset:].copy_(t.reshape(-1))
    return buf[offset:].view(t.shape)


def same_bits(xs, ys):
    return all(x is None or np.array_equal(bits(x), bits(y)) for x, y in zip(xs, ys))


def draw_lengths(rs, b, n, npoint=None):
    """Per-cloud lengths of a padded (b, n) batch: boundary values (1, 2, 3, n − 1, n, npoint ± 1, multiples of
    32 / 64 / 128 ± 1, the 2048 / 9700 ball-query thresholds below an n above them) mixed with U[1, n].  The form
    alternates between a host list, int32 and int64 device tensors, and device tensors holding 0 or n + 5 (clamped
    to [1, n] by the kernels).  Returns {"form", "raw" (what is passed), "lengths" (what each cloud has)}."""
    pool = [1, 2, 3, n - 1, n]
    if npoint:
        pool += [npoint - 1, npoint, npoint + 1]
    for k in (32, 64, 128):
        q = k * int(rs.randint(1, n // k + 2))
        pool += [q - 1, q + 1]
    if n > 2048:
        pool += [2047, 2048, int(rs.randint(1, 2048))]
    if n > 9700:
        pool += [9700, 9699, int(rs.randint(2048, 9701))]
    vals = [int(pool[rs.randint(len(pool))]) if rs.rand() < 0.6 else int(rs.randint(1, n + 1)) for _ in range(b)]
    vals = [min(max(v, 1), n) for v in vals]
    form = str(rs.choice(["host", "int32", "int64", "clamp"], p=[0.35, 0.25, 0.25, 0.15]))
    raw = list(vals)
    if form == "clamp":
        for i in range(b):
            if rs.rand() < 0.5:
                raw[i] = int(rs.choice([0, -3, n + 5]))
                vals[i] = 1 if raw[i] < 1 else n
        form = "clamp_" + str(rs.choice(["int32", "int64"]))
    return dict(form=form, raw=raw, lengths=vals)


def lengths_arg(spec):
    if spec["form"] == "host":
        return list(spec["raw"])
    dtype = torch.int64 if spec["form"].endswith("int64") else torch.int32
    return torch.tensor(spec["raw"], dtype=dtype, device=dev)


def both_paddings(fn, arrays, lengths):
    """fn(*padded device arrays) with poisoned and with copied padding: (outputs of the poisoned run, bit-identical?)"""
    outs = [fn(*[NUM.pad_rows(a, lengths, kind) for a in arrays]) for kind in ("poison", "copy")]
    return outs[0], same_bits(outs[0], outs[1])


def radius_for(rs, xyz, lo, hi):
    ext = float(np.nanmax(xyz) - np.nanmin(xyz)) + 1e-3
    return float(np.float32(ext * np.exp(rs.uniform(np.log(lo), np.log(hi)))))


def free_points(rs, xyz, b, m):
    lo, hi = float(xyz.min()), float(xyz.max())
    return (lo + (hi - lo + 1e-3) * rs.random_sample((b, m, 3)) * 1.2 - 0.1).astype(np.float32)


def zipf_index(rs, shape, n):
    """indices in [0, n) with a heavy head (a few rows collect most entries: long lists), in a random order of rows"""
    z = rs.zipf(1.2 + rs.rand(), shape) - 1
    return rs.permutation(n)[z % n].astype(np.int32)


def check_grad(got_bits, want_f32, ref64, mass, count, fmt, exact):
    """``exact`` (per target row): bit-exact to the float32 ordered sum rounded once; elsewhere the float64 bound"""
    want = want_bits(want_f32, fmt)
    ok_exact = np.all((got_bits == want) | ~exact[:, None])
    got = NUM.decode(got_bits, fmt) if fmt != "f32" else got_bits.view(np.float32)
    inb = NUM.within_bound(got, ref64, mass, np.maximum(count, 1)[:, None], fmt)
    return bool(ok_exact and np.all(inb | exact[:, None]))


# --------------------------------------------------------------------------------------------------------- FPS
CHAIN_PLANS = [((256, 16), 4096), ((128, 8), 1024), ((256, 4), 1024)]  # (threads, points per thread), capacity


def draw_fps_ragged(rs):
    b, n = int(rs.randint(1, 7)), log_n(rs, 1, 40000)
    npoint = int(rs.choice([1, 2, 3, n // 7 + 1, n // 2 + 1, n - 1, n, n + 3]))
    npoint = max(1, min(npoint, 600, 2 * 10 ** 7 // n))
    kind, xyz = cloud(rs, b, n)
    lens = draw_lengths(rs, b, n, npoint)
    plan = None
    if rs.rand() < 0.25:
        r = rs.rand()
        chains = [tp for tp, cap in CHAIN_PLANS if n <= cap]
        if r < 0.3 and chains:  # one CTA per cloud, the plain (-1) or packed (-2) chain
            t, pp = chains[rs.randint(len(chains))]
            plan = (t, pp, int(rs.choice([-1, -2])))
        elif r < 0.85:  # the register + shared-memory cluster kernel; +0 / +1 / +2 = built-in / packed / plain chain
            ppt = int(rs.choice([44, 48, 52]))
            cmin = max(2, -(-n // (512 * ppt)))
            plan = (512 + int(rs.randint(0, 3)), ppt, int(rs.randint(cmin, 17)))
        else:  # global scratch
            plan = (1024, 1, 0)
    return dict(case="fps_ragged", b=b, n=n, npoint=npoint, kind=kind, lens=lens, plan=plan, xyz=xyz)


def run_fps_ragged(p):
    lib, x, ls = _lib.load(), p["xyz"], p["lens"]["lengths"]
    try:
        if p["plan"]:
            lib.pn2_set_fps_config(*p["plan"])
        (idx, nx), ok = both_paddings(lambda a: farthest_point_sample_and_gather(p["npoint"], T(a), lengths=lengths_arg(p["lens"])),
                                      [x], ls)
    finally:
        lib.pn2_set_fps_config(0, 0, 0)
    idx, nx = N(idx), N(nx)
    for i, l in enumerate(ls):
        c = x[i:i + 1, :l]
        o = O.oracle_fps(p["npoint"], c)
        ok = ok and np.array_equal(idx[i:i + 1], o) and np.array_equal(nx[i:i + 1].view(np.int32),
                                                                         O.oracle_gather_point(c, o).view(np.int32))
    return ok


# -------------------------------------------------------------------------------------------------- ball query
def draw_ball_ragged(rs):
    b = int(rs.randint(1, 6))
    n = log_n(rs, 2048, 20000) if rs.rand() < 0.35 else log_n(rs, 1, 20000)
    m, s = log_n(rs, 1, 600), int(rs.choice([1, 2, 8, 16, 32, 33, 64, 128]))
    kind, xyz = cloud(rs, b, n)
    lens = draw_lengths(rs, b, n)
    r = radius_for(rs, xyz, 0.005, 0.7)
    if rs.rand() < 0.5:  # queries are points of the truncated clouds
        q = np.stack([xyz[i, rs.randint(0, l, m)] for i, l in enumerate(lens["lengths"])])
    else:
        q = free_points(rs, xyz, b, m)
    return dict(case="ball_ragged", b=b, n=n, m=m, s=s, r=r, kind=kind, lens=lens, mode=int(rs.randint(0, 3)),
                group=int(rs.choice([0, 0, 1, 2, 4, 8, 16, 32])), xyz=xyz, q=q)


def run_ball_ragged(p):
    lib, x, ls = _lib.load(), p["xyz"], p["lens"]["lengths"]
    qd = T(p["q"])
    try:
        lib.pn2_set_bq_mode(p["mode"])
        lib.pn2_set_bq_group(p["group"])
        (idx, cnt), ok = both_paddings(lambda a: query_ball_point(p["r"], p["s"], T(a), qd, lengths=lengths_arg(p["lens"])), [x], ls)
    finally:
        lib.pn2_set_bq_mode(0)
        lib.pn2_set_bq_group(0)
    idx, cnt = N(idx), N(cnt)
    for i, l in enumerate(ls):
        oi, oc = O.oracle_query_ball_point(p["r"], p["s"], x[i:i + 1, :l], p["q"][i:i + 1])
        ok = ok and np.array_equal(idx[i:i + 1], oi) and np.array_equal(cnt[i:i + 1], oc)
    return ok


# ------------------------------------------------------------------------------------------------------- layers
def draw_layer_ragged(rs):
    b, n = int(rs.randint(1, 9)), log_n(rs, 1, 12000)
    m = min(max(1, int(rs.choice([1, n // 9 + 1, n // 4 + 1, n, n + 2]))), 400)
    kind, xyz = cloud(rs, b, n)
    scales = int(rs.choice([1, 1, 2, 3]))
    radii = [radius_for(rs, xyz, 0.01, 0.6) for _ in range(scales)]
    ns = [int(rs.choice([1, 4, 16, 32, 64, 128, 150])) for _ in range(scales)]
    return dict(case="layer_ragged", b=b, n=n, m=m, kind=kind, radii=radii, ns=ns, center=bool(rs.rand() < 0.5),
                consumer_ctas=int(rs.choice([0, 2])), lens=draw_lengths(rs, b, n, m), xyz=xyz)


def run_layer_ragged(p):
    lib, x, ls = _lib.load(), p["xyz"], p["lens"]["lengths"]
    m, center = p["m"], p["center"]

    def layer(a):
        if len(p["radii"]) == 1:
            return list(sample_group(m, p["radii"][0], p["ns"][0], T(a), center=center, lengths=lengths_arg(p["lens"])))
        fi, nx, idx, cnt, g = sample_group_msg(m, p["radii"], p["ns"], T(a), center=center, lengths=lengths_arg(p["lens"]))
        return [fi, nx] + [t for k in range(len(idx)) for t in (idx[k], cnt[k], g[k])]
    try:
        lib.pn2_set_sa_consumer_ctas(p["consumer_ctas"])
        out, ok = both_paddings(layer, [x], ls)
    finally:
        lib.pn2_set_sa_consumer_ctas(0)
    out = [N(t) for t in out]
    for i, l in enumerate(ls):
        c = x[i:i + 1, :l]
        o_fi = O.oracle_fps(m, c)
        o_nx = O.oracle_gather_point(c, o_fi)
        ok = ok and np.array_equal(out[0][i:i + 1], o_fi) and np.array_equal(out[1][i:i + 1], o_nx)
        for k, (r, s) in enumerate(zip(p["radii"], p["ns"])):
            oi, oc = O.oracle_query_ball_point(r, s, c, o_nx)
            og = O.oracle_group_point(c, oi)
            if center:
                og = (og - o_nx[:, :, None, :]).astype(np.float32)
            idx, cnt, g = out[2 + 3 * k: 5 + 3 * k]
            ok = ok and np.array_equal(idx[i:i + 1], oi) and np.array_equal(cnt[i:i + 1], oc)
            ok = ok and np.array_equal(g[i:i + 1].view(np.int32), og.view(np.int32))
    return ok


# ----------------------------------------------------------------------------------------- interpolation, forward
def draw_interp_ragged(rs):
    b, n, m = int(rs.randint(1, 5)), log_n(rs, 1, 6000), log_n(rs, 1, 1500)
    c2, c1 = int(rs.choice(WIDTHS)), int(rs.choice([0, 3, 4, 64]))
    k1, xyz1 = cloud(rs, b, n)
    k2, xyz2 = cloud(rs, b, m)
    if rs.rand() < 0.4 and m <= n:
        xyz2 = xyz1[:, :m].copy()  # nested sets as in feature propagation: exact zero distances
    scale = float(rs.choice([1.0, 1.0, 2.0 ** -20, 2.0 ** 12]))
    p2 = W.features(b, m, c2, int(rs.randint(1 << 30))) * np.float32(scale)
    p1 = W.features(b, n, c1, int(rs.randint(1 << 30)))
    return dict(case="interp_ragged", b=b, n=n, m=m, c2=c2, c1=c1, kinds=k1 + k2, scale=scale,
                fmt=str(rs.choice(list(DTYPES))), offset=int(rs.randint(0, 2)), lens=draw_lengths(rs, b, n),
                xyz1=xyz1, xyz2=xyz2, p2=p2, p1=p1)


def run_interp_ragged(p):
    fmt, off, c2, c1 = p["fmt"], p["offset"], p["c2"], p["c1"]
    x1, x2, ls, n = p["xyz1"], p["xyz2"], p["lens"]["lengths"], p["n"]
    p2 = p["p2"]
    x2d, p2d = T(x2), feat(p2, fmt, off)
    (d, i), ok = both_paddings(lambda a: three_nn(T(a), x2d, lengths=lengths_arg(p["lens"])), [x1], ls)
    (out, dd, ii, ww), ok2 = both_paddings(
        lambda a: three_nn_interpolate(T(a), x2d, p2d, return_aux=True, lengths=lengths_arg(p["lens"])), [x1], ls)
    (cat,), ok3 = both_paddings(
        lambda a, q: [fp_interpolate_concat(T(a), x2d, feat(q, fmt, off) if c1 else None, p2d, lengths=lengths_arg(p["lens"]))],
        [x1, p["p1"]], ls)
    ok = ok and ok2 and ok3
    real = np.arange(n)[None, :] < np.asarray(ls)[:, None]
    # three_nn: the oracle on each truncated cloud; the fused kernel's dist / idx are the same
    d, i, dd, ii, ww = bits(d), bits(i), bits(dd), bits(ii), N(ww)
    for k, l in enumerate(ls):
        od, oi = O.oracle_three_nn(x1[k:k + 1, :l], x2[k:k + 1])
        ok = ok and np.array_equal(d[k, :l], od[0].view(np.int32)) and np.array_equal(i[k, :l], oi[0])
    ok = ok and np.array_equal(dd, d) and np.array_equal(ii, i)
    # weights: what the call without lengths gives on the copied padding
    wd = N(three_nn_interpolate(T(NUM.pad_rows(x1, ls, "copy")), x2d, p2d, return_aux=True)[3])
    ok = ok and np.array_equal(ww[real].view(np.int32), wd[real].view(np.int32))
    # interpolated part: the float32 oracle on the upcast features with the kernel's own weights, rounded once
    want = want_bits(O.oracle_three_interpolate(NUM.quantize(p2, fmt), ii, ww), fmt)
    out, cat = bits(out), bits(cat)
    ok = ok and np.array_equal(out[real], want[real]) and np.array_equal(cat[..., :c2][real], want[real])
    if c1:
        ok = ok and np.array_equal(cat[..., c2:][real], want_bits(NUM.quantize(p["p1"], fmt), fmt)[real])
    # padding rows: idx 0, dist +inf, weight 0, features 0
    pad = ~real
    inf = np.float32(np.inf).view(np.int32)
    ok = ok and (d[pad] == inf).all() and (dd[pad] == inf).all() and (i[pad] == 0).all() and (ii[pad] == 0).all()
    ok = ok and (ww[pad] == 0).all() and (out[pad] == 0).all() and (cat[pad] == 0).all()
    return bool(ok)


# ---------------------------------------------------------------------------------------- interpolation, gradient
GRAD_MODES = ["atomic_f32", "det_f32", "det_bf16", "det_f16"]


def draw_interp_grad(rs):
    b, n = int(rs.randint(1, 5)), log_n(rs, 1, 8000)
    r = rs.rand()
    m = int(rs.randint(1, 16)) if r < 0.25 else int(rs.randint(16001, 20001)) if r < 0.4 else log_n(rs, 1, 2000)
    c = int(rs.choice(WIDTHS))
    if rs.rand() < 0.5:
        idx = rs.randint(0, m, (b, n, 3)).astype(np.int32)
        src = "uniform"
    else:
        idx = zipf_index(rs, (b, n, 3), m)
        src = "zipf"
    w = rs.random_sample((b, n, 3)).astype(np.float32)
    w[rs.random_sample((b, n, 3)) < 0.1] = 0
    scale = float(rs.choice([1.0, 1.0, 2.0 ** -20, 2.0 ** 6]))
    pts = W.features(b, m, c, int(rs.randint(1 << 30)))
    go = W.features(b, n, c, int(rs.randint(1 << 30))) * np.float32(scale)
    ragged = bool(rs.rand() < 0.6)
    lens = draw_lengths(rs, b, n) if ragged else None
    ls = lens["lengths"] if ragged else [n] * b
    longest = max(int(np.bincount(idx[k, :l].ravel(), minlength=m).max()) for k, l in enumerate(ls))
    return dict(case="interp_grad", b=b, n=n, m=m, c=c, src=src, scale=scale, mode=str(rs.choice(GRAD_MODES)),
                offset=int(rs.randint(0, 2)), lens=lens, longest=longest, idx=idx, w=w, pts=pts, go=go)


def run_interp_grad(p):
    b, n, m, c = p["b"], p["n"], p["m"], p["c"]
    fmt = p["mode"].split("_")[1]
    det = p["mode"] != "atomic_f32"
    lens = p["lens"]
    ls = lens["lengths"] if lens else [n] * b
    idx, w, pts, go = p["idx"], p["w"], p["pts"], p["go"]
    runs = []
    prev = tf_interpolate.DETERMINISTIC_GRAD
    try:
        tf_interpolate.DETERMINISTIC_GRAD = det
        for kind in (("poison", "copy") if lens else ("none", "none")):
            ii, ww = NUM.pad_index_rows(idx, w, ls, kind, m) if lens else (idx, w)
            g = NUM.pad_rows(go, ls, kind) if lens else go
            pt = feat(pts, fmt, p["offset"]).requires_grad_(True)
            out = three_interpolate(pt, T(ii), T(ww), lengths=lengths_arg(lens) if lens else None)
            out.backward(feat(g, fmt, 1 - p["offset"]))
            runs.append((bits(out), bits(pt.grad)))
    finally:
        tf_interpolate.DETERMINISTIC_GRAD = prev
    ok = True
    if det:  # run to run identical, and the padding never matters
        ok = all(np.array_equal(x, y) for x, y in zip(*runs))
    out, grad = runs[0]
    real = np.arange(n)[None, :] < np.asarray(ls)[:, None]
    ptsq, goq = NUM.quantize(pts, fmt), NUM.quantize(go, fmt)
    want = want_bits(O.oracle_three_interpolate(ptsq, idx, w), fmt)
    ok = ok and np.array_equal(out[real], want[real]) and (out[~real] == 0).all()
    for k, l in enumerate(ls):
        o = O.oracle_three_interpolate_grad((1, m, c), idx[k:k + 1, :l], w[k:k + 1, :l], goq[k:k + 1, :l])[0]
        terms = w[k, :l].astype(np.float64).reshape(-1, 1) * np.repeat(goq[k, :l].astype(np.float64), 3, axis=0)
        ref, mass, count = NUM.scatter64(m, idx[k, :l], terms)
        exact = (count <= 256) if det else np.zeros(m, bool)  # lists beyond 256 entries: eight ordered pieces
        ok = ok and check_grad(grad[k], o, ref, mass, count, fmt, exact)
    return bool(ok)


# ------------------------------------------------------------------------------------------- grouping, forward
def draw_group16(rs):
    b, n, c = int(rs.randint(1, 4)), log_n(rs, 1, 5000), int(rs.choice(WIDTHS))
    m, s = log_n(rs, 1, 300), int(rs.choice([1, 3, 8, 16, 32, 64]))
    kind, xyz = cloud(rs, b, n)
    xscale = float(rs.choice([1.0, 1.0, 1e-5, 1e3, 1e5]))  # 1e-5: float16 subnormal differences; 1e5: float16 overflow
    xyz = (xyz * np.float32(xscale)).astype(np.float32)
    new_xyz = xyz[:, rs.randint(0, n, m)].copy() if rs.rand() < 0.5 else free_points(rs, xyz, b, m)
    return dict(case="group16", b=b, n=n, c=c, m=m, s=s, kind=kind, xscale=xscale, fmt=str(rs.choice(list(DTYPES))),
                offset=int(rs.randint(0, 2)), pts=W.features(b, n, c, int(rs.randint(1 << 30))),
                idx=rs.randint(0, n, (b, m, s)).astype(np.int32), xyz=xyz, new_xyz=new_xyz)


def run_group16(p):
    fmt, c, idx = p["fmt"], p["c"], p["idx"]
    pd, di = feat(p["pts"], fmt, p["offset"]), T(idx)
    ptsq = NUM.quantize(p["pts"], fmt)
    wp = want_bits(O.oracle_group_point(ptsq, idx), fmt)
    ok = np.array_equal(bits(group_point(pd, di)), wp)
    diff = (O.oracle_group_point(p["xyz"], idx) - p["new_xyz"][:, :, None, :]).astype(np.float32)  # __fsub_rn
    wx = want_bits(diff, fmt)
    for xyz_first in (True, False):
        cat, gx = group_and_concat(T(p["xyz"]), T(p["new_xyz"]), pd, di, xyz_first=xyz_first)
        cat = bits(cat)
        cx, cp = (cat[..., :3], cat[..., 3:]) if xyz_first else (cat[..., c:], cat[..., :c])
        ok = ok and np.array_equal(cx, wx) and np.array_equal(cp, wp) and np.array_equal(bits(gx), diff.view(np.int32))
    return bool(ok)


# ------------------------------------------------------------------------------------------ grouping, gradient
def draw_group_grad(rs):
    b, c = int(rs.randint(1, 4)), int(rs.choice(WIDTHS))
    if rs.rand() < 0.5:  # real ball queries on duplicate-heavy or lattice clouds: long lists
        n, m = log_n(rs, 64, 4000), log_n(rs, 8, 300)
        s = int(rs.choice([16, 32, 64, 128]))
        src = str(rs.choice(["D", "G"]))
        seed = int(rs.randint(1 << 30))
        if src == "D":
            xyz = W.cloud_duplicates(b, n, seed)
        else:
            xyz = (np.random.RandomState(seed).randint(0, 6, (b, n, 3)) * 0.125).astype(np.float32)
        r = radius_for(rs, xyz, 0.05, 0.5)
        q = xyz[:, rs.randint(0, n, m)].copy()
        idx, _ = _oracle.oracle_query_ball_point(r, s, xyz, q)
    else:
        n, m, s = log_n(rs, 1, 3000), log_n(rs, 1, 300), int(rs.choice([1, 4, 16, 32, 64]))
        src = "zipf"
        xyz = W.cloud_uniform(b, n, int(rs.randint(1 << 30)))
        idx = zipf_index(rs, (b, m, s), n)
    new_xyz = xyz[:, rs.randint(0, n, m)].copy()
    longest = max(int(np.bincount(idx[k].ravel(), minlength=n).max()) for k in range(b))
    return dict(case="group_grad", b=b, n=n, c=c, m=m, s=s, src=src, fmt=str(rs.choice(list(DTYPES))),
                offset=int(rs.randint(0, 2)), xyz_first=bool(rs.rand() < 0.5), longest=longest, idx=idx, xyz=xyz,
                new_xyz=new_xyz, pts=W.features(b, n, c, int(rs.randint(1 << 30))),
                go=W.features(b, m * s, c, int(rs.randint(1 << 30))).reshape(b, m, s, c),
                gcat=W.features(b, m * s, c + 3, int(rs.randint(1 << 30))).reshape(b, m, s, c + 3),
                ggx=W.features(b, m * s, 3, int(rs.randint(1 << 30))).reshape(b, m, s, 3))


def _group_grad_ok(got_bits, g_f32, idx, n, fmt, det):
    """got (b, n, c) against the ordered sums of g_f32 (b, m, s, c) scattered by idx"""
    b = idx.shape[0]
    want = O.oracle_group_point_grad((b, n, g_f32.shape[-1]), idx, g_f32)
    ok = True
    for k in range(b):
        ref, mass, count = NUM.scatter64(n, idx[k].ravel(), g_f32[k].reshape(-1, g_f32.shape[-1]))
        ok = ok and check_grad(got_bits[k], want[k], ref, mass, count, fmt, np.full(n, det))
    return ok


def run_group_grad(p):
    fmt, c, n, idx = p["fmt"], p["c"], p["n"], p["idx"]
    prev = torch.are_deterministic_algorithms_enabled()
    ok = True
    goq, gcq, ggx = NUM.quantize(p["go"], fmt), NUM.quantize(p["gcat"], fmt), p["ggx"]
    lo = 0 if p["xyz_first"] else c
    gfeat = gcq[..., 3:] if p["xyz_first"] else gcq[..., :c]
    gxyz = (gcq[..., lo:lo + 3] + ggx).astype(np.float32)  # what _GroupConcat.backward feeds to group_point_grad
    try:
        for det in (False, True):
            torch.use_deterministic_algorithms(det)
            grads = []
            for _ in range(2 if det else 1):
                pt = feat(p["pts"], fmt, p["offset"]).requires_grad_(True)
                group_point(pt, T(idx)).backward(feat(p["go"], fmt, 1 - p["offset"]))
                pc = feat(p["pts"], fmt, p["offset"]).requires_grad_(True)
                xd = T(p["xyz"]).requires_grad_(True)
                cat, gx = group_and_concat(xd, T(p["new_xyz"]), pc, T(idx), xyz_first=p["xyz_first"])
                torch.autograd.backward([cat, gx], [feat(p["gcat"], fmt, p["offset"]), T(ggx)])
                grads.append((bits(pt.grad), bits(pc.grad), bits(xd.grad)))
                ok = ok and pt.grad.dtype == DTYPES[fmt] and pc.grad.dtype == DTYPES[fmt] and xd.grad.dtype == torch.float32
            if det:
                ok = ok and all(np.array_equal(x, y) for x, y in zip(*grads))
            g_pt, g_pc, g_x = grads[0]
            ok = ok and _group_grad_ok(g_pt, goq, idx, n, fmt, det)
            ok = ok and _group_grad_ok(g_pc, gfeat, idx, n, fmt, det)
            ok = ok and _group_grad_ok(g_x, gxyz, idx, n, "f32", det)
    finally:
        torch.use_deterministic_algorithms(prev)
    return bool(ok)


def draw_gather_grad_det(rs):
    b, n, m = int(rs.randint(1, 5)), log_n(rs, 1, 5000), log_n(rs, 1, 3000)
    idx = rs.randint(0, n, (b, m)).astype(np.int32) if rs.rand() < 0.5 else zipf_index(rs, (b, m), n)
    return dict(case="gather_grad_det", b=b, n=n, m=m, idx=idx, xyz=W.cloud_uniform(b, n, int(rs.randint(1 << 30))),
                go=W.features(b, m, 3, int(rs.randint(1 << 30))))


def run_gather_grad_det(p):
    prev = torch.are_deterministic_algorithms_enabled()
    try:
        torch.use_deterministic_algorithms(True)
        x = T(p["xyz"]).requires_grad_(True)
        out = gather_point(x, T(p["idx"]))
        out.backward(T(p["go"]))
    finally:
        torch.use_deterministic_algorithms(prev)
    ok = np.array_equal(bits(out), O.oracle_gather_point(p["xyz"], p["idx"]).view(np.int32))
    want = O.oracle_gather_point_grad(p["xyz"].shape, p["idx"], p["go"])
    return bool(ok and np.array_equal(bits(x.grad), want.view(np.int32)))


# --------------------------------------------------------------------------------------- split grid ball query
def draw_bq_prebuilt(rs):
    b, n = int(rs.randint(1, 5)), log_n(rs, 2048, 30000)
    m, s = log_n(rs, 1, 600), int(rs.choice([1, 8, 16, 32, 64, 128]))
    kind, xyz = cloud(rs, b, n)
    r = radius_for(rs, xyz, 0.005, 0.3)
    q = xyz[:, rs.randint(0, n, m)].copy() if rs.rand() < 0.5 else free_points(rs, xyz, b, m)
    return dict(case="bq_prebuilt", b=b, n=n, m=m, s=s, r=r, kind=kind, small_n=log_n(rs, 1, 2047), xyz=xyz, q=q)


def run_bq_prebuilt(p):
    lib = _lib.load()
    b, n, m, s, r = p["b"], p["n"], p["m"], p["s"], p["r"]
    x, q = T(p["xyz"]), T(p["q"])
    wsb = int(lib.pn2_query_ball_point_workspace_bytes(b, n))
    ws = torch.empty(max(wsb, 1), dtype=torch.uint8, device=dev)
    idx = torch.empty((b, m, s), dtype=torch.int32, device=dev)
    cnt = torch.empty((b, m), dtype=torch.int32, device=dev)
    cur = torch.cuda.current_stream(dev)
    side = torch.cuda.Stream(dev)
    side.wait_stream(cur)  # x and ws were written on the current stream
    with torch.cuda.stream(side):
        rc_build = lib.pn2_ball_grid_build(b, n, r, s, ptr(x), ptr(ws), wsb, stream_ptr(dev))
    ws.record_stream(side)
    x.record_stream(side)
    built = torch.cuda.Event()
    built.record(side)
    cur.wait_event(built)
    rc_query = lib.pn2_query_ball_point_prebuilt(b, n, m, r, s, ptr(x), ptr(q), ptr(idx), ptr(cnt), ptr(ws), wsb,
                                                 stream_ptr(dev))
    oi, oc = O.oracle_query_ball_point(r, s, p["xyz"], p["q"])
    ok = wsb > 0 and rc_build == 0 and rc_query == 0 and np.array_equal(N(idx), oi) and np.array_equal(N(cnt), oc)
    # where the whole-path entry would fall back to brute force, both halves refuse: fewer than 2048 points, no
    # workspace, a radius at or below 1e-20
    ns = p["small_n"]
    xs = T(p["xyz"][:, :ns])
    refusals = [
        lib.pn2_ball_grid_build(b, ns, r, s, ptr(xs), ptr(ws), ws.numel(), stream_ptr(dev)),
        lib.pn2_query_ball_point_prebuilt(b, ns, m, r, s, ptr(xs), ptr(q), ptr(idx), ptr(cnt), ptr(ws), ws.numel(), stream_ptr(dev)),
        lib.pn2_ball_grid_build(b, n, r, s, ptr(x), None, wsb, stream_ptr(dev)),
        lib.pn2_query_ball_point_prebuilt(b, n, m, r, s, ptr(x), ptr(q), ptr(idx), ptr(cnt), None, wsb, stream_ptr(dev)),
        lib.pn2_ball_grid_build(b, n, 1e-20, s, ptr(x), ptr(ws), wsb, stream_ptr(dev)),
        lib.pn2_query_ball_point_prebuilt(b, n, m, 1e-20, s, ptr(x), ptr(q), ptr(idx), ptr(cnt), ptr(ws), wsb, stream_ptr(dev)),
    ]
    return bool(ok and all(rc == CUDA_ERROR_INVALID_VALUE for rc in refusals))


CASES = ["fps_ragged", "ball_ragged", "layer_ragged", "interp_ragged", "interp_grad", "group16", "group_grad",
         "gather_grad_det", "bq_prebuilt"]
DRAW = {name: globals()["draw_" + name] for name in CASES}
RUN = {name: globals()["run_" + name] for name in CASES}


def draws(seed: int, iterations: int):
    """The parameters ``run(seed, iterations)`` uses, without a device (the run_* functions draw nothing)."""
    rs = np.random.RandomState(seed)
    return [DRAW[CASES[it % len(CASES)]](rs) for it in range(iterations)]


def public(p):
    """the parameters of a case without its input arrays (they follow from the seed and the iteration)"""
    return {k: v for k, v in p.items() if not isinstance(v, np.ndarray)}


def _one(rs, it, seed, counts, fails, calls, catch):
    name = CASES[it % len(CASES)]
    p = DRAW[name](rs)
    before = O.calls
    try:
        ok = RUN[name](p)
    except Exception as e:  # noqa: BLE001 — report the exception as a failure of that case
        if not catch:
            raise
        ok = False
        p = dict(p, error=f"{type(e).__name__}: {e}")
    counts[name] = counts.get(name, 0) + 1
    calls[name] = calls.get(name, 0) + O.calls - before
    if not ok:
        fails.append(dict(public(p), seed=seed, iteration=it))
    return ok, fails[-1] if not ok else None


def run(seed: int, iterations: int, oracle_calls: dict | None = None):
    """``iterations`` random cases (round-robin over CASES); returns (counts, failures).  ``oracle_calls``, if given,
    receives the oracle calls per case."""
    rs = np.random.RandomState(seed)
    counts, fails, calls = {}, [], {} if oracle_calls is None else oracle_calls
    for it in range(iterations):
        _one(rs, it, seed, counts, fails, calls, catch=False)
    return counts, fails


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=float, default=120)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--json", type=str, default=None)
    args = ap.parse_args()
    rs = np.random.RandomState(args.seed)
    counts, fails, calls, secs = {}, [], {}, {}
    t0 = time.time()
    it = 0
    while time.time() - t0 < args.seconds:
        t1 = time.time()
        ok, fail = _one(rs, it, args.seed, counts, fails, calls, catch=True)
        name = CASES[it % len(CASES)]
        secs[name] = secs.get(name, 0.0) + time.time() - t1
        if not ok:
            print("FAIL", json.dumps(fail), flush=True)
        it += 1
    summary = dict(seed=args.seed, seconds=round(time.time() - t0, 1), cases=counts, oracle_calls=calls,
                   case_seconds={k: round(v, 1) for k, v in secs.items()}, failures=fails)
    print(json.dumps(summary))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(summary, f, indent=1)
    sys.exit(1 if fails else 0)


if __name__ == "__main__":
    main()
