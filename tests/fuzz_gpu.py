#!/usr/bin/env python
"""Randomised differential test of every op against the oracle (TEST TOOL, runs on a GPU box).

    python tests/fuzz_gpu.py [--seconds 120] [--seed 0]

Draws random shapes / distributions / radii, runs the CUDA op and the C oracle on the same input and
requires bit-equal outputs (tolerance only where float atomics reorder sums).  Every failing case
is printed with the parameters that reproduce it; exit code 1 on any failure.
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
import numerics as NUM  # noqa: E402
from oracle import oracle as O  # noqa: E402
from pointnet2_b200 import workloads as W  # noqa: E402
from pointnet2_b200 import _lib  # noqa: E402
from pointnet2_b200.sa_layer import ball_group, sample_group, sample_group_msg  # noqa: E402
from pointnet2_b200.tf_grouping import group_point, knn_point, query_ball_point, select_top_k  # noqa: E402
from pointnet2_b200.tf_interpolate import fp_interpolate_concat, three_interpolate, three_nn, three_nn_interpolate  # noqa: E402
from pointnet2_b200.tf_sampling import farthest_point_sample_and_gather, gather_point, prob_sample  # noqa: E402
from pointnet2_b200.pointnet_util import group_and_concat  # noqa: E402

dev = torch.device("cuda:0")  # only dereferenced when a case runs


def T(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


def N(t):
    return t.detach().cpu().numpy()


def cloud(rs, b, n):
    kind = rs.choice(["U", "S", "D", "G", "L"])
    seed = int(rs.randint(1 << 30))
    if kind == "S" and n < 8:
        kind = "U"  # the surface generator needs a few points per shape
    if kind in "USD":
        return kind, W.DISTRIBUTIONS[kind](b, n, seed)
    if kind == "G":  # points on a coarse lattice: many exact ties in every distance
        return kind, (np.random.RandomState(seed).randint(0, 6, (b, n, 3)) * 0.125).astype(np.float32)
    x = np.zeros((b, n, 3), np.float32)  # collinear, unevenly spaced
    x[:, :, 0] = np.sort(np.random.RandomState(seed).random_sample((b, n)).astype(np.float32) ** 3, axis=1)
    return kind, x


def log_n(rs, lo, hi):
    return int(round(np.exp(rs.uniform(np.log(lo), np.log(hi)))))


def case_fps(rs):
    b, n = int(rs.randint(1, 5)), log_n(rs, 1, 40000)
    m = max(1, int(rs.choice([1, 2, n // 7 + 1, n // 2 + 1, n, n + 3])))
    m = min(m, 600)
    kind, xyz = cloud(rs, b, n)
    p = dict(op="fps", b=b, n=n, m=m, kind=kind)
    forced = None
    if rs.random_sample() < 0.25:  # force the register + shared-memory cluster kernel at a random cluster size (2..16)
        ppt = int(rs.choice([44, 48, 52]))
        cmin = max(2, -(-n // (512 * ppt)))
        forced = (512, ppt, int(rs.randint(cmin, 17)))
        p["forced"] = forced
        _lib.load().pn2_set_fps_config(*forced)
    try:
        idx, new_xyz = farthest_point_sample_and_gather(m, T(xyz))
    finally:
        if forced:
            _lib.load().pn2_set_fps_config(0, 0, 0)
    want = O.oracle_fps(m, xyz)
    ok = np.array_equal(N(idx), want) and np.array_equal(N(new_xyz), O.oracle_gather_point(xyz, want))
    ok = ok and np.array_equal(N(gather_point(T(xyz), idx)), N(new_xyz))
    return ok, p


def case_ball(rs):
    b, n = int(rs.randint(1, 5)), log_n(rs, 1, 20000)
    m = log_n(rs, 1, 600)
    s = int(rs.choice([1, 2, 8, 16, 32, 33, 64, 128]))
    kind, xyz = cloud(rs, b, n)
    ext = float(xyz.max() - xyz.min()) + 1e-3
    r = float(np.float32(ext * np.exp(rs.uniform(np.log(0.005), np.log(0.7)))))
    if rs.rand() < 0.5:
        q = xyz[:, rs.randint(0, n, m)].copy()  # queries are data points (set abstraction)
    else:
        q = (xyz.min() + (xyz.max() - xyz.min() + 1e-3) * rs.random_sample((b, m, 3)) * 1.2 - 0.1).astype(np.float32)
    p = dict(op="ball", b=b, n=n, m=m, s=s, r=r, kind=kind)
    idx, cnt = query_ball_point(r, s, T(xyz), T(q))
    oi, oc = O.oracle_query_ball_point(r, s, xyz, q)
    return np.array_equal(N(idx), oi) and np.array_equal(N(cnt), oc), p


def case_group(rs):
    b, n, c = int(rs.randint(1, 4)), log_n(rs, 1, 5000), int(rs.choice([1, 2, 3, 4, 5, 8, 31, 64, 67, 128, 131, 320]))
    m, s = log_n(rs, 1, 300), int(rs.choice([1, 3, 8, 16, 32, 64]))
    pts = W.features(b, n, c, int(rs.randint(1 << 30)))
    idx = rs.randint(0, n, (b, m, s)).astype(np.int32)
    p = dict(op="group", b=b, n=n, c=c, m=m, s=s)
    tp = T(pts).requires_grad_(True)
    out = group_point(tp, T(idx))
    ok = np.array_equal(N(out), O.oracle_group_point(pts, idx))
    go = W.features(b, m * s, c, 5).reshape(b, m, s, c)
    out.backward(T(go))
    # float atomics reorder the sum: the float64 bound on the absolute mass scattered into each element
    got = N(tp.grad)
    ok_grad = True
    for k in range(b):
        ref, mass, count = NUM.scatter64(n, idx[k].ravel(), go[k].reshape(-1, c))
        ok_grad = ok_grad and bool(NUM.within_bound(got[k], ref, mass, np.maximum(count, 1)[:, None], "f32").all())
    p["forward_ok"], p["grad_ok"] = bool(ok), ok_grad
    ok = ok and ok_grad
    # fused centre-subtract + concat, both channel orders
    xyz = W.cloud_uniform(b, n, 6)
    new_xyz = xyz[:, rs.randint(0, n, m)].copy()
    for xyz_first in (True, False):
        cat, gx = group_and_concat(T(xyz), T(new_xyz), T(pts), T(idx), xyz_first=xyz_first)
        wx = O.oracle_group_point(xyz, idx) - new_xyz[:, :, None, :]
        wp = O.oracle_group_point(pts, idx)
        want = np.concatenate([wx, wp] if xyz_first else [wp, wx], -1)
        ok = ok and np.array_equal(N(cat), want) and np.array_equal(N(gx), wx)
    return ok, p


def case_interp(rs):
    b, n, m, c = int(rs.randint(1, 4)), log_n(rs, 1, 6000), log_n(rs, 1, 1500), int(rs.choice([1, 3, 4, 5, 64, 128, 130, 512]))
    k1, xyz1 = cloud(rs, b, n)
    k2, xyz2 = cloud(rs, b, m)
    if rs.rand() < 0.4 and m <= n:
        xyz2 = xyz1[:, :m].copy()  # nested sets as in feature propagation: exact zero distances
    pts = W.features(b, m, c, int(rs.randint(1 << 30)))
    p = dict(op="interp", b=b, n=n, m=m, c=c, kinds=k1 + k2)
    d, i = three_nn(T(xyz1), T(xyz2))
    od, oi = O.oracle_three_nn(xyz1, xyz2)
    ok = np.array_equal(N(d), od) and np.array_equal(N(i), oi)
    dd = np.maximum(od, 1e-10)
    w = ((1.0 / dd) / (1.0 / dd).sum(axis=2, keepdims=True)).astype(np.float32)
    w = np.nan_to_num(w, nan=0.0, posinf=0.0, neginf=0.0).astype(np.float32)
    tp = T(pts).requires_grad_(True)
    out = three_interpolate(tp, T(oi), T(w))
    ok = ok and np.array_equal(N(out), O.oracle_three_interpolate(pts, oi, w))  # bit-exact
    go = W.features(b, n, c, 9)
    out.backward(T(go))
    # the deterministic backward: the oracle's ordered sum bit for bit on lists of up to 256 entries, longer lists
    # (eight ordered pieces) within the float64 bound
    want = O.oracle_three_interpolate_grad(pts.shape, oi, w, go)
    got = N(tp.grad)
    for k in range(b):
        terms = w[k].astype(np.float64).reshape(-1, 1) * np.repeat(go[k].astype(np.float64), 3, axis=0)
        ref, mass, count = NUM.scatter64(m, oi[k], terms)
        short = count <= 256
        ok = ok and np.array_equal(got[k][short], want[k][short])
        ok = ok and bool(NUM.within_bound(got[k], ref, mass, np.maximum(count, 1)[:, None], "f32").all())
    if m >= 3:  # fused front end against the unfused torch weights
        fused = three_nn_interpolate(T(xyz1), T(xyz2), T(pts))
        dist = torch.clamp(d, min=1e-10)
        wt = (1.0 / dist) / (1.0 / dist).sum(dim=2, keepdim=True)
        ok = ok and np.allclose(N(fused), N(three_interpolate(T(pts), i, wt)), atol=1e-5, rtol=1e-5)
    return ok, p


def case_sort(rs):
    b, m, n = int(rs.randint(1, 4)), log_n(rs, 1, 200), log_n(rs, 1, 700)
    k = int(rs.randint(1, min(n, 40) + 1))
    dist = rs.random_sample((b, m, n)).astype(np.float32)
    if rs.rand() < 0.5:
        dist = np.round(dist * 8) / 8  # ties
    p = dict(op="sort", b=b, m=m, n=n, k=k)
    oi, od = select_top_k(k, T(dist))
    wi, wd = O.oracle_selection_sort(k, dist)
    return np.array_equal(N(oi), wi) and np.array_equal(N(od), wd), p


def case_prob(rs):
    b, n, m = int(rs.randint(1, 5)), log_n(rs, 1, 60000), log_n(rs, 1, 3000)
    pr = rs.random_sample((b, n)).astype(np.float32)
    if rs.rand() < 0.5:
        pr[:, rs.randint(0, n, n // 2 + 1)] = 0
    r = rs.random_sample((b, m)).astype(np.float32)
    p = dict(op="prob", b=b, n=n, m=m)
    return np.array_equal(N(prob_sample(T(pr), T(r))), O.oracle_prob_sample(pr, r)), p


def case_layer(rs):
    """The overlapped sampling+grouping layer (and its multi-scale form, and ball_group on its own) against the
    oracle's op-by-op composite."""
    b, n = int(rs.randint(1, 6)), log_n(rs, 1, 12000)
    m = min(max(1, int(rs.choice([1, n // 9 + 1, n // 4 + 1, n, n + 2]))), 400)
    kind, xyz = cloud(rs, b, n)
    ext = float(xyz.max() - xyz.min()) + 1e-3
    scales = int(rs.choice([1, 1, 2, 3]))
    radii = [float(np.float32(ext * np.exp(rs.uniform(np.log(0.01), np.log(0.6))))) for _ in range(scales)]
    ns = [int(rs.choice([1, 4, 16, 32, 64, 128, 150])) for _ in range(scales)]
    center = bool(rs.rand() < 0.5)
    p = dict(op="layer", b=b, n=n, m=m, radii=radii, ns=ns, kind=kind, center=center)
    o_fi = O.oracle_fps(m, xyz)
    o_nx = O.oracle_gather_point(xyz, o_fi)
    x = T(xyz)
    if scales == 1:
        fi, nx, idx, cnt, g = sample_group(m, radii[0], ns[0], x, center=center)
        idxs, cnts, gs = [idx], [cnt], [g]
    else:
        fi, nx, idxs, cnts, gs = sample_group_msg(m, radii, ns, x, center=center)
    ok = np.array_equal(N(fi), o_fi) and np.array_equal(N(nx), o_nx)
    for r, s, idx, cnt, g in zip(radii, ns, idxs, cnts, gs):
        oi, oc = O.oracle_query_ball_point(r, s, xyz, o_nx)
        og = O.oracle_group_point(xyz, oi)
        if center:
            og = og - o_nx[:, :, None, :]
        ok = ok and np.array_equal(N(idx), oi) and np.array_equal(N(cnt), oc) and np.array_equal(N(g), og)
    if n <= 9700:  # the same kernel with free queries
        q = (xyz.min() + (xyz.max() - xyz.min() + 1e-3) * rs.random_sample((b, m, 3)) * 1.2 - 0.1).astype(np.float32)
        idx, cnt, g = ball_group(radii[0], ns[0], x, T(q), center=center)
        oi, oc = O.oracle_query_ball_point(radii[0], ns[0], xyz, q)
        og = O.oracle_group_point(xyz, oi) - (q[:, :, None, :] if center else 0)
        ok = ok and np.array_equal(N(idx), oi) and np.array_equal(N(cnt), oc) and np.array_equal(N(g), og.astype(np.float32))
    return ok, p


def case_knn(rs):
    b, n, m = int(rs.randint(1, 4)), log_n(rs, 1, 3000), log_n(rs, 1, 200)
    k = int(min(n, rs.choice([1, 2, 3, 8, 16, 32, 64, 128])))
    kind, xyz = cloud(rs, b, n)  # G / D / L clouds: exact ties, where the selection sort's swaps decide the order
    q = xyz[:, rs.randint(0, n, m)].copy() if rs.rand() < 0.6 else cloud(rs, b, m)[1]
    p = dict(op="knn", b=b, n=n, m=m, k=k, kind=kind)
    val, idx = knn_point(k, T(xyz), T(q))
    wv, wi = O.oracle_knn_point(k, xyz, q)
    return np.array_equal(N(idx), wi) and np.array_equal(N(val), wv), p


def case_fp(rs):
    """Fused FP front end + concat, and the deterministic gradient of three_interpolate."""
    b, n, m = int(rs.randint(1, 4)), log_n(rs, 1, 5000), log_n(rs, 1, 1200)
    c2, c1 = int(rs.choice([1, 4, 5, 64, 128, 256])), int(rs.choice([0, 0, 3, 4, 64]))
    k1, xyz1 = cloud(rs, b, n)
    k2, xyz2 = cloud(rs, b, m)
    p2, p1 = W.features(b, m, c2, int(rs.randint(1 << 30))), (W.features(b, n, c1, 3) if c1 else None)
    p = dict(op="fp", b=b, n=n, m=m, c2=c2, c1=c1, kinds=k1 + k2)
    got = N(fp_interpolate_concat(T(xyz1), T(xyz2), T(p1) if c1 else None, T(p2)))
    od, oi = O.oracle_three_nn(xyz1, xyz2)
    out, d, i, w = three_nn_interpolate(T(xyz1), T(xyz2), T(p2), return_aux=True)
    ok = np.array_equal(N(d), od) and np.array_equal(N(i), oi)
    ok = ok and np.array_equal(got[..., :c2], O.oracle_three_interpolate(p2, oi, N(w)))  # the kernel's own weights: bit-exact
    if c1:
        ok = ok and np.array_equal(got[..., c2:], p1)
    # deterministic gradient: bit-exact with the reference's accumulation order when no list exceeds 256 entries
    lib = _lib.load()
    go = W.features(b, n, c2, 11)
    wts = np.abs(W.features(b, n, 3, 12)).astype(np.float32)
    gp = torch.empty((b, m, c2), dtype=torch.float32, device=dev)
    wsb = int(lib.pn2_three_interpolate_grad_det_workspace_bytes(b, n, m))
    ws = torch.empty(wsb, dtype=torch.uint8, device=dev)
    tg, ti, tw = T(go), T(oi), T(wts)
    rc = lib.pn2_three_interpolate_grad_det(b, n, c2, m, tg.data_ptr(), ti.data_ptr(), tw.data_ptr(), gp.data_ptr(), ws.data_ptr(), wsb, None)
    torch.cuda.synchronize()
    want = O.oracle_three_interpolate_grad((b, m, c2), oi, wts, go)
    longest = max(int(np.bincount(oi[j].ravel(), minlength=m).max()) for j in range(b))
    if longest <= 256:
        ok = ok and rc == 0 and np.array_equal(N(gp), want)
    else:
        mass = O.oracle_three_interpolate_grad((b, m, c2), oi, wts, np.abs(go))
        ok = ok and rc == 0 and bool((np.abs(N(gp) - want) <= 1e-5 * mass + 1e-6).all())
    p["longest_list"] = longest
    return ok, p


CASES = [case_fps, case_ball, case_group, case_interp, case_sort, case_prob, case_layer, case_knn, case_fp]


def run(seed: int, iterations: int):
    """`iterations` random cases (round-robin over the ops); returns (counts, failures)."""
    rs = np.random.RandomState(seed)
    counts, fails = {}, []
    for it in range(iterations):
        fn = CASES[it % len(CASES)]
        ok, p = fn(rs)
        counts[p["op"]] = counts.get(p["op"], 0) + 1
        if not ok:
            fails.append(p)
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
        fn = CASES[it % len(CASES)]
        it += 1
        try:
            ok, p = fn(rs)
        except Exception as e:  # noqa: BLE001 — report the exception as a failure of that op
            ok, p = False, dict(op=fn.__name__, error=f"{type(e).__name__}: {e}")
        counts[p["op"]] = counts.get(p["op"], 0) + 1
        if not ok:
            fails.append(p)
            print("FAIL", json.dumps(p), flush=True)
    summary = dict(seed=args.seed, seconds=round(time.time() - t0, 1), cases=counts, failures=fails)
    print(json.dumps(summary))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(summary, f, indent=1)
    sys.exit(1 if fails else 0)


if __name__ == "__main__":
    main()
