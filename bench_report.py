"""Per-kernel tables and tuning sweeps (NOT the driver contract — that is bench.py's default mode).

    python bench.py --report gpurun_out/report.json     # every BASELINE.json config, per kernel
    python bench.py --fps-sweep                          # FPS kernel variants (threads, pts/thread, cluster)
    python bench.py --bq-sweep                           # ball query lanes-per-query

All timings: CUDA events on the launching stream, >= 3 warm-ups, L2 flushed (256 MiB memset)
before every timed launch, median of the repeats.
"""
from __future__ import annotations

import json
import os
import statistics
import sys

import numpy as np


def _setup():
    import torch
    from pointnet2_b200 import _lib
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    lib = _lib.load()
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    return torch, lib, dev, flush


def timeit(torch, flush, fn, reps=10, warm=3):
    st = torch.cuda.current_stream()
    for _ in range(warm):
        fn()
    ts = []
    for _ in range(reps):
        flush.zero_()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(st)
        fn()
        b.record(st)
        b.synchronize()
        ts.append(a.elapsed_time(b))
    return statistics.median(ts)


def timeit_batch(torch, fn, min_ms=4.0, warm=3):
    """Back-to-back launches (keeps the SM clock at its loaded frequency; the FPS input is tiny, so
    L2 residency is irrelevant to it): returns the mean ms per launch over >= min_ms of work."""
    st = torch.cuda.current_stream()
    for _ in range(warm):
        fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record(st)
    fn()
    b.record(st)
    b.synchronize()
    one = max(a.elapsed_time(b), 1e-3)
    reps = int(min(max(min_ms / one, 3), 400))
    a.record(st)
    for _ in range(reps):
        fn()
    b.record(st)
    b.synchronize()
    return a.elapsed_time(b) / reps


def spin_up(torch, dev, ms=300):
    """Keep the GPU busy for a while so the clocks are at their loaded frequency."""
    x = torch.randn(4096, 4096, device=dev)
    t0 = torch.cuda.Event(enable_timing=True)
    t1 = torch.cuda.Event(enable_timing=True)
    t0.record()
    while True:
        for _ in range(20):
            x = (x @ x).clamp_(-1, 1)
        t1.record()
        t1.synchronize()
        if t0.elapsed_time(t1) > ms:
            break


def fps_sweep(out_path=None):
    torch, lib, dev, flush = _setup()
    from pointnet2_b200 import workloads as W
    rows = []
    spin_up(torch, dev)
    cases = [(32, 128, 64), (32, 512, 128), (32, 1024, 512), (32, 2048, 512), (32, 4096, 1024), (16, 8192, 1024), (2, 8192, 1024),
             (8, 16384, 4096), (8, 65536, 2048), (1, 65536, 2048), (8, 262144, 512), (1, 262144, 512)]
    if os.environ.get("PN2_SWEEP_SMALL"):
        cases = [c for c in cases if c[1] <= 8192]
    if os.environ.get("PN2_SWEEP_LARGE"):
        cases = [(32, 4096, 1024), (8, 16384, 4096), (1, 16384, 4096), (8, 65536, 2048), (1, 65536, 2048), (8, 131072, 512), (8, 262144, 256), (1, 262144, 256)]
    variants = [(128, 1, 1), (256, 1, 1), (512, 1, 1), (512, 2, 1), (512, 4, 1), (512, 8, 1), (512, 16, 1), (1024, 1, 1),
                (1024, 2, 1), (1024, 4, 1), (1024, 8, 1)]
    variants += [(128, p, 1) for p in (2, 4, 8, 16, 32)] + [(256, p, 1) for p in (2, 4, 8, 16, 32)]
    for C in (2, 4, 8, 16):
        for (t, p) in [(512, 1), (512, 2), (512, 4), (512, 8), (512, 16), (512, 32), (1024, 2), (1024, 4), (1024, 8),
                       (256, 2), (256, 4), (256, 8), (256, 16), (256, 32), (128, 4), (128, 8), (128, 16), (128, 32)]:
            if (C * t) % 512 == 0:
                variants.append((t, p, C))
    for (b, n, m) in cases:
        xyz = torch.from_numpy(W.cloud_uniform(b, n, 100)).to(dev)
        idx = torch.empty((b, m), dtype=torch.int32, device=dev)
        nx = torch.empty((b, m, 3), dtype=torch.float32, device=dev)
        ref = None
        for (t, p, c) in [(0, 0, 0)] + variants:
            cc = c if c > 0 else 1
            if t and (t * p * cc < n or t * p * cc > 16 * n or b * cc > 8 * 132):
                continue
            lib.pn2_set_fps_config(t, p, c)
            rc = [0]

            def fn():
                rc[0] |= lib.pn2_fps_gather(b, n, m, xyz.data_ptr(), None, idx.data_ptr(), nx.data_ptr(), None)
            try:
                ms = timeit_batch(torch, fn)
            except Exception as e:  # noqa: BLE001
                rows.append(dict(b=b, n=n, m=m, cfg=[t, p, c], error=str(e)))
                continue
            finally:
                lib.pn2_set_fps_config(0, 0, 0)
            if rc[0]:
                rows.append(dict(b=b, n=n, m=m, cfg=[t, p, c], error=f"rc={rc[0]}"))
                continue
            if ref is None:
                ref = idx.clone()
            ok = bool(torch.equal(ref, idx))
            row = dict(b=b, n=n, m=m, cfg=[t, p, c], ms=ms, us_per_iter=1e3 * ms / (m - 1), same_as_default=ok,
                       pairs_per_s=b * (m - 1) * n / (ms * 1e-3))
            rows.append(row)
            print(json.dumps(row), flush=True)
    if out_path:
        json.dump(rows, open(out_path, "w"), indent=1)
    return rows


def bq_sweep(out_path=None):
    torch, lib, dev, flush = _setup()
    from pointnet2_b200 import workloads as W
    rows = []
    cases = [("U", 32, 4096, 1024, 0.001, 32), ("U", 32, 4096, 1024, 0.1, 32), ("S", 32, 1024, 512, 0.1, 16), ("S", 32, 1024, 512, 0.4, 128),
             ("S", 32, 512, 128, 0.8, 128), ("D", 2, 8192, 1024, 0.1, 32), ("D", 16, 8192, 1024, 0.1, 32),
             ("U", 8, 16384, 4096, 0.1, 32), ("U", 1, 65536, 16384, 0.1, 32)]
    for (gen, b, n, m, r, s) in cases:
        xyz = torch.from_numpy(W.DISTRIBUTIONS[gen](b, n, 100)).to(dev)
        fi = torch.empty((b, m), dtype=torch.int32, device=dev)
        nx = torch.empty((b, m, 3), dtype=torch.float32, device=dev)
        lib.pn2_fps_gather(b, n, m, xyz.data_ptr(), None, fi.data_ptr(), nx.data_ptr(), None)
        idx = torch.empty((b, m, s), dtype=torch.int32, device=dev)
        cnt = torch.empty((b, m), dtype=torch.int32, device=dev)
        wsb = int(lib.pn2_query_ball_point_workspace_bytes(b, n))
        if wsb:
            ws = torch.empty(wsb, dtype=torch.uint8, device=dev)
            ms = timeit(torch, flush, lambda: lib.pn2_query_ball_point_ws(b, n, m, r, s, xyz.data_ptr(), nx.data_ptr(), idx.data_ptr(),
                                                                          cnt.data_ptr(), ws.data_ptr(), wsb, None), reps=7)
            row = dict(gen=gen, b=b, n=n, m=m, r=r, s=s, group=-1, ms=ms, mean_cnt=float(cnt.float().mean()),
                       GBps=W.bytes_ball_query(b, n, m, s) / (ms * 1e-3) / 1e9, grid_flags=int(ws.view(torch.int32)[::(len(ws) // 4) // b][:b].sum()))
            rows.append(row)
            print(json.dumps(row), flush=True)
        for g in (0, 1, 2, 4, 8, 16, 32):
            lib.pn2_set_bq_group(g)
            ms = timeit(torch, flush, lambda: lib.pn2_query_ball_point(b, n, m, r, s, xyz.data_ptr(), nx.data_ptr(),
                                                                       idx.data_ptr(), cnt.data_ptr(), None), reps=7)
            lib.pn2_set_bq_group(0)
            row = dict(gen=gen, b=b, n=n, m=m, r=r, s=s, group=g, ms=ms, mean_cnt=float(cnt.float().mean()),
                       GBps=W.bytes_ball_query(b, n, m, s) / (ms * 1e-3) / 1e9)
            rows.append(row)
            print(json.dumps(row), flush=True)
    if out_path:
        json.dump(rows, open(out_path, "w"), indent=1)
    return rows


def config_rows(torch, lib, dev, flush, peak, kind, world=1, rank=0, reps=10, full=True, echo=True):
    """Per-kernel time, algorithmic GB/s and fraction of the measured HBM peak for BASELINE.json's
    configs, as a list of dict rows (deterministic order: the same on every rank).

    full=True (bench.py --report): cfg2 in three input distributions, cfg3, cfg4 at B=16 and at the
    2-clouds-per-GPU shard, cfg5 at B=8 and B=1, with gradients and the brute-force-only ball query.
    full=False (the `configs` block of bench.py's driver line): cfg3, cfg4 and cfg5 at THIS rank's
    shard of the batch (B/world clouds: cfg4 16/world, cfg5 8/world), forward kernels only.
    """
    from pointnet2_b200 import workloads as W
    rows = []
    lane_rate = 132 * 128 * 1.98e9  # H100 SXM FP32 lanes x max SM clock: the secondary bound for the pair-evaluation kernels

    def add(cfg, kernel, ms, nbytes, extra=None):
        gbps = nbytes / (ms * 1e-3) / 1e9
        row = dict(config=cfg, kernel=kernel, ms=ms, algorithmic_MB=nbytes / 1e6, GBps=gbps, frac_of_peak=gbps / peak)
        if full:
            row["peak"] = f"{peak} GB/s of {kind}"
        if extra:
            row.update(extra)
            if "pairs_per_s" in extra:  # point-pair evaluations per FP32-lane-cycle (1 = one pair per lane per clock)
                row["pairs_per_lane_cycle"] = extra["pairs_per_s"] / lane_rate
        rows.append(row)
        if echo:
            print(json.dumps(row), flush=True)

    def T(a):
        return torch.from_numpy(np.ascontiguousarray(a)).to(dev)

    # what the harness itself costs: a kernel that moves 28 bytes, timed like every row below (event pair around
    # one launch, right after the 256 MiB L2-flush memset).  Every row's ms contains this floor; a kernel that
    # moves tens of MB cannot show more than bytes / (ms - floor) of the HBM peak however good it is.
    one = torch.zeros((1, 1, 3), dtype=torch.float32, device=dev)
    onei = torch.zeros((1, 1), dtype=torch.int32, device=dev)
    oneo = torch.empty((1, 1, 3), dtype=torch.float32, device=dev)
    ms = timeit(torch, flush, lambda: lib.pn2_gather_point(1, 1, 1, one.data_ptr(), onei.data_ptr(), oneo.data_ptr(), None), reps=max(reps, 9))
    add("harness", "timing floor: a 1-thread kernel under the same event pair + L2 flush", ms, 28)

    BF16 = 1  # PN2_BF16

    def sa_layer(tag, xyz, feats, m, r, s, xyz_first=True, bf16_rows=False):
        b, n, _ = xyz.shape
        fi = torch.empty((b, m), dtype=torch.int32, device=dev)
        nx = torch.empty((b, m, 3), dtype=torch.float32, device=dev)
        ms = timeit(torch, flush, lambda: lib.pn2_fps_gather(b, n, m, xyz.data_ptr(), None, fi.data_ptr(), nx.data_ptr(), None), reps=reps)
        add(tag, "fps+gather", ms, W.bytes_fps(b, n, m, True), dict(pairs_per_s=b * (m - 1) * n / (ms * 1e-3), us_per_iter=1e3 * ms / max(m - 1, 1)))
        idx = torch.empty((b, m, s), dtype=torch.int32, device=dev)
        cnt = torch.empty((b, m), dtype=torch.int32, device=dev)
        wsb = int(lib.pn2_query_ball_point_workspace_bytes(b, n))
        ws = torch.empty(max(wsb, 1), dtype=torch.uint8, device=dev)
        ms = timeit(torch, flush, lambda: lib.pn2_query_ball_point_ws(b, n, m, r, s, xyz.data_ptr(), nx.data_ptr(), idx.data_ptr(), cnt.data_ptr(),
                                                                      ws.data_ptr() if wsb else None, wsb, None), reps=reps)
        add(tag, f"query_ball_point r={r} S={s}", ms, W.bytes_ball_query(b, n, m, s), dict(mean_cnt=float(cnt.float().mean())))
        if full:
            lib.pn2_set_bq_mode(1)
            ms = timeit(torch, flush, lambda: lib.pn2_query_ball_point_ws(b, n, m, r, s, xyz.data_ptr(), nx.data_ptr(), idx.data_ptr(), cnt.data_ptr(),
                                                                          ws.data_ptr() if wsb else None, wsb, None), reps=reps)
            lib.pn2_set_bq_mode(0)
            add(tag, f"query_ball_point (brute force only) r={r} S={s}", ms, W.bytes_ball_query(b, n, m, s))
        g = torch.empty((b, m, s, 3), dtype=torch.float32, device=dev)
        ms = timeit(torch, flush, lambda: lib.pn2_group_point(b, n, 3, m, s, xyz.data_ptr(), idx.data_ptr(), g.data_ptr(), None), reps=reps)
        add(tag, f"group_point C=3 S={s}", ms, W.bytes_group(b, n, m, s, 3))
        if lib.pn2_ball_group_fits(n):
            ms = timeit(torch, flush, lambda: lib.pn2_ball_group(b, n, m, r, s, xyz.data_ptr(), nx.data_ptr(), idx.data_ptr(), cnt.data_ptr(), g.data_ptr(), 1, None), reps=reps)
            add(tag, f"ball_group (query_ball_point + group_point(xyz) - centre, one launch) r={r} S={s}", ms,
                W.bytes_ball_query(b, n, m, s) + 12 * b * m * s)
        dwsb = int(lib.pn2_sa_layer_device_workspace_bytes(b, n, m, s))
        dws = torch.empty(max(dwsb, 1), dtype=torch.uint8, device=dev)
        ms = timeit(torch, flush, lambda: lib.pn2_sa_layer_device(b, n, m, r, s, xyz.data_ptr(), fi.data_ptr(), nx.data_ptr(), idx.data_ptr(), cnt.data_ptr(),
                                                                  g.data_ptr(), 1, dws.data_ptr() if dwsb else None, dwsb, None), reps=reps)
        add(tag, f"sa_layer_device (fps+gather+ball query+group xyz, overlapped when it applies) r={r} S={s}", ms, W.bytes_sa_layer(b, n, m, s),
            dict(points_per_s=b * n / (ms * 1e-3)))
        c = 0 if feats is None else feats.shape[2]
        if c:
            gf = torch.empty((b, m, s, c), dtype=torch.float32, device=dev)
            ms = timeit(torch, flush, lambda: lib.pn2_group_point(b, n, c, m, s, feats.data_ptr(), idx.data_ptr(), gf.data_ptr(), None), reps=reps)
            add(tag, f"group_point C={c} S={s}", ms, W.bytes_group(b, n, m, s, c))
            del gf
        if c and full and bf16_rows:  # the same gather on bfloat16 features
            fh = feats.to(torch.bfloat16)
            gh = torch.empty((b, m, s, c), dtype=torch.bfloat16, device=dev)
            ms = timeit(torch, flush, lambda: lib.pn2_group_point_typed(BF16, b, n, c, m, s, fh.data_ptr(), idx.data_ptr(), gh.data_ptr(), None), reps=reps)
            add(tag, f"group_point bf16 C={c} S={s}", ms, W.bytes_group(b, n, m, s, c, esz=2))
            del gh
        if c and full:  # backward of the gather: atomic scatter-add (the caller's zero-fill is part of the op)
            go = torch.randn((b, m, s, c), dtype=torch.float32, device=dev)
            gp = torch.empty((b, n, c), dtype=torch.float32, device=dev)

            def grad():
                gp.zero_()
                lib.pn2_group_point_grad(b, n, c, m, s, go.data_ptr(), idx.data_ptr(), gp.data_ptr(), None)
            ms = timeit(torch, flush, grad, reps=reps)
            add(tag, f"group_point_grad C={c} S={s} (incl. zero-fill)", ms, 4 * b * m * s + 4 * b * m * s * c + 2 * 4 * b * n * c)
            del go, gp
        if c:
            out = torch.empty((b, m, s, 3 + c), dtype=torch.float32, device=dev)
            ms = timeit(torch, flush, lambda: lib.pn2_group_concat(b, n, c, m, s, xyz.data_ptr(), nx.data_ptr(), feats.data_ptr(),
                                                                   idx.data_ptr(), 1 if xyz_first else 0, out.data_ptr(), None, None), reps=reps)
            add(tag, f"group_concat (fused tail) C={c}+3 S={s}", ms, 4 * b * m * s + 4 * b * min(n, m * s) * (c + 3) + 4 * b * m * s * (c + 3))
            del out
            if full and bf16_rows:
                oh = torch.empty((b, m, s, 3 + c), dtype=torch.bfloat16, device=dev)
                ms = timeit(torch, flush, lambda: lib.pn2_group_concat_typed(BF16, b, n, c, m, s, xyz.data_ptr(), nx.data_ptr(), fh.data_ptr(),
                                                                             idx.data_ptr(), 1 if xyz_first else 0, oh.data_ptr(), None, None), reps=reps)
                add(tag, f"group_concat (fused tail) bf16 C={c}+3 S={s}", ms, W.bytes_group_concat(b, n, m, s, c, esz=2))
                del oh, fh
        return nx

    # cfg2 in the three input distributions (the driver line's own workload: --report only)
    c2 = W.CFG2_SSG_SA
    if full:
        for gen in ("U", "S", "D"):
            sa_layer(f"cfg2[{gen}]", T(W.DISTRIBUTIONS[gen](c2["b"], c2["n"], 100)), None, c2["npoint"], c2["radius"], c2["nsample"])
    # cfg3 MSG stack (B=32 per GPU: replicas under torchrun, like the driver line's cfg2)
    c3 = W.CFG3_MSG
    xyz = T(W.cloud_surface(c3["b"], c3["n"], 100 + rank))
    L1, L2 = c3["layers"]
    nx1 = None
    for r, s in zip(L1["radii"], L1["nsamples"]):
        nx1 = sa_layer("cfg3.L1", xyz, None, L1["npoint"], r, s, xyz_first=False)
    feats = T(W.features(c3["b"], L1["npoint"], L2["c"], 103))
    for r, s in zip(L2["radii"], L2["nsamples"]):
        sa_layer("cfg3.L2", nx1, feats, L2["npoint"], r, s, xyz_first=False, bf16_rows=True)

    def msg_layer(tag, x, L):
        """One pn2_sa_layer_msg_device call: the sampling pass + all three scales' ball query and xyz grouping."""
        import ctypes
        b, n, _ = x.shape
        m, k = L["npoint"], len(L["radii"])
        fi = torch.empty((b, m), dtype=torch.int32, device=dev)
        nx = torch.empty((b, m, 3), dtype=torch.float32, device=dev)
        idx = [torch.empty((b, m, s), dtype=torch.int32, device=dev) for s in L["nsamples"]]
        cnt = [torch.empty((b, m), dtype=torch.int32, device=dev) for _ in L["nsamples"]]
        grp = [torch.empty((b, m, s, 3), dtype=torch.float32, device=dev) for s in L["nsamples"]]
        radii = (ctypes.c_float * k)(*L["radii"])
        ns = (ctypes.c_int * k)(*L["nsamples"])
        pi = (ctypes.c_void_p * k)(*[t.data_ptr() for t in idx])
        pc = (ctypes.c_void_p * k)(*[t.data_ptr() for t in cnt])
        pg = (ctypes.c_void_p * k)(*[t.data_ptr() for t in grp])
        ms = timeit(torch, flush, lambda: lib.pn2_sa_layer_msg_device(b, n, m, k, radii, ns, x.data_ptr(), fi.data_ptr(), nx.data_ptr(), pi, pc, pg, 1,
                                                                      None, 0, None), reps=reps)
        nbytes = W.bytes_fps(b, n, m) + W.bytes_gather(b, m) + sum(W.bytes_ball_query(b, n, m, s) + W.bytes_group(b, n, m, s, 3) for s in L["nsamples"])
        add(tag, f"sa_layer_msg_device (one sampling pass + {k} scales of ball query + group xyz, overlapped)", ms, nbytes,
            dict(points_per_s=b * n / (ms * 1e-3)))

    msg_layer("cfg3.L1", xyz, L1)
    msg_layer("cfg3.L2", nx1, L2)
    del feats
    # cfg4 sem-seg: SA chain + FP chain.  --report: B=16 on one GPU and the 2-clouds-per-GPU shard;
    # driver line: this rank's shard of the 16 clouds
    c4 = W.CFG4_SEMSEG
    for b in ((16, 2) if full else (max(1, c4["b"] // world),)):
        cur = T(W.cloud_duplicates(b, c4["n"], 100 + rank))
        levels = [cur]
        for L in c4["sa"]:
            f = T(W.features(b, cur.shape[1], L["c"], 104)) if L["c"] else None
            cur = sa_layer(f"cfg4[B={b}].SA{L['npoint']}", cur, f, L["npoint"], L["radius"], L["nsample"])
            levels.append(cur)
        for F in c4["fp"]:
            x1 = [l for l in levels if l.shape[1] == F["n"]][0]
            x2 = [l for l in levels if l.shape[1] == F["m"]][0]
            p2 = T(W.features(b, F["m"], F["c"], 105))
            n_, m_, c_ = F["n"], F["m"], F["c"]
            d = torch.empty((b, n_, 3), dtype=torch.float32, device=dev)
            i = torch.empty((b, n_, 3), dtype=torch.int32, device=dev)
            ms = timeit(torch, flush, lambda: lib.pn2_three_nn(b, n_, m_, x1.data_ptr(), x2.data_ptr(), d.data_ptr(), i.data_ptr(), None), reps=reps)
            add(f"cfg4[B={b}].FP{n_}<-{m_}", "three_nn", ms, W.bytes_three_nn(b, n_, m_), dict(pairs_per_s=b * n_ * m_ / (ms * 1e-3)))
            w = torch.full((b, n_, 3), 1 / 3, dtype=torch.float32, device=dev)
            o = torch.empty((b, n_, c_), dtype=torch.float32, device=dev)
            ms = timeit(torch, flush, lambda: lib.pn2_three_interpolate(b, m_, c_, n_, p2.data_ptr(), i.data_ptr(), w.data_ptr(), o.data_ptr(), None), reps=reps)
            add(f"cfg4[B={b}].FP{n_}<-{m_}", f"three_interpolate C={c_}", ms, W.bytes_three_interpolate(b, n_, m_, c_))
            if full:
                go = torch.randn((b, n_, c_), dtype=torch.float32, device=dev)
                gp = torch.empty((b, m_, c_), dtype=torch.float32, device=dev)

                def igrad():
                    gp.zero_()
                    lib.pn2_three_interpolate_grad(b, n_, c_, m_, go.data_ptr(), i.data_ptr(), w.data_ptr(), gp.data_ptr(), None)
                ms = timeit(torch, flush, igrad, reps=reps)
                add(f"cfg4[B={b}].FP{n_}<-{m_}", f"three_interpolate_grad C={c_} (atomics, incl. zero-fill)", ms, 2 * 4 * b * m_ * c_ + 24 * b * n_ + 4 * b * n_ * c_)
                if hasattr(lib, "pn2_three_interpolate_grad_det"):
                    dwb = int(lib.pn2_three_interpolate_grad_det_workspace_bytes(b, n_, m_))
                    dw = torch.empty(max(dwb, 1), dtype=torch.uint8, device=dev)
                    ms = timeit(torch, flush, lambda: lib.pn2_three_interpolate_grad_det(b, n_, c_, m_, go.data_ptr(), i.data_ptr(), w.data_ptr(), gp.data_ptr(),
                                                                                         dw.data_ptr(), dwb, None), reps=reps)
                    add(f"cfg4[B={b}].FP{n_}<-{m_}", f"three_interpolate_grad C={c_} (deterministic, inverse index)", ms,
                        2 * 4 * b * m_ * c_ + 24 * b * n_ + 4 * b * n_ * c_)
            ms = timeit(torch, flush, lambda: lib.pn2_three_nn_interpolate(b, n_, m_, c_, x1.data_ptr(), x2.data_ptr(), p2.data_ptr(), o.data_ptr(), None, None, None, None), reps=reps)
            add(f"cfg4[B={b}].FP{n_}<-{m_}", f"three_nn_interpolate (fused) C={c_}", ms, 12 * b * n_ + 12 * b * m_ + 4 * b * m_ * c_ + 4 * b * n_ * c_)
            if full:  # bfloat16 features beside float32: three_interpolate, its deterministic gradient, the FP front end
                tag4 = f"cfg4[B={b}].FP{n_}<-{m_}"
                p2h, goh = p2.to(torch.bfloat16), go.to(torch.bfloat16)
                oh = torch.empty((b, n_, c_), dtype=torch.bfloat16, device=dev)
                gph = torch.empty((b, m_, c_), dtype=torch.bfloat16, device=dev)
                ms = timeit(torch, flush, lambda: lib.pn2_three_interpolate_typed(BF16, b, m_, c_, n_, p2h.data_ptr(), i.data_ptr(), w.data_ptr(), oh.data_ptr(), None), reps=reps)
                add(tag4, f"three_interpolate bf16 C={c_}", ms, W.bytes_three_interpolate(b, n_, m_, c_, esz=2))
                ms = timeit(torch, flush, lambda: lib.pn2_three_interpolate_grad_det_typed(BF16, b, n_, c_, m_, goh.data_ptr(), i.data_ptr(), w.data_ptr(),
                                                                                           gph.data_ptr(), dw.data_ptr(), dwb, None), reps=reps)
                add(tag4, f"three_interpolate_grad bf16 C={c_} (deterministic, inverse index)", ms, W.bytes_three_interpolate_grad(b, n_, m_, c_, esz=2))
                # points1: the dense level's own features, as the sem-seg network feeds them (none at the input level)
                c1 = c4["sa"][next(k for k, lv in enumerate(levels) if lv is x1)]["c"]
                for dt, code, esz, name in ((torch.float32, 0, 4, ""), (torch.bfloat16, BF16, 2, " bf16")):
                    p1 = T(W.features(b, n_, c1, 106)).to(dt) if c1 else None
                    p2d = p2 if dt == torch.float32 else p2h
                    of = torch.empty((b, n_, c_ + c1), dtype=dt, device=dev)
                    ms = timeit(torch, flush, lambda: lib.pn2_fp_interpolate_concat_typed(code, b, n_, m_, c_, c1, x1.data_ptr(), x2.data_ptr(),
                                                                                          p1.data_ptr() if c1 else None, p2d.data_ptr(), of.data_ptr(), None), reps=reps)
                    add(tag4, f"fp_interpolate_concat{name} C={c_}+{c1}", ms, W.bytes_fp_interpolate_concat(b, n_, m_, c_, c1, esz=esz))
                    del p1, of
                del p2h, goh, oh, gph
    if full:
        # n3: knn_point at cfg2's shape — one tiled top-k kernel against the reference's composite
        # (materialised (b,m,n) matrix + selection sort of whole rows, here as torch ops + pn2_selection_sort)
        b, n_, m_, k_ = 32, 4096, 1024, 32
        x1 = T(W.cloud_uniform(b, n_, 141))
        x2 = x1[:, :m_].contiguous()
        val = torch.empty((b, m_, k_), dtype=torch.float32, device=dev)
        ind = torch.empty((b, m_, k_), dtype=torch.int32, device=dev)
        ms = timeit(torch, flush, lambda: lib.pn2_knn_point(b, n_, m_, k_, x1.data_ptr(), x2.data_ptr(), val.data_ptr(), ind.data_ptr(), None), reps=reps)
        add("knn[B=32,N=4096,M=1024,k=32]", "knn_point (tiled top-k, no matrix)", ms, 12 * b * n_ + 12 * b * m_ + 8 * b * m_ * k_,
            dict(pairs_per_s=b * m_ * n_ / (ms * 1e-3)))
        bs = 8  # the composite needs 3 (b,m,n) tensors + the (b,m,n,3) differences: 8 clouds at a time
        x1s, x2s = x1[:bs].contiguous(), x2[:bs].contiguous()
        outi = torch.empty((bs, m_, n_), dtype=torch.int32, device=dev)
        outv = torch.empty((bs, m_, n_), dtype=torch.float32, device=dev)

        def composite():
            diff = x1s.unsqueeze(1) - x2s.unsqueeze(2)
            dist = (diff * diff).sum(-1)
            lib.pn2_selection_sort(bs, n_, m_, k_, dist.data_ptr(), outi.data_ptr(), outv.data_ptr(), None)
        ms = timeit(torch, flush, composite, reps=3, warm=1)
        add("knn[B=8 of 32,N=4096,M=1024,k=32]", "reference composite: (b,m,n) matrix (torch) + selection sort (pn2_selection_sort), 8 of the 32 clouds", ms,
            12 * bs * n_ + 12 * bs * m_ + 8 * bs * m_ * k_, dict(pairs_per_s=bs * m_ * n_ / (ms * 1e-3)))
        del x1, x2, x1s, x2s, outi, outv
        # the same last FP layer on a UNIFORM cloud (no coincident points): the inverse-index gradient's normal case —
        # cfg4's duplicate-heavy clouds make three known points collect thousands of contributions each
        b, n_, m_, c_ = 16, 8192, 1024, 128
        x1 = T(W.cloud_uniform(b, n_, 131))
        x2 = x1[:, :m_].contiguous()
        d = torch.empty((b, n_, 3), dtype=torch.float32, device=dev)
        i = torch.empty((b, n_, 3), dtype=torch.int32, device=dev)
        lib.pn2_three_nn(b, n_, m_, x1.data_ptr(), x2.data_ptr(), d.data_ptr(), i.data_ptr(), None)
        w = torch.full((b, n_, 3), 1 / 3, dtype=torch.float32, device=dev)
        go = torch.randn((b, n_, c_), dtype=torch.float32, device=dev)
        gp = torch.empty((b, m_, c_), dtype=torch.float32, device=dev)

        def igrad_u():
            gp.zero_()
            lib.pn2_three_interpolate_grad(b, n_, c_, m_, go.data_ptr(), i.data_ptr(), w.data_ptr(), gp.data_ptr(), None)
        nb = 2 * 4 * b * m_ * c_ + 24 * b * n_ + 4 * b * n_ * c_
        add("uniform[B=16].FP8192<-1024", "three_interpolate_grad C=128 (atomics, incl. zero-fill)", timeit(torch, flush, igrad_u, reps=reps), nb)
        dwb = int(lib.pn2_three_interpolate_grad_det_workspace_bytes(b, n_, m_))
        dw = torch.empty(dwb, dtype=torch.uint8, device=dev)
        ms = timeit(torch, flush, lambda: lib.pn2_three_interpolate_grad_det(b, n_, c_, m_, go.data_ptr(), i.data_ptr(), w.data_ptr(), gp.data_ptr(),
                                                                             dw.data_ptr(), dwb, None), reps=reps)
        add("uniform[B=16].FP8192<-1024", "three_interpolate_grad C=128 (deterministic, inverse index)", ms, nb)
        del x1, x2, go, gp, dw
    # cfg5 sweep: FPS + gather + ball query.  --report: B=8 and B=1; driver line: this rank's 8/world clouds
    c5 = W.CFG5_SWEEP
    for n in c5["ns"]:
        for b in ((8, 1) if full else (max(1, c5["b"] // world),)):
            if n >= 262144 and b == 8 and os.environ.get("PN2_REPORT_BIG", "1") != "1":
                continue
            xyz = T(W.cloud_uniform(b, n, 100 + int(np.log2(n)) + 16 * rank))
            m = n // 4
            fi = torch.empty((b, m), dtype=torch.int32, device=dev)
            nx = torch.empty((b, m, 3), dtype=torch.float32, device=dev)
            big = n >= 65536
            ms = timeit(torch, flush, lambda: lib.pn2_fps_gather(b, n, m, xyz.data_ptr(), None, fi.data_ptr(), nx.data_ptr(), None),
                        reps=(2 if big else 3), warm=1)
            add(f"cfg5[B={b},N={n}]", "fps+gather", ms, W.bytes_fps(b, n, m, True), dict(pairs_per_s=b * (m - 1) * n / (ms * 1e-3), us_per_iter=1e3 * ms / (m - 1),
                                                                                         points_per_s=b * n / (ms * 1e-3),
                                                                                         fp32_issue_frac_of_gpu=b * (m - 1) * n * 10 / (ms * 1e-3) / lane_rate))
            idx = torch.empty((b, m, 32), dtype=torch.int32, device=dev)
            cnt = torch.empty((b, m), dtype=torch.int32, device=dev)
            wsb = int(lib.pn2_query_ball_point_workspace_bytes(b, n))
            ws = torch.empty(max(wsb, 1), dtype=torch.uint8, device=dev)
            ms2 = timeit(torch, flush, lambda: lib.pn2_query_ball_point_ws(b, n, m, 0.1, 32, xyz.data_ptr(), nx.data_ptr(), idx.data_ptr(), cnt.data_ptr(),
                                                                           ws.data_ptr() if wsb else None, wsb, None), reps=3, warm=1)
            add(f"cfg5[B={b},N={n}]", "query_ball_point", ms2, W.bytes_ball_query(b, n, m, 32), dict(mean_cnt=float(cnt.float().mean()),
                                                                                                   points_per_s_fps_plus_query=b * n / ((ms + ms2) * 1e-3)))
            del xyz, fi, nx, idx, cnt
    return rows


def report(out_path):
    """Per-kernel tables for every BASELINE config (bench.py --report FILE)."""
    torch, lib, dev, flush = _setup()
    from bench import measured_peaks
    peak, kind = measured_peaks()
    rows = config_rows(torch, lib, dev, flush, peak, kind, full=True)
    json.dump(rows, open(out_path, "w"), indent=1)


def main(args):
    os.makedirs("gpurun_out", exist_ok=True)
    if args.fps_sweep:
        fps_sweep("gpurun_out/fps_sweep.json")
    if args.bq_sweep:
        bq_sweep("gpurun_out/bq_sweep.json")
    if args.report:
        report(args.report)


if __name__ == "__main__":
    print("use: python bench.py --report FILE | --fps-sweep | --bq-sweep", file=sys.stderr)
