#!/usr/bin/env python
"""Deterministic against atomic gradients on one GPU: the group_point / gather_point backward at the benchmark layers,
and a whole training step of cls_msg and sem_seg with torch.use_deterministic_algorithms on and off.  The two variants
are timed alternately, 5 rounds each, and the median is reported with the device's name and power limit.

    python tools/det_grad_bench.py [--json OUT]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys

os.environ.setdefault("CUBLAS_WORKSPACE_CONFIG", ":4096:8")
import torch  # noqa: E402

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from pointnet2_b200 import _lib, nets, workloads as W  # noqa: E402
from pointnet2_b200.tf_grouping import query_ball_point  # noqa: E402
from pointnet2_b200.tf_sampling import farthest_point_sample_and_gather  # noqa: E402

ROUNDS = 5


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name()


def event_ms(fn, flush, reps=10):
    st = torch.cuda.current_stream()
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


def alternate(fa, fb, flush):
    fa(), fb(), fa(), fb()  # warm-up
    ta, tb = [], []
    for _ in range(ROUNDS):
        ta.append(event_ms(fa, flush))
        tb.append(event_ms(fb, flush))
    return statistics.median(ta), statistics.median(tb)


def layer_rows(lib, dev, flush):
    rows = []
    c3, c4 = W.CFG3_MSG, W.CFG4_SEMSEG
    l1 = farthest_point_sample_and_gather(c3["layers"][0]["npoint"], torch.from_numpy(W.cloud_surface(c3["b"], c3["n"], 100)).to(dev))[1]
    cur = torch.from_numpy(W.cloud_duplicates(c4["b"], c4["n"], 100)).to(dev)
    layers = [(f"cfg3.L2 r={r}", l1, c3["layers"][1]["npoint"], r, s, 320) for r, s in zip(c3["layers"][1]["radii"], c3["layers"][1]["nsamples"])]
    for L in c4["sa"]:
        if L["c"]:
            layers.append((f"cfg4.SA{L['npoint']}", cur, L["npoint"], L["radius"], L["nsample"], L["c"]))
        cur = farthest_point_sample_and_gather(L["npoint"], cur)[1]
    for tag, xyz, m, r, s, c in layers:
        b, n, _ = xyz.shape
        ctr = farthest_point_sample_and_gather(m, xyz)[1]
        idx, _ = query_ball_point(r, s, xyz, ctr)
        wsb = int(lib.pn2_group_point_grad_det_workspace_bytes(b, n, m, s))
        ws = torch.empty(wsb, dtype=torch.uint8, device=dev)
        longest = int(max(torch.bincount(idx[i].reshape(-1).long(), minlength=n).max() for i in range(b)))
        for dt, code in ((torch.float32, 0), (torch.bfloat16, 1)):
            go = torch.randn((b, m, s, c), device=dev).to(dt)
            gp = torch.empty((b, n, c), dtype=dt, device=dev)
            acc = torch.empty((b, n, c), dtype=torch.float32, device=dev)

            def atomic():
                acc.zero_()
                lib.pn2_group_point_grad_typed(code, b, n, c, m, s, go.data_ptr(), idx.data_ptr(), (acc if code == 0 else gp).data_ptr(),
                                               acc.data_ptr(), None)

            def det():
                lib.pn2_group_point_grad_det_typed(code, b, n, c, m, s, go.data_ptr(), idx.data_ptr(), gp.data_ptr(), ws.data_ptr(), wsb, None)
            ta, td = alternate(atomic, det, flush)
            rows.append(dict(layer=f"{tag} S={s} C={c}", dtype=str(dt).split(".")[1], longest_list=longest, atomic_ms=ta, det_ms=td))
            print(json.dumps(rows[-1]), flush=True)
    c2 = W.CFG2_SSG_SA
    b, n, m = c2["b"], c2["n"], c2["npoint"]
    fi, _ = farthest_point_sample_and_gather(m, torch.from_numpy(W.cloud_uniform(b, n, 100)).to(dev))
    og, ig = torch.randn((b, m, 3), device=dev), torch.empty((b, n, 3), device=dev)
    wsb = int(lib.pn2_group_point_grad_det_workspace_bytes(b, n, m, 1))
    ws = torch.empty(wsb, dtype=torch.uint8, device=dev)

    def gatomic():
        ig.zero_()
        lib.pn2_gather_point_grad(b, n, m, og.data_ptr(), fi.data_ptr(), ig.data_ptr(), None)
    ta, td = alternate(gatomic, lambda: lib.pn2_gather_point_grad_det(b, n, m, og.data_ptr(), fi.data_ptr(), ig.data_ptr(), ws.data_ptr(), wsb, None), flush)
    rows.append(dict(layer="cfg2 gather_point_grad", dtype="float32", atomic_ms=ta, det_ms=td))
    print(json.dumps(rows[-1]), flush=True)
    return rows


def step_rows(dev):
    rows = []
    for name, b, n in (("cls_msg", 16, 1024), ("sem_seg", 8, 8192)):
        torch.manual_seed(0)
        net = (nets.PointNet2ClsMSG(40) if name == "cls_msg" else nets.PointNet2SemSeg(21)).to(dev)
        xyz = torch.from_numpy(W.cloud_surface(b, n, 500)).to(dev)

        def step(det):
            torch.use_deterministic_algorithms(det, warn_only=True)
            try:
                pred, _ = net(xyz)
                pred.float().square().mean().backward()
            finally:
                torch.use_deterministic_algorithms(False)
            net.zero_grad(set_to_none=True)

        for _ in range(3):
            step(False), step(True)
        toff, ton = [], []
        for _ in range(ROUNDS):
            for det, ts in ((False, toff), (True, ton)):
                a, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                step(det)
                e.record()
                e.synchronize()
                ts.append(a.elapsed_time(e))
        rows.append(dict(step=f"{name} B={b} N={n} fp32 forward+backward", det_off_ms=statistics.median(toff), det_on_ms=statistics.median(ton)))
        print(json.dumps(rows[-1]), flush=True)
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("det_grad_bench.py needs a CUDA device")
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    lib = _lib.load()
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    out = dict(gpu=gpu_info(), rounds=ROUNDS, layers=layer_rows(lib, dev, flush), steps=step_rows(dev))
    out["gpu_after"] = gpu_info()
    print(json.dumps(dict(gpu=out["gpu"], gpu_after=out["gpu_after"])))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
