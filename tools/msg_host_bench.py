#!/usr/bin/env python
"""Time the multi-scale host-buffer layer (pn2_sa_layer_msg_host / _ragged) against the two ways a caller with host
clouds had before it, on the reference's cls_msg level-1 layer (B 32, N 1024 -> 512, radii 0.1 / 0.2 / 0.4, nsample
16 / 32 / 128) and on N 4096 -> 1024 with the same scales:

  msg_host      SetAbstractionHost(radius=[...], nsample=[...]): one copy in, one sampling chain, every scale's ball
                query overlapping it, the copies back;
  three_single  three single-scale SetAbstractionHost sessions, one per scale, on the same stream: three copies in and
                three sampling chains;
  torch_msg     a torch copy of the pinned (b, n, 3) batch to the device, sa_layer.sample_group_msg(center=False), and
                non-blocking copies of its outputs into pinned host buffers (the same bytes msg_host copies back).

Each runs dense batches and batches whose lengths are drawn from U[N/2, N] (ragged=True for the host sessions; the
torch variant copies the batch padded to N and passes the lengths), with and without grouped_xyz.  The input is in
pinned host memory before timing starts, so host packing is not timed.  A round enqueues --iters batches of each
variant back to back on one stream, each between two CUDA events; the variants alternate their order by round.  The
JSON has the median and the 10th / 90th percentiles over every timed batch.  fps_only is the device-resident sampling
chain alone (farthest_point_sample_and_gather on the dense batch) for scale.  Before timing, every variant's outputs
are checked bit for bit against msg_host's.  The card's name and power limit are read in the same run.

    python tools/msg_host_bench.py --out DIR [--rounds 5] [--iters 30]
"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from pointnet2_b200 import workloads as W  # noqa: E402
from pointnet2_b200.host import SetAbstractionHost  # noqa: E402
from pointnet2_b200.sa_layer import sample_group_msg  # noqa: E402
from pointnet2_b200.tf_sampling import farthest_point_sample_and_gather  # noqa: E402

B = 32
RADII, NSAMPLES = [0.1, 0.2, 0.4], [16, 32, 128]
SIZES = [(1024, 512), (4096, 1024)]


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = "nvidia-smi unavailable"
    return {"torch_name": name, "nvidia_smi": q}


class MsgHost:
    def __init__(self, x, lengths, m, grouped, dev):
        b, n, _ = x.shape
        self.s = SetAbstractionHost(b, n, m, RADII, NSAMPLES, device=dev, want_grouped=grouped, ragged=lengths is not None)
        if lengths is None:
            self.s.h_xyz.numpy()[...] = x
        else:
            self.s.pack([np.ascontiguousarray(x[i, :l]) for i, l in enumerate(lengths)])

    def enqueue(self):
        self.s.launch()

    def outputs(self):
        o = self.s.outputs()
        return o[0], o[1], o[2], o[3] or []

    def h2d(self):
        return self.s.h2d_bytes


class ThreeSingle:
    def __init__(self, x, lengths, m, grouped, dev):
        b, n, _ = x.shape
        self.s = [SetAbstractionHost(b, n, m, r, k, device=dev, want_grouped=grouped, ragged=lengths is not None)
                  for r, k in zip(RADII, NSAMPLES)]
        for s in self.s:
            if lengths is None:
                s.h_xyz.numpy()[...] = x
            else:
                s.pack([np.ascontiguousarray(x[i, :l]) for i, l in enumerate(lengths)])

    def enqueue(self):
        for s in self.s:
            s.launch()

    def outputs(self):
        o = [s.outputs() for s in self.s]
        return o[0][0], [v[1] for v in o], [v[2] for v in o], [v[3] for v in o if v[3] is not None]

    def h2d(self):
        return sum(s.h2d_bytes for s in self.s)


class TorchMsg:
    def __init__(self, x, lengths, m, grouped, dev):
        b, n, _ = x.shape
        self.m, self.grouped, self.dev = m, grouped, dev
        self.h_x = torch.from_numpy(x).pin_memory()  # padded to n: the rows past a cloud's length are never read
        self.lengths = None if lengths is None else torch.tensor(lengths, dtype=torch.int32).pin_memory()
        pin = dict(pin_memory=True)
        self.h_new = torch.empty((b, m, 3), **pin)
        self.h_idx = [torch.empty((b, m, s), dtype=torch.int32, **pin) for s in NSAMPLES]
        self.h_cnt = [torch.empty((b, m), dtype=torch.int32, **pin) for _ in NSAMPLES]
        self.h_grp = [torch.empty((b, m, s, 3), **pin) for s in NSAMPLES] if grouped else []

    def enqueue(self):
        x = self.h_x.to(self.dev, non_blocking=True)
        lens = None if self.lengths is None else self.lengths.to(self.dev, non_blocking=True)
        _, nx, idx, cnt, grp = sample_group_msg(self.m, RADII, NSAMPLES, x, center=False, want_grouped=self.grouped,
                                                lengths=lens)
        self.h_new.copy_(nx, non_blocking=True)
        for h, d in zip(self.h_idx + self.h_cnt + self.h_grp, idx + cnt + (grp or [])):
            h.copy_(d, non_blocking=True)

    def outputs(self):
        return self.h_new.numpy(), [t.numpy() for t in self.h_idx], [t.numpy() for t in self.h_cnt], [t.numpy() for t in self.h_grp]

    def h2d(self):
        return self.h_x.numel() * 4 + (self.lengths.numel() * 4 if self.lengths is not None else 0)


VARIANTS = {"msg_host": MsgHost, "three_single": ThreeSingle, "torch_msg": TorchMsg}


def same(a, b):
    a, b = np.asarray(a), np.asarray(b)
    return a.shape == b.shape and np.array_equal(a.view(np.int32), b.view(np.int32))


def check_outputs(runs, dev):
    ref = runs["msg_host"]
    for r in runs.values():
        r.enqueue()
    torch.cuda.synchronize(dev)
    want = ref.outputs()
    for name, r in runs.items():
        got = r.outputs()
        ok = same(got[0], want[0]) and all(same(a, b) for k in (1, 2, 3) for a, b in zip(got[k], want[k]))
        ok = ok and all(len(got[k]) == len(want[k]) for k in (1, 2, 3))
        if not ok:
            raise SystemExit(f"{name}: outputs differ from msg_host")


def time_variants(runs, rounds, iters, dev):
    st = torch.cuda.current_stream(dev)
    for r in runs.values():  # warm-up: module loads, function attributes, allocator pools
        for _ in range(3):
            r.enqueue()
    torch.cuda.synchronize(dev)
    times = {name: [] for name in runs}
    names = list(runs)
    for rd in range(rounds):
        for name in (names if rd % 2 == 0 else names[::-1]):
            ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(iters)]
            for a, b in ev:
                a.record(st)
                runs[name].enqueue()
                b.record(st)
            torch.cuda.synchronize(dev)
            times[name] += [a.elapsed_time(b) for a, b in ev]
    return times


def fps_only(x, m, iters, dev):
    xd = torch.from_numpy(x).to(dev)
    for _ in range(3):
        farthest_point_sample_and_gather(m, xd)
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(iters)]
    for a, b in ev:
        a.record()
        farthest_point_sample_and_gather(m, xd)
        b.record()
    torch.cuda.synchronize(dev)
    return float(np.median([a.elapsed_time(b) for a, b in ev]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True, help="directory for msg_host_bench.json")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--iters", type=int, default=30)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("msg_host_bench needs a CUDA device")
    dev = torch.device("cuda:0")
    info = card()
    print(info, flush=True)
    rows = []
    for n, m in SIZES:
        x = W.cloud_uniform(B, n, 700 + n)
        rng = np.random.default_rng(800 + n)
        fps_ms = fps_only(x, m, 50, dev)
        for label, lengths in (("dense", None), ("U[N/2, N]", [int(v) for v in rng.integers(n // 2, n + 1, B)])):
            for grouped in (True, False):
                runs = {name: cls(x, lengths, m, grouped, dev) for name, cls in VARIANTS.items()}
                check_outputs(runs, dev)
                times = time_variants(runs, a.rounds, a.iters, dev)
                row = dict(b=B, n=n, npoint=m, radii=RADII, nsamples=NSAMPLES, lengths=label, grouped_xyz=grouped,
                           mean_length=float(np.mean(lengths)) if lengths else n, stride=max(lengths) if lengths else n,
                           rounds=a.rounds, iters=a.iters, fps_only_dense_ms=round(fps_ms, 4), outputs_identical=True)
                for name, ts in times.items():
                    row[name] = dict(median_ms=round(float(np.median(ts)), 4), p10_ms=round(float(np.percentile(ts, 10)), 4),
                                     p90_ms=round(float(np.percentile(ts, 90)), 4), h2d_bytes=runs[name].h2d())
                rows.append(row)
                print(json.dumps(row), flush=True)
                del runs
                torch.cuda.empty_cache()
    os.makedirs(a.out, exist_ok=True)
    with open(os.path.join(a.out, "msg_host_bench.json"), "w") as f:
        json.dump({"card": info, "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
