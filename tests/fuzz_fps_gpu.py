#!/usr/bin/env python
"""Randomised differential test of every farthest-point-sampling kernel against the C oracle (TEST TOOL, runs on a GPU
box).

    python tests/fuzz_fps_gpu.py [--seconds 120] [--seed 0] [--json out.json]

Four cases, each ``draw_<case>(rs, k)`` (parameters and inputs with numpy alone, no device; k = the case's count so
far in this seed) and ``run_<case>(p)``:

- ``fps_builtin``: the planner's own choice, dense or with per-cloud lengths (``draw_lengths``, clamped values
  included).  ``pn2_fps_plan`` must equal tests/fps_regimes.py's ``plan_fps`` given the device's SM count and
  ``pn2_fps_cluster_capacity``.
- ``fps_forced``: one instantiation of fps.cu, dense or ragged, forced through ``pn2_set_fps_config``.  The k-th forced
  case of a seed takes entry k of a per-seed permutation of ``COMBOS`` (every instantiation, dense and ragged), so a
  seed that runs ``len(COMBOS)`` of them runs every kernel.  The override is any of the encodings that name it (chain
  bits, cluster -1 / -2, the built-in chain); the cluster size is any the kernel takes; n is biased to the capacity,
  capacity - 1 and n << capacity (threads and whole CTAs without points).
- ``fps_scratch``: the global-scratch fallback with 33..80 clouds, so a CTA reuses its scratch row, with a short
  cloud after a long one on the same CTA in the ragged draws.
- ``fps_refused``: overrides the dispatcher must refuse; the call returns cudaErrorInvalidValue, launches nothing
  (``_lib.launch_count``) and writes nothing.

The clouds are fuzz_gpu's U/S/D/G/L kinds, fuzz_ball_gpu's adversarial ones (NaN / ±inf points, clouds NaN on a whole
axis, coordinates near 1e19, 2^-75 lattices, coincident clusters), a NaN point 0, coordinates of 1e19..1e20 (d² at
1e38 or inf), spacings of 1e-23..3e-22 (d² underflows to 0), −0.0 coordinates, clouds of one repeated point and
two-value lattices, with npoint in {1, 2, n - 1, n, n + 3}.  Every case must give the oracle's indices, new_xyz equal
to oracle_gather_point bit for bit (NaN payloads included), and gather_point(xyz, idx) == new_xyz; ragged cases run
with poisoned and with copied padding, which must agree.  tests/test_fuzz_fps_cpu.py replays the fixed slice with the
oracle's step trace and requires every instantiation, tie stage and data regime.  A failure is printed with the seed,
the iteration and its parameters; ``run(seed, iteration + 1)`` reproduces it on any machine.
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

ROOT = os.path.dirname(os.path.abspath(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import fps_regimes as R  # noqa: E402
import numerics as NUM  # noqa: E402
from fuzz_ball_gpu import draw_cloud  # noqa: E402  (the adversarial clouds)
from fuzz_contracts_gpu import both_paddings, draw_lengths, lengths_arg  # noqa: E402
from fuzz_gpu import cloud, log_n  # noqa: E402  (the U/S/D/G/L cloud distributions)
from oracle import oracle as O  # noqa: E402
from pointnet2_b200 import _lib  # noqa: E402

dev = torch.device("cuda:0")  # only dereferenced when a case runs

# the slice tests/test_fuzz_fps_gpu.py runs, and tests/test_fuzz_fps_cpu.py checks the coverage of
SLICE_SEEDS = (81, 82)
SCHEDULE = ["fps_forced", "fps_builtin", "fps_forced", "fps_scratch", "fps_forced", "fps_refused", "fps_forced",
            "fps_builtin"]
COMBOS = [(inst, ragged) for inst in R.INSTANCES if inst.family != "scratch" for ragged in (False, True)]
SLICE_ITERATIONS = 2 * len(COMBOS)  # four of every eight cases are forced: each seed runs every combination once

MAX_WORK = 6_000_000  # b * n * npoint: the oracle's distance evaluations (and the CPU replay's trace)
NAN_BITS = np.int32(0x7FC0BEEF)  # a quiet NaN with a payload the gather must copy
CUDA_ERROR_INVALID_VALUE = 1


def T(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


def N(t):
    return t.detach().cpu().numpy()


def _nan():
    return NAN_BITS.view(np.float32)


# ------------------------------------------------------------------------------------------------------ draws
TIE_HEAVY = ["same", "lattice2", "nan0", "big", "negzero"]  # kinds where many points tie at the maximum, step after step


def draw_xyz(rs, b, n, tie_heavy=False):
    """(kind, xyz (b, n, 3) float32); tie_heavy: one of TIE_HEAVY"""
    if tie_heavy:
        kind = str(rs.choice(TIE_HEAVY, p=[0.3, 0.4, 0.1, 0.1, 0.1]))
    else:
        kind = str(rs.choice(["base", "ball", "nan0", "big", "tiny", "negzero", "same", "lattice2"],
                             p=[0.18, 0.2, 0.08, 0.1, 0.08, 0.08, 0.08, 0.2]))
    if kind == "base":
        k, xyz = cloud(rs, b, n)
        return k, xyz
    if kind == "ball":
        k, xyz, _, _, _ = draw_cloud(rs, b, n)
        return "ball_" + k, xyz
    if kind == "nan0":  # the first pick is NaN: no running minimum moves, every point ties at 1e38
        xyz = rs.random_sample((b, n, 3)).astype(np.float32)
        if rs.rand() < 0.5:
            xyz[:, 0] = _nan()
        else:
            xyz[:, 0, rs.randint(3)] = _nan()
    elif kind == "big":  # d² from ~1e36 to inf: minima saturate at the 1e38 start, or stay below it
        xyz = (rs.uniform(-1, 1, (b, n, 3)) * np.exp(rs.uniform(np.log(1e19), np.log(1e20)))).astype(np.float32)
    elif kind == "tiny":  # lattice spacing 1e-23..3e-22: a square below 2^-150 rounds to 0
        step = np.float32(10.0 ** rs.uniform(-23, -21.5))
        xyz = (rs.randint(-3, 4, (b, n, 3)) * step).astype(np.float32)
    elif kind == "negzero":  # -0.0 and +0.0 coordinates on a small lattice
        xyz = (rs.randint(0, 3, (b, n, 3)) * np.float32(0.5)).astype(np.float32)
        xyz[(xyz == 0) & (rs.rand(b, n, 3) < 0.5)] = np.float32(-0.0)
    elif kind == "same":  # one point n times: after the first pick every minimum is 0
        p = rs.random_sample(3).astype(np.float32)
        if rs.rand() < 0.3:
            p[rs.randint(3)] = np.float32(-0.0)
        xyz = np.broadcast_to(p, (b, n, 3)).astype(np.float32)
    else:  # "lattice2": every coordinate one of two values: eight positions, ties across every boundary
        lo, hi = np.float32(rs.uniform(-1, 0)), np.float32(rs.uniform(0, 1))
        xyz = np.where(rs.rand(b, n, 3) < 0.5, lo, hi).astype(np.float32)
    return kind, np.ascontiguousarray(xyz, np.float32)


def draw_npoint(rs, b, n):
    m = int(rs.choice([1, 2, n - 1, n, n + 3, log_n(rs, 1, 600), log_n(rs, 1, 600)]))
    m = min(max(m, 1), 700)
    return max(1, min(m, max(8, MAX_WORK // (b * n))))


def _lens(rs, b, n, npoint, ragged):
    return draw_lengths(rs, b, n, npoint) if ragged else None


def draw_fps_builtin(rs, k):
    u = rs.rand()
    if u < 0.35:  # single CTA, every table edge
        b = int(rs.choice([1, 2, 5, 16, 33, 140]))
        n = int(rs.choice([1, 2, 127, 128, 129, 255, 256, 257, 511, 512, 513, 1023, 1024, 1025, 2047, 2048, 2049,
                           4095, 4096, 4097, 8191, 8192, log_n(rs, 1, 8192)]))
    elif u < 0.8:  # clusters: the cluster search, and at the largest sizes the cost model
        b = int(rs.choice([1, 2, 3, 4, 8, 9, 17]))
        n = int(rs.choice([8193, 16384, 16385, 32769, 65536, 65537, 131073, 262144, 262145, 425984,
                           log_n(rs, 8193, 425984)]))
        b = min(b, max(1, 1_000_000 // n))
    else:  # beyond every cluster: the global-scratch fallback
        b = int(rs.choice([1, 2]))
        n = int(rs.choice([425985, log_n(rs, 425985, 520000)]))
    npoint = draw_npoint(rs, b, n)
    kind, xyz = draw_xyz(rs, b, n)
    lens = _lens(rs, b, n, npoint, rs.rand() < 0.4)
    return dict(case="fps_builtin", b=b, n=n, npoint=npoint, kind=kind, lens=lens, xyz=xyz)


def encodings(inst, C):
    """every (threads, ppt, cluster) override that names ``inst`` at cluster size C"""
    pk = {(P, T): k for P, T, k in R.CTA_KERNELS}
    pkc = {(P, T): k for P, T, _, k in R.CLUSTER_KERNELS}
    P, Tn = inst.P, inst.T
    if inst.family == "cta":
        if not pk[(P, Tn)]:  # no packed chain: every encoding runs the plain one
            return [(Tn, P, -1), (Tn, P, -2), (Tn + 1, P, 1), (Tn + 2, P, 1), (Tn, P, 1)]
        return [(Tn, P, -2), (Tn + 1, P, 1), (Tn, P, 1)] if inst.V else [(Tn, P, -1), (Tn + 2, P, 1)]
    packed = pkc.get((P, Tn), 1) if inst.family == "cluster" else 1
    if not packed:
        return [(Tn, P, C), (Tn + 1, P, C), (Tn + 2, P, C)]
    return [(Tn + 1, P, C), (Tn, P, C)] if inst.V else [(Tn + 2, P, C)]


def draw_cluster_size(rs, inst):
    if inst.family == "big":  # any size, powers of two or not
        return int(rs.choice([2, 4, 8, 16])) if rs.rand() < 0.4 else int(rs.randint(2, 17))
    if inst.family == "cluster":  # powers of two with C * T a multiple of 512
        return int(rs.choice([c for c in (2, 4, 8, 16) if (c * inst.T) % R.SLOTS == 0]))
    return 1


def draw_fps_forced(rs, k, seed):
    inst, ragged = COMBOS[forced_order(seed)[k % len(COMBOS)]]
    C = draw_cluster_size(rs, inst)
    cap = R.capacity_of(inst, C)
    u = rs.rand()
    if u < 0.3:
        n = cap
    elif u < 0.5:
        n = max(1, cap - 1)
    elif u < 0.75:  # threads and whole CTAs without points
        n = log_n(rs, 1, max(1, cap // 8))
    else:
        n = log_n(rs, max(1, cap // 8), cap)
    b = 1 if n > 100_000 else int(rs.randint(1, 4))
    npoint = draw_npoint(rs, b, n)
    encs = encodings(inst, C)
    override = tuple(int(v) for v in encs[rs.randint(len(encs))])
    got, why = R.dispatch(R.decode_override(*override), n)
    assert got == inst and why is None, (inst, override, got, why)  # the draw table names what it means to run
    kind, xyz = draw_xyz(rs, b, n, tie_heavy=rs.rand() < 0.4)
    return dict(case="fps_forced", b=b, n=n, npoint=npoint, kind=kind, inst=inst.name, C=C, override=override,
                lens=_lens(rs, b, n, npoint, ragged), xyz=xyz)


def draw_fps_scratch(rs, k):
    b = int(rs.randint(33, 81))
    ragged = rs.rand() < 0.6
    n = log_n(rs, 2 if ragged else 1, 6000)
    npoint = draw_npoint(rs, b, n)
    kind, xyz = draw_xyz(rs, b, n)
    lens = _lens(rs, b, n, npoint, ragged)
    if lens:  # a short cloud after a long one on the same CTA (clouds i and i + 32)
        i = int(rs.randint(0, b - 32))
        short = int(rs.randint(1, max(1, n // 4) + 1))
        for at, v in ((i, n), (i + 32, min(short, n - 1))):
            lens["raw"][at] = lens["lengths"][at] = v
    override = (int(rs.choice([1024, 512, 128])), int(rs.choice([0, 1, 8])), 0)
    return dict(case="fps_scratch", b=b, n=n, npoint=npoint, kind=kind, override=override, lens=lens, xyz=xyz)


REFUSALS = ["capacity", "cluster_over_16", "cluster_not_pow2", "ct_not_512", "no_instance", "no_scratch"]


def draw_fps_refused(rs, k):
    why = REFUSALS[k % len(REFUSALS)]
    n = log_n(rs, 1, 200)  # within every capacity below: the refusal is the one named
    b = int(rs.randint(1, 4))
    if why == "capacity":  # one point more than the kernel holds
        inst = [i for i in R.INSTANCES if i.family != "scratch"][rs.randint(len(R.INSTANCES) - 1)]
        C = draw_cluster_size(rs, inst)
        encs = encodings(inst, C)
        override = encs[rs.randint(len(encs))]
        n = R.capacity_of(inst, C) + int(rs.choice([1, 2, 97]))
        b = 1
    elif why == "cluster_over_16":
        override = [(512 + int(rs.randint(0, 3)), int(rs.choice([44, 48, 52])), int(rs.randint(17, 33))),
                    (128, 8, 32), (256, 32, 32)][rs.randint(3)]
    elif why == "cluster_not_pow2":
        override = (int(rs.choice([256, 512, 1024])), int(rs.choice([2, 8, 16])), int(rs.choice([3, 5, 6, 7, 12, 15])))
    elif why == "ct_not_512":  # two CTAs of 128 threads: the reference slots would split across the pair
        override = (128 + int(rs.randint(0, 3)), int(rs.choice([4, 8, 16, 32])), 2)
    elif why == "no_instance":
        override = [(512, 32, 1), (1024, 16, 1), (128, 3, 1), (64, 4, 1), (2048, 1, -2), (128, 2, 4), (1024, 16, 2),
                    (512, 40, 2), (256, 44, 4), (1024, 48, 2), (513, 36, 3)][rs.randint(11)]
    else:  # the scratch plan without its scratch buffer
        override = (1024, 1, 0)
    override = tuple(int(v) for v in override)
    npoint = log_n(rs, 1, 64)
    got, reason = R.dispatch(R.decode_override(*override), n, have_temp=why != "no_scratch")
    assert got is None and reason == why, (override, n, got, reason, why)
    xyz = rs.random_sample((b, n, 3)).astype(np.float32)
    lens = _lens(rs, b, n, npoint, rs.rand() < 0.3)
    return dict(case="fps_refused", b=b, n=n, npoint=npoint, why=why, override=override, lens=lens, xyz=xyz)


def forced_order(seed):
    """the per-seed permutation of COMBOS the forced cases walk through"""
    return np.random.RandomState(seed + 7919).permutation(len(COMBOS))


# -------------------------------------------------------------------------------------------------------- runs
def _fps(npoint, xp, lens):
    from pointnet2_b200.tf_sampling import farthest_point_sample_and_gather
    return farthest_point_sample_and_gather(npoint, T(xp), lengths=lengths_arg(lens) if lens else None)


def check(p, run):
    """``run(xyz)`` -> (idx, new_xyz) against the oracle on every (truncated) cloud, both paddings when ragged"""
    from pointnet2_b200.tf_sampling import gather_point
    x, lens, m = p["xyz"], p["lens"], p["npoint"]
    ls = lens["lengths"] if lens else [p["n"]] * p["b"]
    if lens:
        (idx, nx), ok = both_paddings(run, [x], ls)
        xp = NUM.pad_rows(x, ls, "poison")
    else:
        (idx, nx), ok, xp = run(x), True, x
    ok = ok and np.array_equal(N(gather_point(T(xp), idx)).view(np.int32), N(nx).view(np.int32))
    idx, nx = N(idx), N(nx)
    for i, ln in enumerate(ls):
        c = x[i:i + 1, :ln]
        o = O.oracle_fps(m, c)
        ok = ok and np.array_equal(idx[i:i + 1], o)
        ok = ok and np.array_equal(nx[i:i + 1].view(np.int32), O.oracle_gather_point(c, o).view(np.int32))
    return bool(ok)


def _forced(p, body):
    lib = _lib.load()
    try:
        lib.pn2_set_fps_config(*p["override"])
        return body(lib)
    finally:
        lib.pn2_set_fps_config(0, 0, 0)


def device_plan(lib, b, n):
    t, pp, c = ctypes.c_int(), ctypes.c_int(), ctypes.c_int()
    assert lib.pn2_fps_plan(b, n, ctypes.byref(t), ctypes.byref(pp), ctypes.byref(c)) == 0
    return t.value, pp.value, c.value


def live_capacity(lib):
    return lambda t, pp, c, packed: int(lib.pn2_fps_cluster_capacity(t + (0 if packed else 2), pp, c))


def run_fps_builtin(p):
    lib = _lib.load()
    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    want = R.plan_fps(p["b"], p["n"], sms=sms, capacity=live_capacity(lib))
    p["plan"] = device_plan(lib, p["b"], p["n"])
    ok = p["plan"] == (want.threads, want.ppt, want.cluster)
    return bool(ok and check(p, lambda a: _fps(p["npoint"], a, p["lens"])))


def run_fps_forced(p):
    def body(lib):
        if p["C"] >= 2 and lib.pn2_fps_cluster_capacity(*p["override"]) <= 0:
            raise AssertionError("the device cannot hold this cluster: the draw table is wrong")
        return check(p, lambda a: _fps(p["npoint"], a, p["lens"]))
    return _forced(p, body)


def run_fps_scratch(p):
    return _forced(p, lambda lib: check(p, lambda a: _fps(p["npoint"], a, p["lens"])))


def run_fps_refused(p):
    from pointnet2_b200._tensor import stream_ptr

    def body(lib):
        b, n, m = p["b"], p["n"], p["npoint"]
        x = T(p["xyz"])
        idx = torch.full((b, m), -7, dtype=torch.int32, device=dev)
        nx = torch.full((b, m, 3), 3.5, dtype=torch.float32, device=dev)
        tb = int(lib.pn2_fps_scratch_bytes(b, n))
        temp = torch.empty(max(tb, 4), dtype=torch.uint8, device=dev) if tb and p["why"] != "no_scratch" else None
        tptr = temp.data_ptr() if temp is not None else None
        torch.cuda.synchronize(dev)
        before = _lib.launch_count()
        if p["lens"]:
            lens = torch.tensor(p["lens"]["lengths"], dtype=torch.int32, device=dev)
            rc = lib.pn2_fps_gather_ragged(b, n, m, x.data_ptr(), lens.data_ptr(), tptr, idx.data_ptr(), nx.data_ptr(),
                                           stream_ptr(dev))
        else:
            rc = lib.pn2_fps_gather(b, n, m, x.data_ptr(), tptr, idx.data_ptr(), nx.data_ptr(), stream_ptr(dev))
        launched = _lib.launch_count() - before
        torch.cuda.synchronize(dev)
        untouched = bool((idx == -7).all()) and bool((nx == 3.5).all())
        return rc == CUDA_ERROR_INVALID_VALUE and launched == 0 and untouched
    return _forced(p, body)


CASES = ["fps_builtin", "fps_forced", "fps_scratch", "fps_refused"]
RUN = {name: globals()["run_" + name] for name in CASES}


class Drawer:
    """The cases of one seed in SCHEDULE order; the k-th case of each kind gets k."""

    def __init__(self, seed):
        self.seed, self.rs, self.seen = seed, np.random.RandomState(seed), {}

    def next(self, it):
        name = SCHEDULE[it % len(SCHEDULE)]
        k = self.seen.get(name, 0)
        self.seen[name] = k + 1
        if name == "fps_forced":
            return name, draw_fps_forced(self.rs, k, self.seed)
        return name, globals()["draw_" + name](self.rs, k)


def draws(seed: int, iterations: int):
    """The parameters ``run(seed, iterations)`` uses, without a device (the run_* functions draw nothing)."""
    d = Drawer(seed)
    return [d.next(it)[1] for it in range(iterations)]


def public(p):
    """the parameters of a case without its input arrays (they follow from the seed and the iteration)"""
    return {k: v for k, v in p.items() if not isinstance(v, np.ndarray)}


def _one(d, it, counts, fails, catch):
    name, p = d.next(it)
    try:
        ok = RUN[name](p)
    except Exception as e:  # noqa: BLE001 — report the exception as a failure of that case
        if not catch:
            raise
        ok = False
        p = dict(p, error=f"{type(e).__name__}: {e}")
    counts[name] = counts.get(name, 0) + 1
    if not ok:
        fails.append(dict(public(p), seed=d.seed, iteration=it))
    return name, ok


def run(seed: int, iterations: int):
    """``iterations`` random cases in SCHEDULE order; returns (counts, failures)."""
    d = Drawer(seed)
    counts, fails = {}, []
    for it in range(iterations):
        _one(d, it, counts, fails, catch=False)
    return counts, fails


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=float, default=120)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--json", type=str, default=None)
    args = ap.parse_args()
    d = Drawer(args.seed)
    counts, fails, secs = {}, [], {}
    t0 = time.time()
    it = 0
    while time.time() - t0 < args.seconds:
        t1 = time.time()
        name, ok = _one(d, it, counts, fails, catch=True)
        secs[name] = secs.get(name, 0.0) + time.time() - t1
        if not ok:
            print("FAIL", json.dumps(fails[-1], default=str), flush=True)
        it += 1
    summary = dict(seed=args.seed, seconds=round(time.time() - t0, 1), cases=counts,
                   case_seconds={k: round(v, 1) for k, v in secs.items()}, failures=fails)
    print(json.dumps(summary, default=str))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(summary, f, indent=1, default=str)
    sys.exit(1 if fails else 0)


if __name__ == "__main__":
    main()
