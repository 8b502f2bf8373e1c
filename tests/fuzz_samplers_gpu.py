#!/usr/bin/env python
"""Randomised differential test of the seeded samplers (csrc/voxel.cu, shapes.cu, crops.cu, vscan.cu) against their
numpy oracles (voxel_oracle, shape_oracle, crop_oracle, scan_oracle) and tests/select_regimes.py (TEST TOOL, runs on
a GPU box).

    python tests/fuzz_samplers_gpu.py [--seconds 120] [--seed 0] [--json out.json]

Each case is ``draw_<case>(rs)`` (parameters and inputs with numpy alone, no device) and ``run_<case>(p)``.  Three
draws in four call the C entry point with caller-owned outputs: every output is filled with the byte 0xA5 and has a
guard of GUARD bytes after its end, so a slot that is never written, or one written past the end, fails.  The fourth
goes through the Python wrapper.  Integer outputs and copied coordinates must match the oracle bit for bit; computed
coordinates keep the bound of the op's own GPU test (one float32 ulp of the float64 value plus 1e-12 for the rotated
crops and the shape batches).  The seed is a negative int, one >= 2^63, or a (1,) device tensor (with a different
launch argument, which the kernels must ignore).

- ``voxel``: voxels and pillars, dense and with lengths (0, 1, < N, N, out of range), points on and around the cell
  edges, quotients in (-1, 0), NaN and out-of-grid points, clustered and duplicate-heavy clouds, one-cell clouds and
  clouds built from exact per-cell counts (0, 1, 31, 32, 33, 64, 65, 127, 128 and past 128, on both sides of S).
- ``voxel_planted``: a 2.6M-row cloud with three planted cells whose select boundary splits two rows with equal
  rng_row_key high halves (select_regimes.PLANTED): the select finishes at pass 2, 3 or 4, and 5.
- ``shapes``: subset first or random, votes, with and without normals and parts, dropout on and off.
- ``shapes_planted``: a random-subset batch whose entry select splits a planted pair (passes 4 and 5).
- ``crops``: rooms with npoints below, equal to, one under and far under the members; unlabelled scenes (every
  attempt invalid: attempt 9) and duplicate scenes.
- ``vscan``: scenes with fewer than 100 near points, with visible < min_points and visible > npoints, every scan mode.
- ``refused``: a refused call returns cudaErrorInvalidValue, launches nothing and leaves the outputs poisoned.

Every case also has out-of-range and empty entries.  tests/test_fuzz_samplers_cpu.py replays the fixed slice through
select_regimes and requires every regime.  A failure is printed with the seed, the iteration and its parameters;
``run(seed, iteration + 1)`` reproduces it on any machine.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.abspath(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import crop_oracle as CO  # noqa: E402
import scan_oracle as SO  # noqa: E402
import select_regimes as R  # noqa: E402
import shape_oracle as SH  # noqa: E402
import voxel_oracle as VO  # noqa: E402
from pointnet2_b200 import _lib  # noqa: E402
from pointnet2_b200 import workloads as W  # noqa: E402

dev = torch.device("cuda:0")  # only dereferenced when a case runs

# the slice tests/test_fuzz_samplers_gpu.py runs, and tests/test_fuzz_samplers_cpu.py checks the coverage of
SLICE_SEEDS = (81, 82)
SCHEDULE = ["voxel", "shapes", "crops", "voxel", "vscan", "voxel_planted", "shapes", "voxel", "crops", "refused",
            "shapes_planted", "voxel", "crops", "vscan", "voxel", "shapes", "shapes", "voxel"]
SLICE_ITERATIONS = 2 * len(SCHEDULE)

POISON = 0xA5      # every output byte before a call
GUARD = 64         # poisoned bytes after each output
CUDA_ERROR_INVALID_VALUE = 1
PLANT_N = (1 << 21) + (1 << 19)  # rows of a planted voxel cloud: past every planted row
MAX_SLOTS = 1 << 21              # b * cells * nsample of a voxel draw: grouped stays within 48 MB


def log_int(rs, lo, hi):
    return int(np.clip(np.exp(rs.uniform(np.log(lo), np.log(hi + 1))), lo, hi))


def draw_seed(rs):
    """(seed as the wrappers take it, kind): negative, >= 2^63, small, or read from a device tensor"""
    kind = str(rs.choice(["negative", "high", "small", "device"]))
    v = {"negative": -int(rs.randint(1, 1 << 62)), "high": (1 << 63) + int(rs.randint(0, 1 << 62)),
         "small": int(rs.randint(0, 1000)), "device": int(rs.randint(-(1 << 62), 1 << 62))}[kind]
    return v, kind


def signed(seed):
    return seed - (1 << 64) if seed >= (1 << 63) else seed


def draw_api(rs):
    return "wrapper" if rs.rand() < 0.25 else "c"


# ------------------------------------------------------------------------------------------------------- voxel
VOXEL_KINDS = ["uniform", "edges", "clustered", "duplicates", "one_cell", "counts"]
COUNT_LADDER = [0, 1, 31, 32, 33, 64, 65, 127, 128, 129, 200, 700]
NSAMPLES = [1, 2, 31, 32, 33, 64, 65, 100, 127, 128, 129, 130, 200, 257, 1000, 16384]


def _cell_points(rs, cells, dim, dims, radius):
    """one float32 point strictly inside each given cell"""
    voxel = 2 * radius / dim
    coord = np.stack([cells // dim, cells % dim], 1) if dims == 2 else \
        np.stack([cells // (dim * dim), (cells // dim) % dim, cells % dim], 1)
    p = (coord + rs.uniform(0.25, 0.75, coord.shape)) * voxel - radius
    if dims == 2:
        p = np.concatenate([p, rs.uniform(-3, 3, (len(cells), 1))], 1)
    return p.astype(np.float32)


ONE_CELL_EDGES = ["m1", "c_eq_m_plus_1", "m_max"]


def draw_voxel(rs, k=0):
    """draw k of a seed: k % 3 == 0 a cloud of exact per-cell counts, k % 3 == 2 a one-cell cloud at an edge of m
    (1, c - 1 or kSelectMaxRows), else in turn a uniform, duplicate-heavy, edge or clustered cloud"""
    dims = int(rs.choice([2, 3]))
    dim = int(rs.choice([1, 2, 3, 5, 8, 12] if dims == 3 else [1, 3, 7, 12, 31]))
    radius = float(rs.choice([1.0, 0.5, 2.5, 0.3]))
    cells = dim ** dims
    kind = "counts" if k % 3 == 0 else ["uniform", "duplicates", "edges", "clustered"][(k // 3) % 4]
    edge = ONE_CELL_EDGES[(k // 3) % 3] if k % 3 == 2 else None
    if edge:
        kind, dims, dim = "one_cell", 3, int(rs.choice([1, 2]))
        cells = dim ** dims
    nsample = int(rs.choice(NSAMPLES))
    b = int(rs.randint(1, 4))
    voxel = 2 * radius / dim
    if kind == "counts":  # exact per-cell counts: every warp key width and both CTA key types
        want = rs.choice(COUNT_LADDER, (b, cells))
        if rs.rand() < 0.3 and 64 <= cells <= 1000:  # more listed cells than 2 x SMs CTAs
            b = max(b, -(-(2 * R.SMS + 10) // cells))
            want = rs.randint(129, 140, (b, cells))
        n = int(want.sum(1).max()) + int(rs.randint(0, 50))
        xyz = np.full((b, n, 3), np.nan, np.float32)
        for i in range(b):
            cl = np.repeat(np.arange(cells), want[i])
            xyz[i, :len(cl)] = _cell_points(rs, cl, dim, dims, radius)
            xyz[i] = xyz[i, rs.permutation(n)]
        # S above the ladder's CTA cells (row keys, no select), or inside it (seeded warp and CTA cells)
        nsample = 300 if k % 6 == 0 else int(rs.choice([31, 33, 64, 100, 128, 129, 150]))
    else:
        n = log_int(rs, 1, 20000) if kind != "one_cell" else int(rs.choice([129, 500, 16385, 20000, 40000]))
        if kind == "uniform":
            xyz = rs.uniform(-1.05 * radius, 1.05 * radius, (b, n, 3))
        elif kind == "edges":  # on the cell edges, one float32 ulp to either side, and quotients in (-1, 0)
            k = rs.randint(0, dim + 1, (b, n, 3))
            xyz = (k * np.float32(voxel) - np.float32(radius)).astype(np.float32)
            xyz = np.where(rs.rand(b, n, 3) < 0.3, np.nextafter(xyz, np.float32(np.inf)), xyz)
            xyz = np.where(rs.rand(b, n, 3) < 0.3, np.nextafter(xyz, np.float32(-np.inf)), xyz)
            neg = rs.rand(b, n, 3) < 0.1
            xyz = np.where(neg, -radius - rs.uniform(0, 1.2, (b, n, 3)) * voxel, xyz)
        elif kind == "clustered":
            c = rs.uniform(-0.9, 0.9, (b, 3, 3)) * radius
            xyz = c[np.arange(b)[:, None], rs.randint(0, 3, (b, n))] + rs.normal(0, 0.02 * radius, (b, n, 3))
        elif kind == "duplicates":
            base = rs.uniform(-radius, radius, (b, 5, 3))
            xyz = base[np.arange(b)[:, None], rs.randint(0, 5, (b, n))]
        else:  # the whole cloud in one cell
            cell = rs.randint(0, cells, b)
            xyz = np.stack([_cell_points(rs, np.full(n, c), dim, dims, radius) for c in cell])
            if edge:
                nsample = {"m1": 1, "c_eq_m_plus_1": n - 1, "m_max": R.MAX_ROWS}[edge]
                n = {"m1": int(rs.randint(2, 129)), "c_eq_m_plus_1": n, "m_max": max(n, 20000)}[edge]
                xyz = np.stack([_cell_points(rs, np.full(n, c), dim, dims, radius) for c in cell])
            elif rs.rand() < 0.5:
                nsample = int(rs.choice([128, 129, n - 1 if n > 1 else 1, 16384]))
        xyz = np.asarray(xyz, np.float32)
        if not edge:  # NaN and out-of-grid rows
            u = rs.rand(b, n)
            xyz[u < 0.02] = np.nan
            xyz[(u >= 0.02) & (u < 0.04)] = np.float32(radius * 3)
    nsample = int(min(max(nsample, 1), R.MAX_ROWS, max(1, MAX_SLOTS // (b * cells))))
    lkind = "none" if edge else str(rs.choice(["none", "mixed"]))
    lengths = None
    if lkind == "mixed":
        lengths = np.array([int(rs.choice([0, 1, max(n // 2, 1), n, -3, n + 5])) for _ in range(b)], np.int32)
    seed, skind = draw_seed(rs)
    return dict(case="voxel", kind=kind, dims=dims, dim=dim, radius=radius, nsample=nsample, b=b, n=n, xyz=xyz,
                lengths=lengths, lengths_kind=lkind, seed=seed, seed_kind=skind, api=draw_api(rs))


def plant_cell(rs, seed, e, j1, j2, s, pool, extra):
    """rows of cell entry e: the pair (j1 < j2, equal key high halves), s - 1 rows of ``pool`` with smaller keys and
    ``extra`` with larger ones, so that a select of s rows takes j1 last and leaves j2"""
    k = R.row_keys(seed, VO.STREAM_CELL, e, pool)
    k1 = int(R.row_keys(seed, VO.STREAM_CELL, e, [j1])[0])
    small, large = pool[k < np.uint64(k1)], pool[k > np.uint64(k1)]
    assert len(small) >= s - 1 and len(large) >= extra, (len(small), len(large))
    return np.concatenate([[j1, j2], rs.choice(small, s - 1, replace=False), rs.choice(large, extra, replace=False)])


def pass2_pair(seed, e, lo, count):
    """rows whose full orders agree in their top 22 bits (a select boundary between them finishes at pass 2)"""
    j = np.arange(lo, lo + count, dtype=np.int64)
    k = R.row_keys(seed, VO.STREAM_CELL, e, j)
    top = k >> np.uint64(42)
    o = np.argsort(top, kind="stable")
    d = np.nonzero(top[o][1:] == top[o][:-1])[0]
    a, b2 = sorted((int(j[o[d[0]]]), int(j[o[d[0] + 1]])))
    return a, b2


def draw_voxel_planted(rs, k=0):
    """cells 0, 5 and 11 of a 3^3 grid, cloud 0: passes 3 or 4 (alternating), 2 and 5"""
    which = 3 if k % 2 == 0 else 4
    seed, e0, a0, b0 = R.PLANTED[("voxel", which)]
    _, e11, a11, b11 = R.PLANTED[("voxel", 5)]
    s = int(rs.randint(30, 300))
    pools = [np.arange(lo, lo + 400000) for lo in (0, 400000, 800000)]
    p2 = pass2_pair(seed, 5, 1300000, 1 << 16)
    rows0 = plant_cell(rs, seed, e0, a0, b0, s, pools[0], max(0, 129 - s) + int(rs.randint(0, 50)))
    rows5 = plant_cell(rs, seed, 5, p2[0], p2[1], s, pools[1], max(0, 129 - s) + int(rs.randint(0, 50)))
    rows11 = plant_cell(rs, seed, e11, a11, b11, s, pools[2], max(0, 129 - s) + int(rs.randint(0, 50)))
    xyz = np.full((1, PLANT_N, 3), np.nan, np.float32)
    for cell, rows in ((0, rows0), (5, rows5), (11, rows11)):
        xyz[0, rows] = _cell_points(rs, np.full(len(rows), cell), 3, 3, 1.0)
    dev_seed = bool(rs.rand() < 0.5)
    return dict(case="voxel_planted", kind="planted", dims=3, dim=3, radius=1.0, nsample=s, b=1, n=PLANT_N, xyz=xyz,
                lengths=None, lengths_kind="none", seed=seed, seed_kind="device" if dev_seed else "small",
                api="c", planted={0: which, 5: 2, 11: 5})


# ------------------------------------------------------------------------------------------------------ shapes
def draw_shape_set(rs, sizes, normals, parts):
    pts = [rs.uniform(-1, 1, (n, 3)).astype(np.float32) for n in sizes]
    if rs.rand() < 0.3:  # a duplicate-heavy shape
        pts[0] = pts[0][rs.randint(0, max(1, len(pts[0]) // 7), len(pts[0]))]
    return dict(xyz=pts, label=[int(rs.randint(0, 40)) for _ in sizes],
                normals=[rs.standard_normal((n, 3)).astype(np.float32) for n in sizes] if normals else None,
                part=[rs.randint(0, 50, n).astype(np.int32) for n in sizes] if parts else None)


def draw_shapes(rs, k=0, planted=None):
    votes = int(rs.choice([0, 0, 0, 1, 3])) if planted is None and k % 4 in (0, 3) else 0
    ns = int(rs.randint(1, 5))
    sizes = [log_int(rs, 1, R.MAX_ROWS) for _ in range(ns)]
    if rs.rand() < 0.3:
        sizes[0] = R.MAX_ROWS
    subset = "first" if votes else str(rs.choice(["first", "random"]))
    with_normals, parts = bool(rs.rand() < 0.5), bool(rs.rand() < 0.5)
    b = int(rs.randint(1, 10))
    ref = sizes[int(rs.randint(ns))]
    npoints = int(rs.choice([1, max(ref - 1, 1), ref, min(ref + 1, R.MAX_ROWS), R.MAX_ROWS,
                             log_int(rs, 1, R.MAX_ROWS)]))
    if k % 4 == 1:  # one row of many
        npoints, sizes[0], subset = 1, max(sizes[0], 2), "random"
    elif k % 4 == 2:  # a random subset of shape 0 one row short of it
        sizes[0] = max(sizes[0], 2)
        subset, npoints = "random", sizes[0] - 1
    elif k % 4 == 3:  # every pool shorter than npoints
        sizes = [min(v, R.MAX_ROWS - 1) for v in sizes]
        npoints = max(sizes) + 1
    aug = dict(rotate=False, perturb=False, scale=None, shift=0.0, jitter=None, max_dropout=0.0)
    if not votes:
        aug = dict(rotate=bool(rs.rand() < 0.5), perturb=bool(rs.rand() < 0.5),
                   scale=(0.8, 1.25) if rs.rand() < 0.5 else None, shift=float(rs.choice([0.0, 0.1])),
                   jitter=(0.01, 0.05) if rs.rand() < 0.5 else None,
                   max_dropout=float(rs.choice([0.0, 0.875, 1.0, rs.uniform(0, 1)])))
    idx = rs.randint(0, ns, b)
    idx[0] = 0
    if rs.rand() < 0.3:
        idx[int(rs.randint(b))] = int(rs.choice([-1, ns, 1 << 40]))
    seed, skind = draw_seed(rs)
    p = dict(case="shapes", votes=votes, subset=subset, with_normals=with_normals, parts=parts, sizes=sizes,
             npoints=npoints, b=b, shape_idx=idx, seed=seed, seed_kind=skind, api=draw_api(rs), **aug)
    if planted is not None:  # entry e of a random-subset batch splits the planted pair
        which = planted
        seed, e, j1, j2 = R.PLANTED[("shapes", which)]
        ps = j2 + 1 + int(rs.randint(0, R.MAX_ROWS - j2))
        keys = R.row_keys(seed, SH.STREAM_KEY, e, np.arange(ps))
        rank = int((keys < keys[j1]).sum())
        sizes = [ps] + sizes[1:]
        idx = rs.randint(0, len(sizes), e + 1 + int(rs.randint(0, 3)))
        idx[e] = 0
        p.update(case="shapes_planted", subset="random", sizes=sizes, npoints=rank + 1, b=len(idx), shape_idx=idx,
                 seed=seed, seed_kind="small", planted={e: which}, max_dropout=0.0)
    p["set"] = draw_shape_set(rs, p["sizes"], with_normals, parts)
    return p


def draw_shapes_planted(rs, k=0):
    return draw_shapes(rs, planted=4 if k % 2 == 0 else 5)


# ------------------------------------------------------------------------------------------------ crops, vscan
def draw_scenes(rs, kinds):
    out = []
    for kind in kinds:
        if kind in ("room", "big_room"):
            lo, hi = (3000, 40000) if kind == "room" else (60000, 150000)
            out.append(W.scene_room(log_int(rs, lo, hi), int(rs.randint(1 << 20))))
        elif kind == "unlabelled":
            p, lab = W.scene_room(log_int(rs, 3000, 20000), int(rs.randint(1 << 20)))
            out.append((p, np.zeros_like(lab)))
        elif kind == "duplicates":
            d = (rs.random_sample((int(rs.randint(200, 1500)), 3)) * [2.5, 2.5, 1.0]).astype(np.float32)
            out.append((np.repeat(d, int(rs.randint(2, 20)), axis=0), None))
            out[-1] = (out[-1][0], rs.randint(0, 21, len(out[-1][0])))
        elif kind == "away":  # nothing within reach of the view-0 camera: fewer than 100 near points
            blobs = [np.array(c) + rs.uniform(-0.2, 0.2, (300, 3)) for c in ((-3, 0, 1.5), (1.5, 6, 1.5))]
            pts = np.concatenate(blobs).astype(np.float32)
            out.append((pts, np.ones(len(pts), np.int64)))
        else:  # "small": a room whose scans see fewer than 300 points
            out.append(W.scene_room(2600, int(rs.randint(1 << 20))))
    return [(np.asarray(p, np.float32), np.asarray(lab, np.int64)) for p, lab in out]


CROP_NPOINTS = ["below", "equal", "one_under", "far_under", "max", "one"]


def draw_crops(rs, k=0):
    """the k-th draw of a seed puts npoints CROP_NPOINTS[k % 6] of crop 0's members"""
    nk = CROP_NPOINTS[k % len(CROP_NPOINTS)]
    kinds = ["big_room" if nk == "max" else "room"]
    kinds += [str(rs.choice(["room", "unlabelled", "duplicates"])) for _ in range(int(rs.randint(0, 3)))]
    scenes = draw_scenes(rs, kinds)
    b = int(rs.randint(1, 6))
    cs = rs.randint(0, len(scenes), b)
    cs[0] = 0
    if k % 2 == 1 or rs.rand() < 0.3:
        cs = np.concatenate([cs, [int(rs.choice([-1, len(scenes)]))]])
        b += 1
    seed, skind = draw_seed(rs)
    # npoints around crop 0's members: c is that of its chosen attempt
    pts, lab = scenes[0]
    att = CO.crop_attempts(pts, lab, pts[:, 2].min(), pts[:, 2].max(), seed, 0)
    c = len(att[CO.choose(att)]["members"])
    npoints = {"below": c + 1 + int(rs.randint(0, 100)), "equal": c, "one_under": c - 1, "far_under": max(1, c // 10),
               "max": R.MAX_ROWS, "one": 1}[nk]
    npoints = int(min(max(npoints, 1), R.MAX_ROWS))
    return dict(case="crops", kinds=kinds, scenes=scenes, b=b, crop_scene=cs, seed=seed, seed_kind=skind,
                npoints=npoints, npoints_kind=nk, context0=c, max_dropout=float(rs.choice([0.0, 0.875, 1.0])),
                rotate=bool(rs.rand() < 0.5), api=draw_api(rs))


SCAN_MODES = [-1, 0, 1, 2, 3, 4, 5, 6, 7, 8, -2]


def draw_vscan(rs, k=0):
    """the k-th draw of a seed takes scan modes SCAN_MODES[6 k ..] in turn"""
    kinds = ["big_room", "away" if k % 2 == 0 else "small"] + [str(rs.choice(["room", "away", "small"]))
                                                             for _ in range(int(rs.randint(0, 2)))]
    scenes = draw_scenes(rs, kinds)
    b = int(rs.randint(6, 8))
    ss = rs.randint(0, len(scenes), b)
    ss[:len(scenes)] = np.arange(len(scenes))
    if rs.rand() < 0.3:
        ss[int(rs.randint(1, b))] = int(rs.choice([-1, len(scenes)]))
    modes = np.array([SCAN_MODES[(6 * k + i) % len(SCAN_MODES)] for i in range(b)], np.int64)
    seed, skind = draw_seed(rs)
    npoints = int(rs.choice([1, 64, 500, 2047, 2048, 2049, 4096, 7000, R.MAX_ROWS]))
    return dict(case="vscan", kinds=kinds, scenes=scenes, b=b, scan_scene=ss, scan_mode=modes, seed=seed,
                seed_kind=skind, npoints=npoints, min_points=int(rs.choice([0, 300, 5000])), api=draw_api(rs))


# ---------------------------------------------------------------------------------------------------- refused
REFUSALS = ["voxel_nsample_0", "voxel_nsample_16385", "voxel_ws_short", "voxel_ws_misaligned", "voxel_bn_2_31",
            "voxel_bc_2_31", "shapes_npoints_0", "shapes_npoints_16385", "shapes_be_2_31", "crops_npoints_0",
            "crops_npoints_16385", "crops_ws_short", "crops_ws_misaligned", "crops_bn_2_31", "vscan_npoints_0",
            "vscan_npoints_16385", "vscan_b_4097", "vscan_ws_short", "vscan_ws_misaligned"]


def draw_refused(rs):
    """every refusal, each with its own poisoned outputs"""
    return dict(case="refused", whys=list(REFUSALS), seed=int(rs.randint(1 << 30)))


# ---------------------------------------------------------------------------------------------------- buffers
_LIVE = []  # device inputs of the running case: they must outlive the launch


def _ptr(t):
    import ctypes
    return None if t is None else ctypes.c_void_p(t.data_ptr())


def dev_in(a, dtype=None):
    t = torch.from_numpy(np.ascontiguousarray(a if dtype is None else np.asarray(a, dtype))).to(dev)
    _LIVE.append(t)
    return t


class Out:
    """a poisoned output of numel elements of a numpy dtype, with a poisoned guard after it"""

    def __init__(self, numel, dtype):
        self.numel, self.dtype = int(numel), np.dtype(dtype)
        self.raw = torch.full((self.numel * self.dtype.itemsize + GUARD,), POISON, dtype=torch.uint8, device=dev)
        _LIVE.append(self.raw)

    def ptr(self):
        return _ptr(self.raw)

    def host(self):
        """(body, guard untouched)"""
        a = self.raw.cpu().numpy()
        nb = self.numel * self.dtype.itemsize
        return a[:nb].view(self.dtype).copy(), bool((a[nb:] == POISON).all())

    def untouched(self):
        return bool((self.raw.cpu().numpy() == POISON).all())


def workspace(nbytes, misaligned=False):
    ws = torch.full((nbytes + 512,), 0x5A, dtype=torch.uint8, device=dev)
    _LIVE.append(ws)
    import ctypes
    return ctypes.c_void_p(ws.data_ptr() + (8 if misaligned else 0))


def seed_pair(p):
    """(launch argument, device seed tensor or None): with a device seed the launch argument is something else"""
    s = signed(p["seed"] & ((1 << 64) - 1)) if p["seed"] >= 0 else p["seed"]
    if p["seed_kind"] == "device":
        return s ^ 0x5A5A5A5A, dev_in(np.array([s], np.int64))
    return s, None


def wrapper_seed(p):
    if p["seed_kind"] == "device":
        return dev_in(np.array([signed(p["seed"] & ((1 << 64) - 1))], np.int64))
    return p["seed"]


# ------------------------------------------------------------------------------------------------ comparators
def bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.dtype(f"u{a.dtype.itemsize}")) if a.dtype.kind in "fb" else a


def compare(got: dict, want: dict, exact, ulp=None) -> list:
    """the names of the fields that differ: ``exact`` fields bit for bit (bools as bytes), ``ulp`` = {field: float64
    truth}, each value within one float32 ulp plus 1e-12; a field "guards" of False (a guard or pad overwritten)"""
    bad = [k for k, v in got.get("guards", {}).items() if not v]
    for f in exact:
        g, w = np.asarray(got[f]), np.asarray(want[f])
        if w.dtype == bool:  # flags: the C outputs are read back as bytes
            g, w = g.view(np.uint8) if g.dtype == bool else g, w.astype(np.uint8)
        if g.shape != w.shape or g.dtype != w.dtype or not np.array_equal(bits(g), bits(w)):
            bad.append(f)
    for f, truth in (ulp or {}).items():
        g = np.asarray(got[f], np.float64)
        tol = np.spacing(np.abs(truth).astype(np.float32)).astype(np.float64) + 1e-12
        poisoned = (bits(np.asarray(got[f], np.float32)) == np.uint32(0x01010101 * POISON)).any()
        if g.shape != truth.shape or poisoned or not (np.abs(g - truth) <= tol).all():
            bad.append(f)
    return bad


def _read(outs: dict) -> dict:
    got, guards = {}, {}
    for k, o in outs.items():
        got[k], guards[k] = o.host()
    got["guards"] = guards
    return got


# ------------------------------------------------------------------------------------------------------ oracle
def want_voxel(p):
    return dict(zip(("idx", "count", "grouped"), VO.oracle_voxel_group(p["xyz"], p["dim"], p["radius"], p["nsample"],
                                                                      p["seed"], p["dims"], p["lengths"])))


def shape_host(p):
    st = p["set"]
    sizes = np.asarray(p["sizes"], np.int64)
    off = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
    return dict(xyz=np.concatenate(st["xyz"]), label=np.asarray(st["label"], np.int32), offsets=off,
                normals=np.concatenate(st["normals"]) if st["normals"] is not None else None,
                part=np.concatenate(st["part"]) if st["part"] is not None else None)


def want_shapes(p):
    h = shape_host(p)
    return SH.oracle_shapes(h["xyz"], h["label"], h["offsets"], p["shape_idx"], p["seed"], p["npoints"], p["subset"],
                            p["rotate"], p["perturb"], p["scale"], p["shift"], p["jitter"], p["max_dropout"],
                            p["with_normals"], h["normals"], h["part"], p["votes"])


def scene_host(p):
    sc = p["scenes"]
    sizes = np.array([len(s[0]) for s in sc], np.int64)
    return dict(xyz=np.concatenate([s[0] for s in sc]), label=np.concatenate([s[1] for s in sc]).astype(np.int32),
                offsets=np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64), sizes=sizes,
                lo=np.stack([s[0].min(0) for s in sc]), hi=np.stack([s[0].max(0) for s in sc]),
                mean=np.stack([s[0].astype(np.float64).mean(0) for s in sc]),
                lw=(1 / np.log(1.2 + np.arange(1, 22, dtype=np.float32) / 231)).astype(np.float32))


def want_crops(p):
    h = scene_host(p)
    return CO.oracle_crops(h["xyz"], h["label"], h["offsets"], h["lo"], h["hi"], h["lw"], p["crop_scene"], p["seed"],
                           p["npoints"], p["max_dropout"], p["rotate"])


def want_vscan(p):
    h = scene_host(p)
    return SO.oracle_scans(h["xyz"], h["label"], h["offsets"], h["mean"], h["lw"], p["scan_scene"], p["scan_mode"],
                           p["seed"], p["npoints"], p["min_points"])


# --------------------------------------------------------------------------------------------------------- run
def lib():
    return _lib.load()


def run_voxel(p):
    b, n, S, dim, dims = p["b"], p["n"], p["nsample"], p["dim"], p["dims"]
    want = want_voxel(p)
    cells = dim ** dims
    xyz = dev_in(p["xyz"])
    lens = dev_in(p["lengths"], np.int32) if p["lengths"] is not None else None
    if p["api"] == "wrapper":
        from pointnet2_b200 import pc_util
        idx, count, grouped = pc_util.voxel_group(xyz, dim, p["radius"], S, wrapper_seed(p), dims=dims, lengths=lens)
        got = dict(idx=idx.cpu().numpy(), count=count.cpu().numpy(), grouped=grouped.cpu().numpy())
    else:
        outs = dict(count=Out(b * cells, np.int32), idx=Out(b * cells * S, np.int32),
                    grouped=Out(b * cells * S * 3, np.float64))
        wsb = int(lib().pn2_voxel_group_workspace_bytes(b, n, dim, dims))
        if wsb != R.voxel_workspace_bytes(b, n, dim, dims):
            return False
        sv, sd = seed_pair(p)
        rc = lib().pn2_voxel_group(b, n, _ptr(xyz), _ptr(lens), dim, dims, p["radius"], S, sv, _ptr(sd),
                                   outs["count"].ptr(), outs["idx"].ptr(), outs["grouped"].ptr(), workspace(wsb), wsb,
                                   None)
        if rc != 0:
            return False
        got = _read(outs)
        got["count"] = got["count"].reshape(b, cells)
        got["idx"] = got["idx"].reshape(b, cells, S)
        got["grouped"] = got["grouped"].reshape(b, cells, S, 3)
    return not compare(got, want, ("count", "idx", "grouped"))


run_voxel_planted = run_voxel
SHAPE_EXACT = ("label", "lengths", "point_idx")


def run_shapes(p):
    want = want_shapes(p)
    h = shape_host(p)
    ne = p["b"] * p["votes"] if p["votes"] else p["b"]
    ch = 6 if p["with_normals"] else 3
    exact = SHAPE_EXACT + (("part",) if p["parts"] else ())
    npoints = p["npoints"]
    if p["api"] == "wrapper":
        from pointnet2_b200 import shapes
        st = p["set"]
        ss = shapes.ShapeSet(st["xyz"], st["label"], st["normals"], st["part"], num_class=40, normalize=False,
                             device=dev)
        idx = dev_in(p["shape_idx"], np.int64)
        if p["votes"]:
            out = shapes.vote_batch(ss, idx, p["votes"], wrapper_seed(p), npoints, p["with_normals"])
        else:
            out = shapes.sample_shapes(ss, idx, wrapper_seed(p), npoints, p["subset"], p["rotate"], p["perturb"],
                                       p["scale"], p["shift"], p["jitter"], p["max_dropout"], p["with_normals"])
        got = {f: getattr(out, f).cpu().numpy() for f in ("points", "label", "lengths", "point_idx")}
        if p["parts"]:
            got["part"] = out.part.cpu().numpy()
    else:
        outs = dict(points=Out(ne * npoints * ch, np.float32), label=Out(ne, np.int64), lengths=Out(ne, np.int32),
                    point_idx=Out(ne * npoints, np.int32))
        if p["parts"]:
            outs["part"] = Out(ne * npoints, np.int64)
        sv, sd = seed_pair(p)
        sc = p["scale"] or (1.0, 1.0)
        jt = p["jitter"] or (0.0, 1.0)
        x, lab, off = dev_in(h["xyz"]), dev_in(h["label"]), dev_in(h["offsets"])
        nrm = dev_in(h["normals"]) if h["normals"] is not None else None
        part = dev_in(h["part"]) if h["part"] is not None else None
        rc = lib().pn2_shape_batch(len(p["sizes"]), int(sum(p["sizes"])), int(max(p["sizes"])), _ptr(x), _ptr(nrm),
                                   _ptr(lab), _ptr(part), _ptr(off), p["b"], _ptr(dev_in(p["shape_idx"], np.int64)),
                                   sv, _ptr(sd), p["votes"], npoints, int(p["subset"] == "random"), int(p["rotate"]),
                                   int(p["perturb"]), int(p["scale"] is not None), sc[0], sc[1], p["shift"],
                                   int(p["jitter"] is not None), jt[0], jt[1], p["max_dropout"], int(p["with_normals"]),
                                   outs["points"].ptr(), outs["label"].ptr(),
                                   outs["part"].ptr() if p["parts"] else None, outs["lengths"].ptr(),
                                   outs["point_idx"].ptr(), None)
        if rc != 0:
            return False
        got = _read(outs)
        got["points"] = got["points"].reshape(ne, npoints, ch)
        for f in ("point_idx", "part"):
            if f in got:
                got[f] = got[f].reshape(ne, npoints)
    return not compare(got, want, exact, {"points": want["points64"]})


run_shapes_planted = run_shapes
CROP_EXACT = ("label", "weight", "lengths", "point_idx", "core", "attempt", "valid")


def run_crops(p):
    want = want_crops(p)
    h = scene_host(p)
    b, npoints = p["b"], p["npoints"]
    lw = dev_in(h["lw"])
    if p["api"] == "wrapper":
        from pointnet2_b200 import scene
        ss = scene.SceneSet([s[0] for s in p["scenes"]], [s[1] for s in p["scenes"]], num_class=21, device=dev)
        out = scene.sample_crops(ss, dev_in(p["crop_scene"], np.int64), wrapper_seed(p), lw, npoints,
                                 p["max_dropout"], p["rotate"])
        got = {f: getattr(out, f).cpu().numpy() for f in ("xyz",) + CROP_EXACT}
    else:
        outs = dict(xyz=Out(b * npoints * 3, np.float32), label=Out(b * npoints, np.int64),
                    weight=Out(b * npoints, np.float32), lengths=Out(b, np.int32), point_idx=Out(b * npoints, np.int32),
                    core=Out(b * npoints, np.uint8), attempt=Out(b, np.int32), valid=Out(b, np.uint8))
        wsb = int(lib().pn2_scene_crops_workspace_bytes(b, npoints))
        if wsb != R.crops_workspace_bytes(b, npoints):
            return False
        sv, sd = seed_pair(p)
        rc = lib().pn2_scene_crops(len(h["sizes"]), int(h["sizes"].sum()), int(h["sizes"].max()),
                                   _ptr(dev_in(h["xyz"])), _ptr(dev_in(h["label"])), _ptr(dev_in(h["offsets"])), _ptr(dev_in(h["lo"])),
                                   _ptr(dev_in(h["hi"])), 21, _ptr(lw), b, _ptr(dev_in(p["crop_scene"], np.int64)), sv,
                                   _ptr(sd), npoints, p["max_dropout"], int(p["rotate"]), *[outs[k].ptr() for k in
                                   ("xyz", "label", "weight", "lengths", "point_idx", "core", "attempt", "valid")],
                                   workspace(wsb), wsb, None)
        if rc != 0:
            return False
        got = _read(outs)
        for f in ("label", "weight", "point_idx", "core"):
            got[f] = got[f].reshape(b, npoints)
        got["xyz"] = got["xyz"].reshape(b, npoints, 3)
    if p["rotate"]:
        return not compare(got, want, CROP_EXACT, {"xyz": want["xyz64"]})
    return not compare(got, want, CROP_EXACT + ("xyz",))


SCAN_FIELDS = ("xyz", "label", "weight", "lengths", "point_idx", "visible", "valid")


def run_vscan(p):
    want = want_vscan(p)
    h = scene_host(p)
    b, npoints = p["b"], p["npoints"]
    lw = dev_in(h["lw"])
    if p["api"] == "wrapper":
        from pointnet2_b200 import scene
        ss = scene.SceneSet([s[0] for s in p["scenes"]], [s[1] for s in p["scenes"]], num_class=21, device=dev)
        out = scene.sample_virtual_scans(ss, dev_in(p["scan_scene"], np.int64), dev_in(p["scan_mode"], np.int64),
                                         wrapper_seed(p), lw, npoints, p["min_points"])
        got = {f: getattr(out, f).cpu().numpy() for f in SCAN_FIELDS}
    else:
        outs = dict(xyz=Out(b * npoints * 3, np.float32), label=Out(b * npoints, np.int64),
                    weight=Out(b * npoints, np.float32), lengths=Out(b, np.int32), point_idx=Out(b * npoints, np.int32),
                    visible=Out(b, np.int32), valid=Out(b, np.uint8))
        ms = int(h["sizes"].max())
        wsb = int(lib().pn2_virtual_scans_workspace_bytes(b, ms, npoints))
        if wsb != R.vscan_workspace_bytes(b, ms, npoints):
            return False
        sv, sd = seed_pair(p)
        rc = lib().pn2_virtual_scans(len(h["sizes"]), int(h["sizes"].sum()), ms, _ptr(dev_in(h["xyz"])),
                                     _ptr(dev_in(h["label"])), _ptr(dev_in(h["offsets"])), _ptr(dev_in(h["mean"])), 21,
                                     _ptr(lw), b, _ptr(dev_in(p["scan_scene"], np.int64)),
                                     _ptr(dev_in(p["scan_mode"], np.int64)), sv, _ptr(sd), npoints, p["min_points"],
                                     *[outs[k].ptr() for k in SCAN_FIELDS], workspace(wsb), wsb, None)
        if rc != 0:
            return False
        got = _read(outs)
        for f in ("label", "weight", "point_idx"):
            got[f] = got[f].reshape(b, npoints)
        got["xyz"] = got["xyz"].reshape(b, npoints, 3)
    # an exact comparison needs every decision of the oracle a margin above 1e-12: entries without one are left out
    ok = want["margin"] > 1e-12
    def sub(d):
        return {k: (v[ok] if k != "guards" else v) for k, v in d.items() if k in SCAN_FIELDS or k == "guards"}
    return not compare(sub(got), sub(want), SCAN_FIELDS)


def run_refused(p):
    return all(refused_one(p, why) for why in p["whys"])


def refused_one(p, why):
    L = lib()
    op, rest = why.split("_", 1)
    small = Out(4096, np.int32)
    outs = [Out(256, np.int32) for _ in range(8)]
    buf = dev_in(np.zeros(4096, np.float32))
    i64 = dev_in(np.zeros(64, np.int64))
    P = [o.ptr() for o in outs]
    torch.cuda.synchronize(dev)
    before = _lib.launch_count()
    if op == "voxel":
        b, n, dim, dims, S = 1, 300, 3, 3, 32
        if rest.startswith("nsample"):
            S = 0 if rest.endswith("_0") else R.MAX_ROWS + 1
        if rest == "bn_2_31":
            b, n = 2, 1 << 30
        if rest == "bc_2_31":
            b, dim = 2, 1025
        wsb = R.voxel_workspace_bytes(1, 300, 3, 3)
        rc = L.pn2_voxel_group(b, n, _ptr(buf), None, dim, dims, 1.0, S, p["seed"], None, P[0], P[1], P[2],
                               workspace(wsb, rest == "ws_misaligned"), wsb - (rest == "ws_short"), None)
    elif op == "shapes":
        b, npoints = 2, 64
        if rest.startswith("npoints"):
            npoints = 0 if rest.endswith("_0") else R.MAX_ROWS + 1
        if rest == "be_2_31":
            b, npoints = 65536, R.MAX_ROWS
        off = dev_in(np.array([0, 100], np.int64))
        rc = L.pn2_shape_batch(1, 100, 100, _ptr(buf), None, _ptr(small.raw), None, _ptr(off), b, _ptr(i64), p["seed"],
                               None, 0, npoints, 0, 0, 0, 0, 1.0, 1.0, 0.0, 0, 0.0, 1.0, 0.0, 0, P[0], P[1], None,
                               P[2], P[3], None)
    elif op == "crops":
        b, npoints = 2, 64
        if rest.startswith("npoints"):
            npoints = 0 if rest.endswith("_0") else R.MAX_ROWS + 1
        if rest == "bn_2_31":
            b, npoints = 65535, R.MAX_ROWS
        wsb = R.crops_workspace_bytes(2, 64)
        off = dev_in(np.array([0, 100], np.int64))
        rc = L.pn2_scene_crops(1, 100, 100, _ptr(buf), _ptr(small.raw), _ptr(off), _ptr(buf), _ptr(buf), 21, _ptr(buf),
                               b, _ptr(i64), p["seed"], None, npoints, 0.5, 1, *P, workspace(wsb, rest == "ws_misaligned"),
                               wsb - (rest == "ws_short"), None)
    else:
        b, npoints = 2, 64
        if rest.startswith("npoints"):
            npoints = 0 if rest.endswith("_0") else R.MAX_ROWS + 1
        if rest == "b_4097":
            b = R.SCAN_MAX_BATCH + 1
        wsb = R.vscan_workspace_bytes(2, 100, 64)
        off = dev_in(np.array([0, 100], np.int64))
        mean = dev_in(np.zeros(3, np.float64))
        rc = L.pn2_virtual_scans(1, 100, 100, _ptr(buf), _ptr(small.raw), _ptr(off), _ptr(mean), 21, _ptr(buf), b,
                                 _ptr(i64), _ptr(i64), p["seed"], None, npoints, 300, *P[:7],
                                 workspace(wsb, rest == "ws_misaligned"), wsb - (rest == "ws_short"), None)
    launched = _lib.launch_count() - before
    torch.cuda.synchronize(dev)
    return rc == CUDA_ERROR_INVALID_VALUE and launched == 0 and all(o.untouched() for o in outs)


CASES = ["voxel", "voxel_planted", "shapes", "shapes_planted", "crops", "vscan", "refused"]
DRAW = {name: globals()["draw_" + name] for name in CASES}
RUN = {name: globals()["run_" + name] for name in CASES}
# draws that are told their index k among the seed's draws of that case (to cycle through fixed edges)
COUNTED = ("voxel", "voxel_planted", "shapes", "shapes_planted", "crops", "vscan")


def draws(seed: int, iterations: int):
    """The parameters ``run(seed, iterations)`` uses, without a device (the run_* functions draw nothing)."""
    rs = np.random.RandomState(seed)
    return [_draw(rs, it) for it in range(iterations)]


def _draw(rs, it):
    name = SCHEDULE[it % len(SCHEDULE)]
    if name in COUNTED:
        return DRAW[name](rs, sum(1 for i in range(it) if SCHEDULE[i % len(SCHEDULE)] == name))
    return DRAW[name](rs)


def public(p):
    """the parameters of a case without its input arrays (they follow from the seed and the iteration)"""
    keep = ("sizes", "kinds", "whys")
    return {k: v for k, v in p.items() if not isinstance(v, (np.ndarray, list, dict)) or k in keep}


def _one(rs, seed, it, counts, fails, catch):
    name = SCHEDULE[it % len(SCHEDULE)]
    p = _draw(rs, it)
    _LIVE.clear()
    try:
        ok = RUN[name](p)
    except Exception as e:  # noqa: BLE001 — report the exception as a failure of that case
        if not catch:
            raise
        ok = False
        p = dict(p, error=f"{type(e).__name__}: {e}")
    _LIVE.clear()
    counts[name] = counts.get(name, 0) + 1
    if not ok:
        fails.append(dict(public(p), seed=seed, iteration=it))
    return name, ok


def run(seed: int, iterations: int):
    """``iterations`` random cases in SCHEDULE order; returns (counts, failures)."""
    rs = np.random.RandomState(seed)
    counts, fails = {}, []
    for it in range(iterations):
        _one(rs, seed, it, counts, fails, catch=True)
    return counts, fails


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=float, default=120)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--iterations", type=int, default=None, help="stop after this many cases")
    ap.add_argument("--json", type=str, default=None)
    args = ap.parse_args()
    rs = np.random.RandomState(args.seed)
    counts, fails, secs = {}, [], {}
    t0 = time.time()
    it = 0
    while time.time() - t0 < args.seconds and (args.iterations is None or it < args.iterations):
        t1 = time.time()
        name, ok = _one(rs, args.seed, it, counts, fails, catch=True)
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
