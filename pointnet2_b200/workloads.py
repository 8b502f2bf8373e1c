"""Synthetic input recipes for the set-abstraction path (SURVEY.md §8d), shared by bench.py and the
tests.  All numpy, all seeded, no I/O.

Distributions (the reference ships no data; these replay what its loaders feed the ops):
  U  uniform [0,1)^3 — the reference's own op smoke-test distribution (tf_grouping.py:79-88).
  S  surface-like: points on random axis-aligned box / sphere surfaces, then pc_normalize
     (modelnet_dataset.py:15-21: centre, scale to unit max radius) -> coordinates in [-1,1].
  D  duplicates: N draws WITH replacement from 0.3N distinct points in a 1.5 x 1.5 x 3 block,
     then a random <= 87.5 % of rows overwritten by row 0 (scannet_dataset.py:54 resampling and
     scannet/train.py:192-196 point dropout) — exercises FPS ties and ball-query early exit.
"""
from __future__ import annotations

import numpy as np

F32 = np.float32


def cloud_uniform(b: int, n: int, seed: int) -> np.ndarray:
    return np.random.RandomState(seed).random_sample((b, n, 3)).astype(F32)


def pc_normalize(pc: np.ndarray) -> np.ndarray:
    pc = pc - pc.mean(axis=0, keepdims=True)
    m = np.sqrt((pc.astype(np.float64) ** 2).sum(axis=1)).max()
    return (pc / max(m, 1e-12)).astype(F32)


def cloud_surface(b: int, n: int, seed: int) -> np.ndarray:
    rs = np.random.RandomState(seed)
    out = np.empty((b, n, 3), F32)
    for i in range(b):
        parts, left = [], n
        nshape = rs.randint(2, 5)
        for s in range(nshape):
            cnt = left if s == nshape - 1 else max(1, left // (nshape - s))
            left -= cnt
            ctr = rs.uniform(-0.5, 0.5, 3)
            if rs.rand() < 0.5:  # sphere surface
                v = rs.normal(size=(cnt, 3))
                v /= np.maximum(np.linalg.norm(v, axis=1, keepdims=True), 1e-9)
                p = ctr + v * rs.uniform(0.2, 0.6)
            else:  # box surface: pick a face, uniform on it
                half = rs.uniform(0.15, 0.6, 3)
                p = rs.uniform(-1, 1, (cnt, 3)) * half
                ax = rs.randint(0, 3, cnt)
                sg = rs.choice([-1.0, 1.0], cnt)
                p[np.arange(cnt), ax] = sg * half[ax]
                p = ctr + p
            parts.append(p)
        pc = np.concatenate(parts, 0)
        rs.shuffle(pc)
        out[i] = pc_normalize(pc)
    return out


def cloud_duplicates(b: int, n: int, seed: int, drop: bool = True) -> np.ndarray:
    rs = np.random.RandomState(seed)
    out = np.empty((b, n, 3), F32)
    distinct = max(1, int(0.3 * n))
    for i in range(b):
        base = (rs.random_sample((distinct, 3)) * np.array([1.5, 1.5, 3.0])).astype(F32)
        pc = base[rs.randint(0, distinct, n)]
        if drop:
            ratio = rs.random_sample() * 0.875
            pc[rs.random_sample(n) <= ratio] = pc[0]
        out[i] = pc
    return out


DISTRIBUTIONS = {"U": cloud_uniform, "S": cloud_surface, "D": cloud_duplicates}


def features(b: int, n: int, c: int, seed: int) -> np.ndarray:
    return np.random.RandomState(seed).standard_normal((b, n, c)).astype(F32)


def part_shapes(b: int, n: int, seed: int, offsets):
    """A synthetic part-segmentation batch (the reference's ShapeNet part data is not shipped): (b, n, 6) float32
    points (xyz, then unit normals), (b,) int64 categories and (b, n) int64 part labels.  Category k of the
    len(offsets) - 1 is a sphere, a cylinder side or a box surface (k mod 3), taller with k // 3, with analytic normals,
    rotated about the up axis, scaled and centred into the unit sphere.  Its parts offsets[k] .. offsets[k + 1] - 1
    are equal height bands, bottom to top."""
    rs = np.random.RandomState(seed)
    cls = rs.randint(0, len(offsets) - 1, b)
    pts = np.empty((b, n, 6), F32)
    label = np.empty((b, n), np.int64)
    rows = np.arange(n)
    for i, k in enumerate(cls):
        th, z = 2 * np.pi * rs.rand(n), 2 * rs.rand(n) - 1
        kind = k % 3
        if kind == 0:    # sphere
            r = np.sqrt(1 - z * z)
            p = np.stack([r * np.cos(th), r * np.sin(th), z], 1)
            nrm = p.copy()
        elif kind == 1:  # cylinder side
            p = np.stack([np.cos(th), np.sin(th), z], 1)
            nrm = np.stack([np.cos(th), np.sin(th), np.zeros(n)], 1)
        else:            # box surface
            p = rs.uniform(-1, 1, (n, 3))
            ax, sg = rs.randint(0, 3, n), rs.choice([-1.0, 1.0], n)
            p[rows, ax] = sg
            nrm = np.zeros((n, 3))
            nrm[rows, ax] = sg
        h = 1.0 + 0.25 * (k // 3)  # stretch z by h: the normals scale by 1 / h there
        p[:, 2] *= h
        nrm[:, 2] /= h
        nrm /= np.linalg.norm(nrm, axis=1, keepdims=True)
        a = rs.uniform(0, 2 * np.pi)
        rot = np.array([[np.cos(a), -np.sin(a), 0], [np.sin(a), np.cos(a), 0], [0, 0, 1]])
        p, nrm = p @ rot.T, nrm @ rot.T
        parts = offsets[k + 1] - offsets[k]
        zq = (p[:, 2] - p[:, 2].min()) / max(np.ptp(p[:, 2]), 1e-12)
        label[i] = offsets[k] + np.minimum((zq * parts).astype(np.int64), parts - 1)
        pts[i, :, :3] = pc_normalize(p * rs.uniform(0.8, 1.25))
        pts[i, :, 3:] = nrm
    return pts, cls.astype(np.int64), label


def scene_room(p: int, seed: int):
    """A synthetic indoor scene (the reference's ScanNet data is not shipped): (p, 3) float32 points in metres and (p,)
    int64 labels in 0..20.  A rectangular room whose floor area grows with p (about 5000 points per square metre of floor,
    a 1.5e5-point room is about 5.5 m across): floor (label 2), four 2.5 m walls (1), box furniture on the floor, each
    box's surface carrying one label of 3..20, 3 % unlabelled clutter (0) anywhere in the room, and 2 % of the rows
    exact duplicates of other rows.  Rows are shuffled."""
    rs = np.random.RandomState(seed)
    side = 5.5 * np.sqrt(max(p, 1) / 1.5e5)
    w, d, h = side * rs.uniform(0.9, 1.1), side * rs.uniform(0.8, 1.0), 2.5
    n_floor, n_wall, n_clutter = int(0.35 * p), int(0.30 * p), int(0.03 * p)
    n_dup = int(0.02 * p)
    n_furn = p - n_floor - n_wall - n_clutter - n_dup
    floor = np.stack([rs.uniform(0, w, n_floor), rs.uniform(0, d, n_floor), np.zeros(n_floor)], 1)
    # walls: perimeter parameter t in [0, 2(w + d)), height uniform
    t = rs.uniform(0, 2 * (w + d), n_wall)
    wx = np.select([t < w, t < w + d, t < 2 * w + d], [t, w, 2 * w + d - t], 0.0)
    wy = np.select([t < w, t < w + d, t < 2 * w + d], [0.0, t - w, d], 2 * (w + d) - t)
    wall = np.stack([wx, wy, rs.uniform(0, h, n_wall)], 1)
    # furniture: boxes resting on the floor, points on their five visible faces
    nbox = max(1, int(round(w * d / 4)))
    size = rs.uniform([0.4, 0.4, 0.4], [2.0, 1.2, 1.8], (nbox, 3))
    corner = rs.uniform(0, 1, (nbox, 2)) * np.maximum(np.array([w, d]) - size[:, :2], 0)
    box_label = rs.randint(3, 21, nbox)
    which = rs.randint(0, nbox, n_furn)
    fp = rs.uniform(0, 1, (n_furn, 3))
    face = rs.randint(0, 5, n_furn)  # 0..3: side faces, 4: top
    ax = np.where(face < 2, 0, np.where(face < 4, 1, 2))
    fp[np.arange(n_furn), ax] = np.where(face == 4, 1.0, (face % 2).astype(np.float64))
    furn = fp * size[which]
    furn[:, :2] += corner[which]
    clutter = rs.uniform(0, 1, (n_clutter, 3)) * np.array([w, d, h])
    pts = np.concatenate([floor, wall, furn, clutter], 0)
    lab = np.concatenate([np.full(n_floor, 2), np.full(n_wall, 1), box_label[which], np.zeros(n_clutter, np.int64)])
    dup = rs.randint(0, len(pts), n_dup) if len(pts) else np.zeros(0, np.int64)
    pts, lab = np.concatenate([pts, pts[dup]], 0), np.concatenate([lab, lab[dup]])
    order = rs.permutation(len(pts))
    return pts[order].astype(F32), lab[order].astype(np.int64)


# ---- BASELINE.json configs ---------------------------------------------------------------------
CFG2_SSG_SA = dict(name="cfg2_ssg_sa_layer", b=32, n=4096, npoint=1024, nsample=32, radius=0.1, dist="U", seed=100)
CFG1_FPS_CPU = dict(name="cfg1_fps_plumbing", b=8, n=1024, npoint=512, dist="U", seed=100)
CFG3_MSG = dict(name="cfg3_msg_cls", b=32, n=1024, dist="S", seed=100,
                layers=[dict(npoint=512, radii=[0.1, 0.2, 0.4], nsamples=[16, 32, 128], c=0),
                        dict(npoint=128, radii=[0.2, 0.4, 0.8], nsamples=[32, 64, 128], c=320)])
CFG4_SEMSEG = dict(name="cfg4_scannet_semseg", b=16, n=8192, dist="D", seed=100,
                   sa=[dict(npoint=1024, radius=0.1, nsample=32, c=0), dict(npoint=256, radius=0.2, nsample=32, c=64),
                       dict(npoint=64, radius=0.4, nsample=32, c=128), dict(npoint=16, radius=0.8, nsample=32, c=256)],
                   fp=[dict(n=64, m=16, c=512), dict(n=256, m=64, c=256), dict(n=1024, m=256, c=256),
                       dict(n=8192, m=1024, c=128)])
CFG5_SWEEP = dict(name="cfg5_sweep", b=8, ns=[4096, 16384, 65536, 262144], nsample=32, radius=0.1, dist="U")


# ---- algorithmic bytes (BASELINE.md §4): each tensor touched once -------------------------------
# `esz` is the size of a FEATURE element (4 = float32, 2 = bfloat16 / float16); coordinates, weights and indices are
# always 4 bytes.
def bytes_fps(b, n, m, with_new_xyz=False):
    return 12 * b * n + 4 * b * m + (12 * b * m if with_new_xyz else 0)


def bytes_gather(b, m):
    return 4 * b * m + 12 * b * m + 12 * b * m


def bytes_ball_query(b, n, m, s):
    return 12 * b * n + 12 * b * m + 4 * b * m * s + 4 * b * m


def bytes_group(b, n, m, s, c, esz=4):
    return 4 * b * m * s + esz * b * min(n, m * s) * c + esz * b * m * s * c


def bytes_three_nn(b, n, m):
    return 12 * b * n + 12 * b * m + 24 * b * n


def bytes_three_interpolate(b, n, m, c, esz=4):
    return esz * b * m * c + 24 * b * n + esz * b * n * c


def bytes_group_concat(b, n, m, s, c, esz=4):
    """group_concat: idx, xyz + features of the distinct source rows, (3 + c)-wide output rows."""
    return 4 * b * m * s + (12 + esz * c) * b * min(n, m * s) + esz * b * m * s * (3 + c)


def bytes_three_interpolate_grad(b, n, m, c, esz=4):
    """three_interpolate's gradient: grad_out read, grad_points written (read-modify-write for the atomics)."""
    return 2 * esz * b * m * c + 24 * b * n + esz * b * n * c


def bytes_fp_interpolate_concat(b, n, m, c2, c1, esz=4):
    return 12 * b * n + 12 * b * m + esz * b * m * c2 + esz * b * n * c1 + esz * b * n * (c2 + c1)


def bytes_sa_layer(b, n, m, s, c=3):
    """FPS + gather_point + query_ball_point + group_point(xyz): the metric's unit of work."""
    return bytes_fps(b, n, m) + bytes_gather(b, m) + bytes_ball_query(b, n, m, s) + bytes_group(b, n, m, s, c)
