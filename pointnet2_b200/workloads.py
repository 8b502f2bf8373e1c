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
