"""Plain numpy restatement of the shape batches (pointnet2_b200.shapes.sample_shapes / vote_batch, DESIGN.md §6.11) for
the tests and tools/shape_batch_bench.py (test infrastructure only).

The draws are crop_oracle's ``draw`` / ``unit``, with the streams of §6.11:
normal           Box-Muller over two draws
entry_transform  the entry's matrix M, scale, shift and dropout threshold
row_order        a pool's rows in ascending (key, row) order
oracle_shapes    every output field, one entry at a time, vectorised over rows; the points also in float64
"""
from __future__ import annotations

import numpy as np

from crop_oracle import draw, unit

STREAM_KEY, STREAM_RATIO, STREAM_DROP, STREAM_ANGLE, STREAM_PERTURB, STREAM_SCALE, STREAM_SHIFT, STREAM_JITTER = range(1, 9)


def normal(seed: int, s: int, e: int, i):
    """sqrt(-2 ln(1 - u(draw(seed,s,e,2i)))) * cos(2 pi u(draw(seed,s,e,2i+1))); ``i`` may be an array."""
    i = np.asarray(i, np.uint64)
    u1 = unit(draw(seed, s, e, 2 * i))
    u2 = unit(draw(seed, s, e, 2 * i + np.uint64(1)))
    return np.sqrt(-2.0 * np.log(1.0 - u1)) * np.cos(2.0 * np.pi * u2)


def rot_x(a):
    return np.array([[1, 0, 0], [0, np.cos(a), -np.sin(a)], [0, np.sin(a), np.cos(a)]])


def rot_y(a):
    return np.array([[np.cos(a), 0, np.sin(a)], [0, 1, 0], [-np.sin(a), 0, np.cos(a)]])


def rot_z(a):
    return np.array([[np.cos(a), -np.sin(a), 0], [np.sin(a), np.cos(a), 0], [0, 0, 1]])


def perturb_angles(seed: int, e: int):
    return np.clip(0.06 * normal(seed, STREAM_PERTURB, e, np.arange(3)), -0.18, 0.18)


def entry_transform(seed: int, e: int, rotate=True, perturb=True, scale=(0.8, 1.25), shift=0.1, max_dropout=0.0,
                    vote=None):
    """M (3x3, p' = p M), s, t (3,) and the dropout ratio of entry e.  vote=(v, V): the vote's rotation, nothing else."""
    m = np.eye(3)
    if vote is not None:
        v, nv = vote
        return {"m": rot_y(v / float(nv) * np.pi * 2), "s": None, "t": None, "ratio": None}
    if rotate:
        m = rot_y(unit(draw(seed, STREAM_ANGLE, e, 0)) * 2 * np.pi)
    if perturb:
        a = perturb_angles(seed, e)
        m = m @ (rot_z(a[2]) @ (rot_y(a[1]) @ rot_x(a[0])))
    s = scale[0] + (scale[1] - scale[0]) * unit(draw(seed, STREAM_SCALE, e, 0)) if scale is not None else None
    t = -shift + 2 * shift * unit(draw(seed, STREAM_SHIFT, e, np.arange(3))) if shift > 0 else None
    ratio = unit(draw(seed, STREAM_RATIO, e, 0)) * max_dropout if max_dropout > 0 else None
    return {"m": m if (rotate or perturb) else None, "s": s, "t": t, "ratio": ratio}


def row_order(seed: int, e: int, q: int) -> np.ndarray:
    """Rows 0 .. q-1 in ascending (draw(seed, 1, e, j) >> 32, j) order."""
    j = np.arange(q)
    key = draw(seed, STREAM_KEY, e, j.astype(np.uint64)) >> np.uint64(32)
    return np.lexsort((j, key))


def oracle_shapes(xyz, label, offsets, shape_idx, seed: int, npoints=1024, subset="first", rotate=True, perturb=True,
                  scale=(0.8, 1.25), shift=0.1, jitter=(0.01, 0.05), max_dropout=0.0, with_normals=False, normals=None,
                  part=None, votes=0) -> dict:
    """The fields of sample_shapes (votes=0) or vote_batch (votes=V) as numpy arrays, for a shape set given as host
    arrays (xyz (P, 3) float32, label (S,), offsets (S + 1,), normals (P, 3) float32 or None, part (P,) or None), plus
    ``points64``, the points in float64 before the final rounding."""
    xyz = np.asarray(xyz, np.float32)
    shape_idx = np.asarray(shape_idx, np.int64)
    b = len(shape_idx)
    ne = b * votes if votes else b
    ch = 6 if with_normals else 3
    out = {"points": np.zeros((ne, npoints, ch), np.float32), "points64": np.zeros((ne, npoints, ch)),
           "label": np.zeros(ne, np.int64), "lengths": np.zeros(ne, np.int32),
           "point_idx": np.full((ne, npoints), -1, np.int32)}
    if part is not None:
        out["part"] = np.zeros((ne, npoints), np.int64)
    for e in range(ne):
        v, i = (e // b, e % b) if votes else (0, e)
        sv = int(shape_idx[i])
        if not 0 <= sv < len(offsets) - 1:
            continue
        o0, o1 = int(offsets[sv]), int(offsets[sv + 1])
        ps = o1 - o0
        q = ps if (subset == "random" and not votes) else min(ps, npoints)
        rows = row_order(seed, e, q)[:npoints]
        m = len(rows)
        if votes:
            x = entry_transform(seed, e, vote=(v, votes))
            jit = None
        else:
            x = entry_transform(seed, e, rotate, perturb, scale, shift, max_dropout)
            jit = jitter
        r = np.arange(m)
        keep = np.ones(m, bool)
        if x["ratio"] is not None:
            keep = unit(draw(seed, STREAM_DROP, e, r.astype(np.uint64))) > x["ratio"]
            keep[0] = True
        g = o0 + rows
        p = xyz[g].astype(np.float64)
        if x["m"] is not None:
            p = p[:, 0:1] * x["m"][0] + p[:, 1:2] * x["m"][1] + p[:, 2:3] * x["m"][2]
        if x["s"] is not None:
            p = p * x["s"]
        if x["t"] is not None:
            p = p + x["t"]
        if jit is not None:
            k = 3 * r[:, None] + np.arange(3)
            p = p + np.clip(jit[0] * normal(seed, STREAM_JITTER, e, k), -jit[1], jit[1])
        if with_normals:
            n = np.asarray(normals, np.float32)[g].astype(np.float64)
            if x["m"] is not None:
                n = n[:, 0:1] * x["m"][0] + n[:, 1:2] * x["m"][1] + n[:, 2:3] * x["m"][2]
            p = np.concatenate([p, n], 1)
        p, g = p[keep], g[keep]
        n_keep = len(g)
        out["points64"][e, :n_keep] = p
        out["points"][e, :n_keep] = p.astype(np.float32)
        out["label"][e] = int(label[sv])
        out["lengths"][e] = n_keep
        out["point_idx"][e, :n_keep] = g
        if part is not None:
            out["part"][e, :n_keep] = np.asarray(part)[g]
    return out
