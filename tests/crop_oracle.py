"""Plain numpy restatement of the training crops (pointnet2_b200.scene.sample_crops, DESIGN.md §6.10) for the tests and
tools/scene_crop_bench.py (test infrastructure only).

draw / unit      the counter-based random draws, in uint64 wrap-around arithmetic
crop_attempts    the ten attempts of one crop: context members, core mask, voxel count, validity
oracle_crops     every output field of sample_crops, one crop at a time, vectorised over points; xyz also in float64;
                 a crop whose scene index is outside [0, S) is empty, attempt -1
"""
from __future__ import annotations

import numpy as np

M64 = (1 << 64) - 1
G = np.uint64(0x9E3779B97F4A7C15)
ATTEMPTS = 10
STREAM_CENTRE, STREAM_KEY, STREAM_RATIO, STREAM_DROP, STREAM_ANGLE = 1, 2, 3, 4, 5


def _u64(v):
    return np.asarray(v, dtype=np.uint64)


def mix(x):
    """SplitMix64's finaliser on uint64 arrays."""
    with np.errstate(over="ignore"):
        x = _u64(x)
        x = x ^ (x >> np.uint64(30))
        x = x * np.uint64(0xBF58476D1CE4E5B9)
        x = x ^ (x >> np.uint64(27))
        x = x * np.uint64(0x94D049BB133111EB)
        x = x ^ (x >> np.uint64(31))
    return x


def draw(seed: int, stream: int, b: int, i):
    """mix(mix(mix(seed + stream*G) + b*G) + i*G), the seed taken as uint64 (two's complement); ``i`` may be an array."""
    with np.errstate(over="ignore"):
        h = mix(_u64(seed & M64) + _u64(stream) * G)
        h = mix(h + _u64(b) * G)
        return mix(h + _u64(i) * G)


def unit(d):
    """(d >> 11) * 2^-53: a double in [0, 1)."""
    return (_u64(d) >> np.uint64(11)).astype(np.float64) * 2.0 ** -53


def crop_attempts(pts: np.ndarray, labels: np.ndarray, lo_z: np.float32, hi_z: np.float32, seed: int, b: int):
    """The ten attempts of crop b on one scene (float32 (P, 3) points, integer labels): a list of dicts with the context
    members (ascending scene-local index), their core mask, the voxel count V and the validity."""
    out = []
    for a in range(ATTEMPTS):
        centre = pts[int(draw(seed, STREAM_CENTRE, b, a)) % len(pts)].astype(np.float64)
        curmin = np.array([centre[0] - 0.75, centre[1] - 0.75, np.float64(lo_z)])
        curmax = np.array([centre[0] + 0.75, centre[1] + 0.75, np.float64(hi_z)])
        p64 = pts.astype(np.float64)
        ctx = np.all((p64 >= curmin - 0.2) & (p64 <= curmax + 0.2), axis=1)
        members = np.nonzero(ctx)[0]
        core = np.all((p64[members] >= curmin - 0.01) & (p64[members] <= curmax + 0.01), axis=1)
        v = np.ceil((p64[members][core] - curmin) / (curmax - curmin) * np.array([31.0, 31.0, 62.0]))
        keys = v[:, 0] * 31.0 * 62.0 + v[:, 1] * 62.0 + v[:, 2]
        nvox = len(np.unique(keys))
        labelled = int(np.sum(labels[members] > 0))
        valid = labelled / len(members) >= 0.7 and nvox / 31.0 / 31.0 / 62.0 >= 0.02
        out.append({"members": members, "core": core, "nvox": nvox, "valid": bool(valid), "keys": keys})
    return out


def choose(attempts) -> int:
    """The first valid attempt, otherwise the last."""
    for a, t in enumerate(attempts):
        if t["valid"]:
            return a
    return ATTEMPTS - 1


def row_order(members: np.ndarray, seed: int, b: int) -> np.ndarray:
    """Positions into ``members`` in ascending (draw(seed, 2, b, j) >> 32, j) order."""
    key = draw(seed, STREAM_KEY, b, members.astype(np.uint64)) >> np.uint64(32)
    return np.lexsort((members, key))


def oracle_crops(xyz, label, offsets, lo, hi, label_weights, crop_scene, seed: int, npoints=8192, max_dropout=0.875,
                 rotate=True) -> dict:
    """The fields of sample_crops as numpy arrays for a scene set given as host arrays (xyz (P, 3) float32, label (P,),
    offsets (S + 1,), lo / hi (S, 3) float32, label_weights (C,) float32, crop_scene (B,)), plus ``xyz64``, the
    coordinates in float64 before the final rounding."""
    xyz = np.asarray(xyz, np.float32)
    label = np.asarray(label)
    lw = np.asarray(label_weights, np.float32)
    bsz = len(crop_scene)
    out = {"xyz": np.zeros((bsz, npoints, 3), np.float32), "xyz64": np.zeros((bsz, npoints, 3), np.float64),
           "label": np.zeros((bsz, npoints), np.int64), "weight": np.zeros((bsz, npoints), np.float32),
           "lengths": np.zeros(bsz, np.int32), "point_idx": np.full((bsz, npoints), -1, np.int32),
           "core": np.zeros((bsz, npoints), bool), "attempt": np.zeros(bsz, np.int32), "valid": np.zeros(bsz, bool),
           "context": np.zeros(bsz, np.int64)}
    for b, s in enumerate(np.asarray(crop_scene, np.int64)):
        if not 0 <= s < len(offsets) - 1:  # a scene index outside [0, S): an empty crop, attempt -1
            out["attempt"][b] = -1
            continue
        o0, o1 = int(offsets[s]), int(offsets[s + 1])
        pts, lab = xyz[o0:o1], label[o0:o1]
        att = crop_attempts(pts, lab, lo[s][2], hi[s][2], seed, b)
        a = choose(att)
        members, core = att[a]["members"], att[a]["core"]
        order = row_order(members, seed, b)[:npoints]
        rows, rcore = members[order], core[order]
        m = len(rows)
        ratio = unit(draw(seed, STREAM_RATIO, b, 0)) * max_dropout
        dropped = unit(draw(seed, STREAM_DROP, b, np.arange(m))) <= ratio
        keep = ~dropped
        keep[0] = True
        w = np.where(rcore, lw[lab[rows]], np.float32(0)).astype(np.float32)
        if dropped[0]:
            w[0] = 0
        rows, rcore, w = rows[keep], rcore[keep], w[keep]
        n = len(rows)
        p = pts[rows].astype(np.float64)
        if rotate:
            theta = unit(draw(seed, STREAM_ANGLE, b, 0)) * 2 * np.pi
            c, sn = np.cos(theta), np.sin(theta)
            p = np.stack([p[:, 0] * c - p[:, 1] * sn, p[:, 0] * sn + p[:, 1] * c, p[:, 2]], 1)
        out["xyz64"][b, :n] = p
        out["xyz"][b, :n] = p.astype(np.float32)
        out["label"][b, :n] = lab[rows]
        out["weight"][b, :n] = w
        out["lengths"][b] = n
        out["point_idx"][b, :n] = o0 + rows
        out["core"][b, :n] = rcore
        out["attempt"][b] = a
        out["valid"][b] = att[a]["valid"]
        out["context"][b] = len(members)
    return out
