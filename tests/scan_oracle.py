"""Plain numpy restatement of the virtual scans (pointnet2_b200.scene.sample_virtual_scans, DESIGN.md §6.12) for the
tests and tools/virtual_scan_bench.py (test infrastructure only).

view          the camera location and the (az, el) of the 30,000 rays of one view
scan          one scan: the visible points (virtual_scan's smpidx), the near count and the smallest decision margin
oracle_scans  every output field of sample_virtual_scans, plus each entry's smpidx, near count and margin

The nearest ray is found with scipy's cKDTree (k = 2) and both candidates' distances are then recomputed with the
definition's expression, so the margin (the distance to the 0.01 threshold, the gap to the second-nearest ray, and the
gap between a ray's nearest and next range) says how far every decision is from flipping.
"""
from __future__ import annotations

import numpy as np
from scipy.spatial import cKDTree

from crop_oracle import draw, unit

STREAM_AZIMUTH, STREAM_TILT, STREAM_DISTANCE, STREAM_KEY = 1, 2, 3, 4
NEAR, MIN_NEAR = 0.01, 100


def cart2sph(v: np.ndarray):
    """(az, el, r) of (N, 3) float64 vectors: atan2(y, x), atan2(z, sqrt(x^2 + y^2)), sqrt((x^2 + y^2) + z^2)."""
    xy = v[:, 0] * v[:, 0] + v[:, 1] * v[:, 1]
    return np.arctan2(v[:, 1], v[:, 0]), np.arctan2(v[:, 2], np.sqrt(xy)), np.sqrt(xy + v[:, 2] * v[:, 2])


def view_draws(seed: int, b: int):
    """u1, u2, u3 of a random view of entry b."""
    return [float(unit(draw(seed, s, b, 0))) for s in (STREAM_AZIMUTH, STREAM_TILT, STREAM_DISTANCE)]


def _normalised(v):
    return v / np.sqrt((v[0] * v[0] + v[1] * v[1]) + v[2] * v[2])


def view(mean, mode: int, draws=None):
    """(camera (3,), rays (30000, 2) as (az, el)) of view ``mode`` from a scene of float64 mean ``mean``; a random view
    (mode -1) takes its three uniform draws from ``draws``."""
    cam = np.array(mean, np.float64).copy()
    cam[2] = 1.5
    if mode == -1:
        u1, u2, u3 = draws
        phi, theta = 2 * np.pi * u1, np.pi / 10 * (u2 - 0.75)
        cam[:2] -= (0.8 + 0.7 * u3) * np.array([np.cos(phi), np.sin(phi)])
    else:
        phi, theta = np.pi / 4 * mode, 0.0
        cam[:2] -= np.array([np.cos(phi), np.sin(phi)])
    ct = np.array([np.cos(theta) * np.cos(phi), np.cos(theta) * np.sin(phi), np.sin(theta)])
    hr = _normalised(np.cross(ct, np.array([0.0, 0.0, 1.0])))
    vt = _normalised(np.cross(hr, ct))
    xx, yy = np.meshgrid(np.linspace(-0.6, 0.6, 200), np.linspace(-0.45, 0.45, 150))
    rays = (xx.reshape(-1, 1) * hr + yy.reshape(-1, 1) * vt) + ct
    az, el, _ = cart2sph(rays)
    return cam, np.stack([az, el], 1)


def scan(pts: np.ndarray, mean, mode: int, draws=None) -> dict:
    """One scan of a scene (P, 3) (float32, widened to float64): smpidx (ascending scene-local indices; empty when
    fewer than 100 points are near), near (the near count), ray (each point's nearest ray), margin (the smallest
    decision margin over the points)."""
    cam, rays = view(mean, mode, draws)
    az, el, r = cart2sph(pts.astype(np.float64) - cam)
    q = np.stack([az, el], 1)
    _, ii = cKDTree(rays).query(q, k=2)
    d = np.sqrt((q[:, None, 0] - rays[ii, 0]) ** 2 + (q[:, None, 1] - rays[ii, 1]) ** 2)
    first = (d[:, 0] < d[:, 1]) | ((d[:, 0] == d[:, 1]) & (ii[:, 0] < ii[:, 1]))
    ray = np.where(first, ii[:, 0], ii[:, 1])
    dmin, dsec = np.where(first, d[:, 0], d[:, 1]), np.where(first, d[:, 1], d[:, 0])
    near = dmin < NEAR
    margins = [np.abs(dmin - NEAR).min(initial=np.inf), (dsec - dmin)[near].min(initial=np.inf)]
    n_near = int(near.sum())
    if n_near < MIN_NEAR:
        return {"smpidx": np.zeros(0, np.int64), "near": n_near, "ray": ray, "margin": min(margins)}
    zbuf = np.full(len(rays), np.inf)
    np.minimum.at(zbuf, ray[near], r[near])
    visible = near & (r == zbuf[ray])
    gap = r[near & ~visible] - zbuf[ray[near & ~visible]]
    margins.append(gap.min(initial=np.inf))
    return {"smpidx": np.nonzero(visible)[0], "near": n_near, "ray": ray, "margin": min(margins)}


def row_order(smpidx: np.ndarray, seed: int, b: int) -> np.ndarray:
    """Positions into ``smpidx`` in ascending (draw(seed, 4, b, j) >> 32, j) order."""
    key = draw(seed, STREAM_KEY, b, smpidx.astype(np.uint64)) >> np.uint64(32)
    return np.lexsort((smpidx, key))


def oracle_scans(xyz, label, offsets, mean, label_weights, scan_scene, scan_mode, seed: int, npoints=8192,
                 min_points=300) -> dict:
    """The fields of sample_virtual_scans as numpy arrays for a scene set given as host arrays (xyz (P, 3) float32,
    label (P,), offsets (S + 1,), mean (S, 3) float64, label_weights (C,) float32), plus per entry ``smpidx``, ``near``
    and ``margin`` (inf for an entry outside [0, S))."""
    xyz = np.asarray(xyz, np.float32)
    label = np.asarray(label)
    lw = np.asarray(label_weights, np.float32)
    s = len(offsets) - 1
    bsz = len(scan_scene)
    out = {"xyz": np.zeros((bsz, npoints, 3), np.float32), "label": np.zeros((bsz, npoints), np.int64),
           "weight": np.zeros((bsz, npoints), np.float32), "lengths": np.zeros(bsz, np.int32),
           "point_idx": np.full((bsz, npoints), -1, np.int32), "visible": np.full(bsz, -1, np.int32),
           "valid": np.zeros(bsz, bool), "smpidx": [None] * bsz, "near": np.zeros(bsz, np.int64),
           "margin": np.full(bsz, np.inf)}
    for b, (sc, mode) in enumerate(zip(np.asarray(scan_scene, np.int64), np.asarray(scan_mode, np.int64))):
        if not 0 <= sc < s:
            continue
        o0, o1 = int(offsets[sc]), int(offsets[sc + 1])
        mode = int(mode)
        got = scan(xyz[o0:o1], mean[sc], mode, view_draws(seed, b) if mode == -1 else None)
        smp = got["smpidx"]
        rows = smp[row_order(smp, seed, b)][:npoints]
        n = len(rows)
        valid = len(smp) >= min_points
        lab = label[o0:o1][rows]
        out["xyz"][b, :n] = xyz[o0:o1][rows]
        out["label"][b, :n] = lab
        out["weight"][b, :n] = lw[lab] if valid else 0
        out["lengths"][b] = n
        out["point_idx"][b, :n] = o0 + rows
        out["visible"][b] = len(smp)
        out["valid"][b] = valid
        out["smpidx"][b], out["near"][b], out["margin"][b] = smp, got["near"], got["margin"]
    return out
