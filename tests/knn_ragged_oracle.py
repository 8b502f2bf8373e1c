"""The ragged kNN contract (include/pn2_api.h, pn2_knn_point_ragged) restated on the C oracle, one cloud at a time.
No device is needed.

With len_i the data length of cloud i, k_i = min(k, len_i) and qlen_i its query length:
- columns [0, k_i) of query row j < qlen_i are oracle_knn_point(k_i, xyz1[i, :len_i], xyz2[i, j]);
- columns [k_i, k) repeat column 0 (val and idx);
- query rows j >= qlen_i are idx 0 / val +inf.
Lengths are clamped to [1, n] and [1, m], as the kernels clamp what they read."""
from __future__ import annotations

import numpy as np

from oracle import oracle as O


def clamp(lengths, i, n):
    return n if lengths is None else min(max(int(lengths[i]), 1), n)


def oracle_knn_ragged(k, xyz1, xyz2, lengths=None, query_lengths=None):
    """(val (b, m, k) float32, idx (b, m, k) int32) of knn_point(k, xyz1, xyz2, lengths=, query_lengths=)"""
    xyz1, xyz2 = np.asarray(xyz1, np.float32), np.asarray(xyz2, np.float32)
    b, n, _ = xyz1.shape
    m = xyz2.shape[1]
    val = np.full((b, m, k), np.inf, np.float32)
    idx = np.zeros((b, m, k), np.int32)
    for i in range(b):
        ln, ql = clamp(lengths, i, n), clamp(query_lengths, i, m)
        ki = min(k, ln)
        v, j = O.oracle_knn_point(ki, xyz1[i:i + 1, :ln], xyz2[i:i + 1, :ql])
        val[i, :ql, :ki], idx[i, :ql, :ki] = v[0], j[0]
        val[i, :ql, ki:], idx[i, :ql, ki:] = v[0, :, :1], j[0, :, :1]
    return val, idx


def oracle_sample_knn_ragged(npoint, k, xyz, lengths, center):
    """(fps_idx, new_xyz, idx, dist, grouped_xyz) of sample_knn(npoint, k, xyz, center, lengths=lengths): the chain
    oracle_fps -> oracle_gather_point -> oracle_knn_point -> oracle_group_point on each truncated cloud, plus the
    column-0 filler of a cloud shorter than k"""
    xyz = np.asarray(xyz, np.float32)
    b, n, _ = xyz.shape
    fi = np.zeros((b, npoint), np.int32)
    nx = np.zeros((b, npoint, 3), np.float32)
    idx = np.zeros((b, npoint, k), np.int32)
    dist = np.zeros((b, npoint, k), np.float32)
    g = np.zeros((b, npoint, k, 3), np.float32)
    for i in range(b):
        c = xyz[i:i + 1, :clamp(lengths, i, n)]
        fi[i] = O.oracle_fps(npoint, c)[0]
        nx[i] = O.oracle_gather_point(c, fi[i:i + 1])[0]
        v, j = oracle_knn_ragged(k, c, nx[i:i + 1])
        dist[i], idx[i] = v[0], j[0]
        gi = O.oracle_group_point(c, j)
        if center:
            with np.errstate(invalid="ignore"):  # inf - inf: NaN, as on the device
                gi = (gi - nx[i:i + 1, :, None, :]).astype(np.float32)
        g[i] = gi[0]
    return fi, nx, idx, dist, g
