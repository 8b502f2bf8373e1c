"""CPU tests of per-cloud lengths for kNN: the contract's restatement (tests/knn_ragged_oracle.py) on hand-made clouds —
lengths 1, k - 1, k and k + 1, ties across the truncation point, NaN in the padding — and the new entries' argument
checks that need no device."""
import ctypes
import inspect

import numpy as np
import pytest
import torch

from knn_ragged_oracle import oracle_knn_ragged, oracle_sample_knn_ragged
from pointnet2_b200 import _lib, pointnet_util, sa_layer, tf_grouping

EINVAL = 1  # cudaErrorInvalidValue


def line_cloud(n):
    """points 0.5 * j on the x axis: from a query at x = -1 the distances grow with the index, with no tie"""
    x = np.zeros((n, 3), np.float32)
    x[:, 0] = 0.5 * np.arange(n, dtype=np.float32)
    return x


def sorted_row(cloud, q, kk):
    d = np.sum((cloud - q) ** 2, axis=1).astype(np.float32)
    order = np.lexsort((np.arange(len(d)), d))[:kk]
    return d[order], order.astype(np.int32)


@pytest.mark.parametrize("k", [1, 5, 32, 33])
@pytest.mark.parametrize("delta", [None, -1, 0, 1])  # len = 1, k - 1, k, k + 1
def test_short_and_long_clouds(k, delta):
    n = 40
    ln = 1 if delta is None else k + delta
    if ln < 1 or ln > n:
        pytest.skip("length outside the cloud")
    x = line_cloud(n)[None]
    q = np.array([[[-1.0, 0.0, 0.0], [7.25, 0.0, 0.0]]], np.float32)
    val, idx = oracle_knn_ragged(k, x, q, lengths=[ln])
    for j in range(2):
        kk = min(k, ln)
        wv, wi = sorted_row(x[0, :ln], q[0, j], kk)
        assert np.array_equal(idx[0, j, :kk], wi) and np.array_equal(val[0, j, :kk], wv)
        # the filler: column 0 again
        assert np.all(idx[0, j, kk:] == idx[0, j, 0]) and np.all(val[0, j, kk:] == val[0, j, 0])
        assert idx[0, j].max() < ln


def test_length_one_is_the_first_point_everywhere():
    x = line_cloud(8)[None]
    q = np.array([[[3.0, 1.0, 0.0]]], np.float32)
    val, idx = oracle_knn_ragged(4, x, q, lengths=[1])
    assert np.all(idx == 0) and np.all(val == np.float32(10.0))


def test_ties_across_the_truncation_point():
    """points l - 1 and l (and l + 1) at one distance from the query: only the one inside the cloud can be picked"""
    k, n, ln = 4, 16, 6
    x = line_cloud(n)
    q = np.array([10.0, 0.0, 0.0], np.float32)
    x[ln - 1] = x[ln] = x[ln + 1] = (10.0, 3.0, 0.0)  # distance 9, like x = 7 and x = 13 on the line
    x[0] = (7.0, 0.0, 0.0)
    val, idx = oracle_knn_ragged(k, x[None], q[None, None], lengths=[ln])
    assert ln not in idx[0, 0] and ln + 1 not in idx[0, 0]
    assert np.array_equal(idx[0, 0], [0, ln - 1, 4, 3])
    assert np.array_equal(val[0, 0], np.array([9, 9, 64, 72.25], np.float32))
    _, full_i = oracle_knn_ragged(k, x[None], q[None, None])
    assert ln in full_i[0, 0]  # the whole cloud would take a padding point


def test_padding_never_changes_a_result():
    rs = np.random.RandomState(3)
    b, n, m, k = 3, 50, 7, 9
    x = rs.uniform(-1, 1, (b, n, 3)).astype(np.float32)
    q = rs.uniform(-1, 1, (b, m, 3)).astype(np.float32)
    lens, qlens = [1, 8, 31], [7, 1, 4]
    want = oracle_knn_ragged(k, x, q, lens, qlens)
    for i, (ln, ql) in enumerate(zip(lens, qlens)):
        x[i, ln::2] = np.nan
        x[i, ln + 1::2] = np.inf
        q[i, ql:] = np.nan
    got = oracle_knn_ragged(k, x, q, lens, qlens)
    assert np.array_equal(got[1], want[1]) and np.array_equal(got[0].view(np.int32), want[0].view(np.int32))
    assert np.all(got[1][1, 1:] == 0) and np.all(np.isinf(got[0][1, 1:]))  # query padding: idx 0 / val +inf
    assert np.all(got[1][0] == 0)  # a one-point cloud


def test_out_of_range_lengths_are_clamped():
    rs = np.random.RandomState(5)
    x = rs.uniform(-1, 1, (2, 20, 3)).astype(np.float32)
    q = rs.uniform(-1, 1, (2, 4, 3)).astype(np.float32)
    a = oracle_knn_ragged(6, x, q, [0, 99], [-3, 50])
    bb = oracle_knn_ragged(6, x, q, [1, 20], [1, 4])
    assert np.array_equal(a[1], bb[1])


def test_layer_oracle_is_the_chain_on_each_truncated_cloud():
    rs = np.random.RandomState(7)
    x = rs.uniform(-1, 1, (2, 40, 3)).astype(np.float32)
    fi, nx, idx, dist, g = oracle_sample_knn_ragged(8, 12, x, [40, 5], center=True)
    assert fi[1].max() < 5 and idx[1].max() < 5
    assert np.all(idx[1, :, 5:] == idx[1, :, :1]) and np.all(dist[1, :, 5:] == dist[1, :, :1])
    assert np.array_equal(g[1, :, 5:], np.repeat(g[1, :, :1], 7, axis=1))


def test_lengths_are_keywords_of_the_kNN_calls():
    for fn, names in ((tf_grouping.knn_point, ("lengths", "query_lengths")), (sa_layer.sample_knn, ("lengths",))):
        params = inspect.signature(fn).parameters
        for name in names:
            assert params[name].kind == inspect.Parameter.KEYWORD_ONLY and params[name].default is None


def test_new_entries_are_exported():
    lib = _lib.load()
    for s in ("pn2_knn_point_ragged", "pn2_sa_knn_layer_device_ragged"):
        assert s in _lib.EXPORTED_SYMBOLS and hasattr(lib, s)


def test_knn_entry_refuses_bad_arguments_before_touching_a_device():
    lib = _lib.load()
    p = ctypes.c_void_p(256)  # never dereferenced: every call below is refused on the host
    for b, n, m, k in ((2, 64, 8, 0), (2, 64, 8, 129), (2, 16, 8, 17), (-1, 64, 8, 4), (2, 0, 8, 1), (2, 64, -1, 4), (70000, 64, 8, 4)):
        assert lib.pn2_knn_point_ragged(b, n, m, k, p, p, p, p, p, p, None) == EINVAL, (b, n, m, k)
    assert lib.pn2_knn_point_ragged(2, 64, 8, 4, None, p, p, p, p, p, None) == EINVAL
    assert lib.pn2_knn_point_ragged(0, 64, 8, 4, None, None, None, None, None, None, None) == 0
    assert lib.pn2_sa_knn_layer_device_ragged(2, 16, 8, 17, p, p, p, p, p, None, None, 1, None, 0, None) == EINVAL
    assert lib.pn2_sa_knn_layer_device_ragged(2, 64, 8, 4, p, p, None, p, p, None, None, 1, None, 0, None) == EINVAL
    assert lib.pn2_sa_knn_layer_device_ragged(0, 64, 8, 4, None, None, None, None, None, None, None, 1, None, 0, None) == 0


def test_sample_knn_checks_its_arguments_before_the_lengths():
    x = torch.zeros(2, 16, 3)
    with pytest.raises(ValueError):
        sa_layer.sample_knn(0, 4, x, lengths=[16, 8])
    with pytest.raises(ValueError):
        sa_layer.sample_knn(4, 0, x, lengths=[16, 8])


def test_group_all_still_refuses_lengths_with_knn():
    x = torch.zeros(2, 16, 3)
    with pytest.raises(ValueError, match="group_all"):
        pointnet_util.pointnet_sa_module(x, None, None, None, None, group_all=True, knn=True, lengths=[16, 8])
