"""CPU tests of the kNN set-abstraction layer's C entry (pn2_sa_knn_layer_device): it is exported, its capacity test
and workspace size are plain arithmetic, and it refuses bad arguments before it touches a device.  Variable-size
clouds stay refused with kNN grouping."""
import ctypes

import pytest
import torch

from pointnet2_b200 import _lib, pointnet_util, sa_layer

EINVAL = 1  # cudaErrorInvalidValue
NEW = ("pn2_sa_knn_layer_fits", "pn2_sa_knn_layer_workspace_bytes", "pn2_sa_knn_layer_device", "pn2_set_sa_knn_path")


def test_new_symbols_are_exported():
    lib = _lib.load()
    for s in NEW:
        assert s in _lib.EXPORTED_SYMBOLS
        assert hasattr(lib, s)


def test_fits_is_the_shared_memory_budget():
    lib = _lib.load()
    for n, k in ((4096, 32), (4096, 64), (8192, 32), (8192, 64), (1, 1), (64, 64), (16000, 1), (16000, 8)):
        assert lib.pn2_sa_knn_layer_fits(n, k) == 1, (n, k)
    # k out of range, k > n, k above the overlapped layer's 64, or a cloud that leaves too little room for the W buffers
    for n, k in ((4096, 0), (4096, -1), (4096, 129), (10, 11), (0, 1), (20000, 8), (17000, 32), (17000, 16), (4096, 65), (4096, 128)):
        assert lib.pn2_sa_knn_layer_fits(n, k) == 0, (n, k)


def test_workspace_follows_the_path():
    lib = _lib.load()
    b, n, m, k = 4, 4096, 1024, 32
    try:
        lib.pn2_set_sa_knn_path(2)  # sequential: knn_point's distances when dist is NULL
        assert lib.pn2_sa_knn_layer_workspace_bytes(b, n, m, k) >= 4 * b * m * k
        lib.pn2_set_sa_knn_path(1)  # overlapped: none
        assert lib.pn2_sa_knn_layer_workspace_bytes(b, n, m, k) == 0
        lib.pn2_set_sa_knn_path(1)  # k > 64 cannot overlap
        assert lib.pn2_sa_knn_layer_workspace_bytes(b, n, m, 128) >= 4 * b * m * 128
    finally:
        lib.pn2_set_sa_knn_path(0)
    assert lib.pn2_sa_knn_layer_workspace_bytes(0, n, m, k) == 0
    assert lib.pn2_sa_knn_layer_workspace_bytes(b, n, m, 0) == 0


def _call(lib, b, n, m, k, xyz, fps_idx, new_xyz, idx):
    return lib.pn2_sa_knn_layer_device(b, n, m, k, xyz, fps_idx, new_xyz, idx, None, None, 1, None, 0, None)


def test_entry_refuses_bad_arguments_before_touching_a_device():
    lib = _lib.load()
    p = ctypes.c_void_p(256)  # never dereferenced: every call below is refused on the host
    for k in (0, -3, 129, 65):
        n = 64 if k == 65 else 4096  # 65 > n
        assert _call(lib, 2, n, 16, k, p, p, p, p) == EINVAL, k
    assert _call(lib, -1, 4096, 16, 8, p, p, p, p) == EINVAL
    assert _call(lib, 2, 0, 16, 8, p, p, p, p) == EINVAL
    assert _call(lib, 2, 4096, -1, 8, p, p, p, p) == EINVAL
    for i in range(4):  # xyz, fps_idx, new_xyz, idx are required
        ptrs = [p] * 4
        ptrs[i] = None
        assert _call(lib, 2, 4096, 16, 8, *ptrs) == EINVAL, i
    assert _call(lib, 0, 4096, 16, 8, None, None, None, None) == 0  # nothing to do
    assert _call(lib, 2, 4096, 0, 8, None, None, None, None) == 0


def test_sample_knn_validates_its_arguments():
    x = torch.zeros(2, 16, 3)
    with pytest.raises(ValueError):
        sa_layer.sample_knn(0, 4, x)
    with pytest.raises(ValueError):
        sa_layer.sample_knn(4, 0, x)


def test_lengths_with_knn_are_still_refused():
    x = torch.zeros(2, 16, 3)
    with pytest.raises(ValueError, match="knn"):
        pointnet_util.sample_and_group(4, 0.2, 4, x, None, knn=True, lengths=[16, 8])
    with pytest.raises(ValueError, match="knn"):
        pointnet_util.sample_and_group(4, 0.2, 4, x, None, knn=True, fused=False, lengths=[16, 8])
