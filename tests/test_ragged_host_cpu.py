"""CPU tests of the host-buffer layer on packed variable-size clouds (pn2_sa_layer_host_ragged): it is exported, its
workspace grows with the capacity, it refuses bad lengths and arguments before it touches a device, and the Python
packing refuses malformed clouds before anything is written."""
import ctypes
import inspect

import numpy as np
import pytest

from pointnet2_b200 import _lib, host, sa_layer

EINVAL = 1  # cudaErrorInvalidValue
EMISALIGNED = 716  # cudaErrorMisalignedAddress
NEW = ("pn2_sa_layer_host_ragged_workspace_bytes", "pn2_sa_layer_host_ragged")


def test_new_symbols_are_exported():
    lib = _lib.load()
    for s in NEW:
        assert s in _lib.EXPORTED_SYMBOLS
        assert hasattr(lib, s)


def test_workspace_is_monotone_in_the_capacity():
    lib = _lib.load()
    # across the ball-query grid's 2048 floor, the global-scratch FPS plan beyond 425 984 points and the grid's 2^20 cap
    ns = [1, 2, 3, 100, 1024, 2047, 2048, 2049, 4096, 9700, 9701, 16384, 262144, 425984, 425985, 600000, 1 << 20,
          (1 << 20) + 1, 1 << 21]
    for b, m, s in ((1, 1, 1), (32, 1024, 32), (40, 64, 8)):
        ws = [int(lib.pn2_sa_layer_host_ragged_workspace_bytes(b, n, m, s)) for n in ns]
        assert all(w > 0 and w % 256 == 0 for w in ws)
        assert ws == sorted(ws), (b, m, s, ws)
        for n, w in zip(ns, ws):
            # the staging area and the padded batch at the capacity, the lengths, the outputs
            assert w >= 4 * b + 2 * 12 * b * n + 4 * b * m * (3 + 2 + 4 * s), (b, n)
            assert w >= int(lib.pn2_sa_layer_workspace_bytes(b, n, m, s)) + 12 * b * n, (b, n)
    for bad in ((0, 16, 4, 4), (2, 0, 4, 4), (2, 16, 0, 4), (2, 16, 4, 0), (-1, 16, 4, 4)):
        assert lib.pn2_sa_layer_host_ragged_workspace_bytes(*bad) == 0


def _call(lib, b, n, lengths, xyz=True, ws_bytes=None, ws_ptr=256, m=8, s=4, radius=0.2):
    """The entry with host arrays for xyz / lengths and a fake device workspace pointer that a refused call never
    dereferences.  ws_bytes defaults to the full size."""
    lens = None if lengths is None else np.ascontiguousarray(lengths, dtype=np.int32)
    rows = int(lens.sum()) if lens is not None and lens.size else 1
    pts = np.zeros((max(rows, 1), 3), np.float32) if xyz else None
    if ws_bytes is None:
        ws_bytes = int(lib.pn2_sa_layer_host_ragged_workspace_bytes(max(b, 1), max(n, 1), m, s))
    p = lambda a: None if a is None else a.ctypes.data_as(ctypes.c_void_p)  # noqa: E731
    return lib.pn2_sa_layer_host_ragged(b, n, m, radius, s, p(pts), p(lens), None, None, None, None,
                                        ctypes.c_void_p(ws_ptr) if ws_ptr else None, ws_bytes, None)


def test_entry_refuses_bad_lengths_and_arguments_before_touching_a_device():
    lib = _lib.load()
    b, n = 3, 100
    for lengths in ([0, 5, 5], [5, 101, 5], [5, 5, -1], [100, 100, 1000000]):
        assert _call(lib, b, n, lengths) == EINVAL, lengths
    assert _call(lib, b, n, [5, 5, 5], xyz=False) == EINVAL
    assert _call(lib, b, n, None) == EINVAL
    assert _call(lib, b, n, [5, 5, 5], ws_ptr=0) == EINVAL
    full = int(lib.pn2_sa_layer_host_ragged_workspace_bytes(b, n, 8, 4))
    assert _call(lib, b, n, [5, 5, 5], ws_bytes=full - 1) == EINVAL
    assert _call(lib, b, n, [5, 5, 5], ws_ptr=256 + 4) == EMISALIGNED
    for bb in (0, -1):
        assert _call(lib, bb, n, [5, 5, 5]) == EINVAL
    assert _call(lib, b, 0, [5, 5, 5]) == EINVAL
    assert _call(lib, b, n, [5, 5, 5], m=0) == EINVAL
    assert _call(lib, b, n, [5, 5, 5], s=0) == EINVAL
    assert _call(lib, b, n, [5, 5, 5], radius=0.0) == EINVAL
    assert _call(lib, b, n, [5, 5, 5], radius=float("nan")) == EINVAL


def _buffers(b, n):
    return np.full((b * n, 3), -7.0, np.float32), np.zeros(b, np.int32)


def test_pack_clouds_writes_the_clouds_back_to_back():
    rng = np.random.default_rng(0)
    lens = [5, 1, 8, 3]
    clouds = [rng.random((l, 3), dtype=np.float32) for l in lens]
    xyz, lengths = _buffers(4, 8)
    assert host.pack_clouds(clouds, 8, xyz, lengths) == sum(lens)
    assert lengths.tolist() == lens
    np.testing.assert_array_equal(xyz[:sum(lens)], np.concatenate(clouds))
    assert (xyz[sum(lens):] == -7.0).all()  # the rest of the capacity is not touched


def test_pack_clouds_refuses_malformed_batches_before_writing():
    b, n = 3, 8
    ok = [np.zeros((4, 3), np.float32) for _ in range(b)]
    cases = [
        (ok[:2], ValueError),                                                          # a list of the wrong length
        (ok + [ok[0]], ValueError),
        (np.zeros((b, 4, 3), np.float32), ValueError),                                 # a dense array is not a list of clouds
        (ok[:2] + [np.zeros((4, 3), np.float64)], TypeError),                          # not float32
        (ok[:2] + [[[0.0, 0.0, 0.0]]], TypeError),                                     # not an array
        (ok[:2] + [np.zeros((4, 2), np.float32)], ValueError),                         # not (., 3)
        (ok[:2] + [np.zeros((4, 3, 1), np.float32)], ValueError),
        (ok[:2] + [np.zeros(12, np.float32)], ValueError),
        (ok[:2] + [np.zeros((n + 1, 3), np.float32)], ValueError),                     # longer than the capacity
        (ok[:2] + [np.zeros((0, 3), np.float32)], ValueError),                         # empty
    ]
    for clouds, err in cases:
        xyz, lengths = _buffers(b, n)
        with pytest.raises(err):
            host.pack_clouds(clouds, n, xyz, lengths)
        assert (xyz == -7.0).all() and not lengths.any()


def test_check_lengths():
    assert host.check_lengths([1, 8, 3], 3, 8).tolist() == [1, 8, 3]
    for bad in ([0, 1, 1], [1, 9, 1], [1, 1], [[1, 1, 1]], [1.0, 2.0, 3.0], np.array([-1, 2, 3])):
        with pytest.raises(ValueError):
            host.check_lengths(bad, 3, 8)


def test_ragged_is_an_opt_in_keyword():
    for cls in (host.SetAbstractionHost, host.SetAbstractionPipeline):
        assert inspect.signature(cls.__init__).parameters["ragged"].default is False, cls.__name__
    assert inspect.signature(sa_layer.SetAbstractionDevice.submit).parameters["lengths"].default is None
    assert inspect.signature(host.SetAbstractionPipeline.submit).parameters["lengths"].default is None
