"""CPU tests of the multi-scale host-buffer layer (pn2_sa_layer_msg_host, pn2_sa_layer_msg_host_ragged): the entries are
declared, exported and in the ctypes table, their workspace covers every output and the device layer's scratch, they
refuse every bad argument before they touch a device, and the Python classes refuse malformed scale lists, cloud lists
and lengths before anything is launched."""
import collections
import ctypes

import numpy as np
import pytest
import torch

from pointnet2_b200 import _lib, host
from test_abi import declared_symbols

EINVAL = 1  # cudaErrorInvalidValue
EMISALIGNED = 716  # cudaErrorMisalignedAddress
NEW = ("pn2_sa_layer_msg_host_workspace_bytes", "pn2_sa_layer_msg_host", "pn2_sa_layer_msg_host_ragged_workspace_bytes",
       "pn2_sa_layer_msg_host_ragged")


def ints(v):
    return (ctypes.c_int * len(v))(*v)


def ws_msg(lib, b, n, m, nsamples, ragged):
    fn = lib.pn2_sa_layer_msg_host_ragged_workspace_bytes if ragged else lib.pn2_sa_layer_msg_host_workspace_bytes
    return int(fn(b, n, m, len(nsamples), ints(nsamples)))


def ws_single(lib, b, n, m, s, ragged):
    fn = lib.pn2_sa_layer_host_ragged_workspace_bytes if ragged else lib.pn2_sa_layer_workspace_bytes
    return int(fn(b, n, m, s))


def test_new_symbols_are_declared_exported_and_typed():
    lib = _lib.load()
    declared = declared_symbols()
    for s in NEW:
        assert s in declared
        assert s in _lib.EXPORTED_SYMBOLS
        assert hasattr(lib, s)


# across the ball-query grid's 2048 floor, the sequential layer beyond 9700, the global-scratch FPS plan beyond
# 425 984 points and the grid's 2^20 cap
NS = [1, 2, 100, 1024, 2047, 2048, 2049, 4096, 9700, 9701, 16384, 262144, 425984, 425985, 600000, 1 << 20, (1 << 20) + 1]
SHAPES = [(1, 1, [1]), (32, 512, [16, 32, 128]), (40, 64, [8, 8]), (3, 100, [5, 1, 64, 2, 3, 4, 7, 9, 11, 13, 17, 19, 23, 29, 31, 37])]


@pytest.mark.parametrize("ragged", [False, True])
def test_workspace_covers_every_output_and_the_single_scale_layer(ragged):
    lib = _lib.load()
    for b, m, nsamples in SHAPES:
        for n in NS:
            w = ws_msg(lib, b, n, m, nsamples, ragged)
            assert w > 0 and w % 256 == 0, (b, n, m, nsamples)
            outputs = 4 * b * m * (3 + 1) + sum(4 * b * m * (s + 1 + 3 * s) for s in nsamples)  # new_xyz, fps_idx; per scale
            inputs = 4 * b + 2 * 12 * b * n if ragged else 12 * b * n  # the lengths, the staging area, the padded batch
            assert w >= outputs + inputs, (b, n, m, nsamples)
            assert w >= ws_single(lib, b, n, m, max(nsamples), ragged), (b, n, m, nsamples)
            # one scale is the single-scale layout
            assert ws_msg(lib, b, n, m, nsamples[:1], ragged) == ws_single(lib, b, n, m, nsamples[0], ragged)


def test_ragged_workspace_never_shrinks_as_the_capacity_grows():
    lib = _lib.load()
    for b, m, nsamples in SHAPES:
        ws = [ws_msg(lib, b, n, m, nsamples, True) for n in NS]
        assert ws == sorted(ws), (b, m, nsamples, ws)


@pytest.mark.parametrize("ragged", [False, True])
def test_workspace_is_zero_for_invalid_arguments(ragged):
    lib = _lib.load()
    fn = lib.pn2_sa_layer_msg_host_ragged_workspace_bytes if ragged else lib.pn2_sa_layer_msg_host_workspace_bytes
    ok = ints([16, 32])
    for b, n, m in ((0, 16, 4), (2, 0, 4), (2, 16, 0), (-1, 16, 4)):
        assert fn(b, n, m, 2, ok) == 0
    assert fn(2, 16, 4, 0, ok) == 0
    assert fn(2, 16, 4, 17, ints([4] * 17)) == 0
    assert fn(2, 16, 4, -1, ok) == 0
    assert fn(2, 16, 4, 2, None) == 0
    assert fn(2, 16, 4, 2, ints([16, 0])) == 0
    assert fn(2, 16, 4, 2, ints([-3, 16])) == 0
    assert fn(2, 16, 4, 16, ints([4] * 16)) > 0


def _call(lib, ragged, b=3, n=100, m=8, radii=(0.1, 0.2, 0.4), nsamples=(4, 8, 16), lengths=(5, 5, 5), nscales=None,
          ws_bytes=None, ws_ptr=256, drop=None, null_idx=None, null_cnt=None):
    """One call of the entry with host arrays and a fake device workspace pointer that a refused call never
    dereferences.  `drop` names one required pointer to pass as NULL; null_idx / null_cnt the scale whose h_idx /
    h_pts_cnt entry is NULL.  ws_bytes defaults to the full size."""
    k = len(nsamples) if nscales is None else nscales
    lens = np.ascontiguousarray(lengths, dtype=np.int32)
    rows = int(lens.sum()) if ragged else b * n
    xyz = np.zeros((max(rows, 1), 3), np.float32)
    new_xyz = np.zeros((max(b * m, 1), 3), np.float32)
    keep = []

    def buf(nbytes):
        a = np.zeros(max(nbytes, 4) // 4, np.int32)
        keep.append(a)
        return a.ctypes.data

    idx = (ctypes.c_void_p * len(nsamples))(*[None if j == null_idx else buf(4 * b * m * s) for j, s in enumerate(nsamples)])
    cnt = (ctypes.c_void_p * len(nsamples))(*[None if j == null_cnt else buf(4 * b * m) for j in range(len(nsamples))])
    c_radii = (ctypes.c_float * len(radii))(*radii)
    c_ns = ints(list(nsamples))
    if ws_bytes is None:
        ws_bytes = ws_msg(lib, max(b, 1), max(n, 1), max(m, 1), [max(s, 1) for s in nsamples], ragged)
    p = lambda a: a.ctypes.data_as(ctypes.c_void_p)  # noqa: E731
    args = dict(radii=c_radii, nsamples=c_ns, xyz=p(xyz), lengths=p(lens), new_xyz=p(new_xyz), idx=idx, cnt=cnt,
                ws=ctypes.c_void_p(ws_ptr))
    if drop:
        args[drop] = None
    head = (b, n, m, k, args["radii"], args["nsamples"], args["xyz"])
    tail = (args["new_xyz"], args["idx"], args["cnt"], None, args["ws"], ws_bytes, None)
    if ragged:
        return lib.pn2_sa_layer_msg_host_ragged(*head, args["lengths"], *tail)
    return lib.pn2_sa_layer_msg_host(*head, *tail)


@pytest.mark.parametrize("ragged", [False, True])
def test_entry_refuses_bad_arguments_before_touching_a_device(ragged):
    """Every refusal returns its own code.  On a machine without a GPU any CUDA call would return another error, so
    the codes show that the checks run before the first one."""
    lib = _lib.load()
    bad = [dict(b=0), dict(b=-1), dict(n=0), dict(m=0), dict(nscales=0), dict(nscales=-2),
           dict(nscales=17, radii=[0.1] * 17, nsamples=[4] * 17),
           dict(radii=(0.1, 0.0, 0.4)), dict(radii=(0.1, 0.2, -1.0)), dict(radii=(float("nan"), 0.2, 0.4)),
           dict(nsamples=(4, 0, 16)), dict(nsamples=(4, 8, -16)),
           dict(drop="radii"), dict(drop="nsamples"), dict(drop="xyz"), dict(drop="new_xyz"), dict(drop="idx"),
           dict(drop="cnt"), dict(drop="ws"), dict(null_idx=2), dict(null_cnt=0),
           dict(ws_bytes=ws_msg(lib, 3, 100, 8, [4, 8, 16], ragged) - 1)]
    if ragged:
        bad += [dict(drop="lengths"), dict(lengths=(0, 5, 5)), dict(lengths=(5, 101, 5)), dict(lengths=(5, 5, -1)),
                dict(lengths=(100, 100, 1000000))]
    for kw in bad:
        assert _call(lib, ragged, **kw) == EINVAL, kw
    assert _call(lib, ragged, ws_ptr=256 + 4) == EMISALIGNED


def test_scale_lists():
    assert host.layer_scales(0.2, 32) is None
    assert host.layer_scales(0.2, 32, want_grouped=False) is None
    assert host.layer_scales([0.1, 0.2], (16, 32)) == ((0.1, 0.2), (16, 32), (True, True))
    assert host.layer_scales(np.array([0.1, 0.2]), [16, 32], want_grouped=False)[2] == (False, False)
    assert host.layer_scales([0.1, 0.2, 0.4], [16, 32, 128], [True, False, True])[2] == (True, False, True)
    assert host.layer_scales([0.1], [16]) == ((0.1,), (16,), (True,))  # one scale in a list is the multi-scale form
    bad = [([], []), ([0.1, 0.2], [16]), ([0.1], [16, 32]), (0.1, [16]), ([0.1], 16), ([0.1] * 17, [4] * 17),
           ([0.1, 0.0], [16, 32]), ([0.1, float("nan")], [16, 32]), ([0.1, 0.2], [16, 0])]
    for radius, nsample in bad:
        with pytest.raises(ValueError):
            host.layer_scales(radius, nsample)
    for want in ([True], [True, False, True], []):
        with pytest.raises(ValueError):
            host.layer_scales([0.1, 0.2], [16, 32], want)
    with pytest.raises(ValueError):
        host.layer_scales(0.1, 16, [True])  # per-scale flags need scale lists


@pytest.mark.parametrize("cls", [host.SetAbstractionHost, host.SetAbstractionPipeline])
def test_classes_refuse_bad_scale_lists_before_touching_a_device(cls):
    for radius, nsample, want in (([0.1, 0.2], [16], True), ([], [], True), ([0.1, 0.2], [16, 32], [True])):
        with pytest.raises(ValueError):
            cls(2, 64, 16, radius, nsample, want_grouped=want)


def _offline_pipeline(ragged, b=3, n=8):
    """A SetAbstractionPipeline of multi-scale slots whose buffers are ordinary CPU tensors.  It is never launched: it
    only reaches the checks that submit and run make before anything is enqueued."""
    slot = object.__new__(host.SetAbstractionHost)
    slot.b, slot.n, slot.m, slot.ragged, slot.msg = b, n, 4, ragged, True
    slot.radii, slot.nsamples = (0.1, 0.2), (4, 8)
    slot.h_xyz = torch.full((b * n, 3) if ragged else (b, n, 3), -7.0)
    slot.h_lengths = torch.zeros(b, dtype=torch.int32) if ragged else None
    pipe = object.__new__(host.SetAbstractionPipeline)
    pipe.ragged, pipe.slots, pipe._inflight, pipe._next = ragged, [slot], collections.deque(), 0
    return pipe, slot


def test_submit_and_run_refuse_malformed_input_before_launching():
    ok = [np.zeros((4, 3), np.float32) for _ in range(3)]
    pipe, slot = _offline_pipeline(ragged=False)
    with pytest.raises(ValueError):
        pipe.submit(lengths=[4, 4, 4])  # lengths need ragged=True
    with pytest.raises(ValueError):
        pipe.submit(np.zeros((3, 7, 3), np.float32))  # not (b, n, 3)
    with pytest.raises(ValueError):
        slot.run(np.zeros((3, 8, 2), np.float32))
    pipe, slot = _offline_pipeline(ragged=True)
    with pytest.raises(ValueError):
        pipe.submit()  # a ragged submit takes clouds or lengths
    with pytest.raises(ValueError):
        pipe.submit(ok, lengths=[4, 4, 4])
    with pytest.raises(ValueError):
        pipe.submit(lengths=[4, 9, 4])  # longer than the capacity
    for clouds, err in ((ok[:2], ValueError), (np.zeros((3, 4, 3), np.float32), ValueError),
                        (ok[:2] + [np.zeros((4, 3), np.float64)], TypeError), (ok[:2] + [np.zeros((9, 3), np.float32)], ValueError),
                        (ok[:2] + [np.zeros((0, 3), np.float32)], ValueError)):
        for call in (pipe.submit, slot.run):
            with pytest.raises(err):
                call(clouds)
    assert (slot.h_xyz == -7.0).all() and not slot.h_lengths.any() and not pipe._inflight

