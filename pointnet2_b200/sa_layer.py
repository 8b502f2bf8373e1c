"""The sampling+grouping half of a set-abstraction layer on device tensors.

``sample_group`` is the call ``sample_and_group`` makes when no gradient flows through ``xyz``
(reference utils/pointnet_util.py:40-46: farthest_point_sample -> gather_point -> query_ball_point
-> group_point(xyz) -> tile/sub): ONE C-ABI call, ``pn2_sa_layer_device``, whose ball query +
grouping run as a programmatically dependent grid on the SMs the sampling chain leaves idle.  The
results are bit-identical to the four separate ops.

``sample_knn`` is the kNN-grouping form (sample_and_group(..., knn=True)): FPS + gather_point + knn_point +
group_point(xyz) in ONE C-ABI call, ``pn2_sa_knn_layer_device``, whose kNN grouping overlaps the sampling chain in
the same way; bit-identical to the separate ops.

``ball_group`` is the same consumer kernel on its own (queries known up front): query_ball_point +
group_point(xyz) in one launch.

``SetAbstractionDevice`` keeps several independent batches in flight on private streams — one layer
occupies 2*b of the 132 SMs, so batches overlap (the device-resident twin of
``host.SetAbstractionPipeline``).
"""
from __future__ import annotations

import collections

import torch

from . import _lib
from ._tensor import device_lengths, on_device, ptr, require_cuda, same_device, stream_ptr


def _check_layer_args(npoint, radius, nsample, xyz):
    npoint, nsample, radius = int(npoint), int(nsample), float(radius)
    if npoint <= 0:
        raise ValueError("FarthestPointSample expects positive npoint")
    if not radius > 0:
        raise ValueError("QueryBallPoint expects positive radius")
    if nsample <= 0:
        raise ValueError("QueryBallPoint expects positive nsample")
    xyz = require_cuda(xyz, "xyz", torch.float32)
    if xyz.dim() != 3 or xyz.shape[2] != 3:
        raise ValueError(f"expected (batch_size, ndataset, 3) xyz shape, got {tuple(xyz.shape)}")
    if xyz.shape[1] <= 0:
        raise ValueError("FarthestPointSample expects at least one point per batch entry")
    return npoint, radius, nsample, xyz


def sample_group(npoint: int, radius: float, nsample: int, xyz: torch.Tensor, center: bool = True,
                 want_grouped: bool = True, *, lengths=None):
    """FPS + gather_point + query_ball_point + group_point(xyz) [- new_xyz] in one call.

    Returns (fps_idx (b,npoint) i32, new_xyz (b,npoint,3), idx (b,npoint,nsample) i32,
    pts_cnt (b,npoint) i32, grouped_xyz (b,npoint,nsample,3) or None).  ``center=True`` subtracts the
    centroid (the reference's ``grouped_xyz -= tile(new_xyz)``, :46); no gradients.
    ``lengths`` (b,) integers, optional: cloud i is ``xyz[i, :lengths[i]]``; each cloud then gets exactly what this
    call returns for it alone, and every index is below its length.  A device tensor is never read on the host, so
    the call can be captured in a CUDA graph and replayed with new lengths written into the same tensor.
    """
    npoint, radius, nsample, xyz = _check_layer_args(npoint, radius, nsample, xyz)
    b, n, _ = xyz.shape
    dev = xyz.device
    lens = device_lengths(lengths, b, n, dev, "sample_group")
    if torch.compiler.is_compiling():
        *res, grouped = torch.ops.pn2.sample_group(npoint, radius, nsample, xyz.detach(), bool(center), bool(want_grouped), lens)
        return (*res, grouped if want_grouped else None)
    return sample_group_launch(npoint, radius, nsample, xyz, center, want_grouped, lens)


def sample_group_launch(npoint: int, radius: float, nsample: int, xyz: torch.Tensor, center: bool, want_grouped: bool, lens):
    b, n, _ = xyz.shape
    dev = xyz.device
    fps_idx = torch.empty((b, npoint), dtype=torch.int32, device=dev)
    new_xyz = torch.empty((b, npoint, 3), dtype=torch.float32, device=dev)
    idx = torch.empty((b, npoint, nsample), dtype=torch.int32, device=dev)
    pts_cnt = torch.empty((b, npoint), dtype=torch.int32, device=dev)
    grouped = torch.empty((b, npoint, nsample, 3), dtype=torch.float32, device=dev) if want_grouped else None
    if b == 0:
        return fps_idx, new_xyz, idx, pts_cnt, grouped
    lib = _lib.load()
    with on_device(xyz):
        wsb = int(lib.pn2_sa_layer_device_workspace_bytes(b, n, npoint, nsample))
        ws = torch.empty(wsb, dtype=torch.uint8, device=dev) if wsb else None
        if lens is None:
            rc = lib.pn2_sa_layer_device(b, n, npoint, radius, nsample, ptr(xyz.detach()), ptr(fps_idx), ptr(new_xyz), ptr(idx),
                                         ptr(pts_cnt), ptr(grouped), 1 if center else 0, ptr(ws), wsb, stream_ptr(dev))
        else:
            rc = lib.pn2_sa_layer_device_ragged(b, n, npoint, radius, nsample, ptr(xyz.detach()), ptr(lens), ptr(fps_idx),
                                                ptr(new_xyz), ptr(idx), ptr(pts_cnt), ptr(grouped), 1 if center else 0, ptr(ws),
                                                wsb, stream_ptr(dev))
    _lib.check(rc, "pn2_sa_layer_device")
    return fps_idx, new_xyz, idx, pts_cnt, grouped


def sample_group_msg(npoint: int, radius_list, nsample_list, xyz: torch.Tensor, center: bool = True, want_grouped: bool = True,
                     *, lengths=None):
    """The multi-scale form (pointnet_sa_module_msg, utils/pointnet_util.py:156-196): ONE sampling pass, then a
    ball query + xyz grouping per scale — one C-ABI call, every scale's grouping grid overlapping the sampling chain.
    ``lengths``: as for sample_group.

    Returns (fps_idx, new_xyz, [idx_k], [pts_cnt_k], [grouped_xyz_k] or None)."""
    if len(radius_list) != len(nsample_list) or not len(radius_list):
        raise ValueError("radius_list and nsample_list must be non-empty and of equal length")
    npoint, _, _, xyz = _check_layer_args(npoint, radius_list[0], nsample_list[0], xyz)
    for r, s in zip(radius_list, nsample_list):
        _check_layer_args(npoint, r, s, xyz)
    b, n, _ = xyz.shape
    dev = xyz.device
    lens = device_lengths(lengths, b, n, dev, "sample_group_msg")
    if torch.compiler.is_compiling():
        fps_idx, new_xyz, idx, cnt, grouped = torch.ops.pn2.sample_group_msg(npoint, [float(r) for r in radius_list],
                                                                             [int(s) for s in nsample_list], xyz.detach(),
                                                                             bool(center), bool(want_grouped), lens)
        return fps_idx, new_xyz, idx, cnt, grouped if want_grouped else None
    return sample_group_msg_launch(npoint, radius_list, nsample_list, xyz, center, want_grouped, lens)


def sample_group_msg_launch(npoint: int, radius_list, nsample_list, xyz: torch.Tensor, center: bool, want_grouped: bool,
                            lens):
    import ctypes
    k = len(radius_list)
    b, n, _ = xyz.shape
    dev = xyz.device
    fps_idx = torch.empty((b, npoint), dtype=torch.int32, device=dev)
    new_xyz = torch.empty((b, npoint, 3), dtype=torch.float32, device=dev)
    idx = [torch.empty((b, npoint, int(s)), dtype=torch.int32, device=dev) for s in nsample_list]
    cnt = [torch.empty((b, npoint), dtype=torch.int32, device=dev) for _ in nsample_list]
    grouped = [torch.empty((b, npoint, int(s), 3), dtype=torch.float32, device=dev) for s in nsample_list] if want_grouped else None
    if b == 0:
        return fps_idx, new_xyz, idx, cnt, grouped
    lib = _lib.load()
    radii = (ctypes.c_float * k)(*[float(r) for r in radius_list])
    nsamples = (ctypes.c_int * k)(*[int(s) for s in nsample_list])
    pidx = (ctypes.c_void_p * k)(*[t.data_ptr() for t in idx])
    pcnt = (ctypes.c_void_p * k)(*[t.data_ptr() for t in cnt])
    pgrp = (ctypes.c_void_p * k)(*[t.data_ptr() for t in grouped]) if want_grouped else None
    with on_device(xyz):
        wsb = int(lib.pn2_sa_layer_device_workspace_bytes(b, n, npoint, max(int(s) for s in nsample_list)))
        ws = torch.empty(wsb, dtype=torch.uint8, device=dev) if wsb else None
        if lens is None:
            rc = lib.pn2_sa_layer_msg_device(b, n, npoint, k, radii, nsamples, ptr(xyz.detach()), ptr(fps_idx), ptr(new_xyz), pidx,
                                             pcnt, pgrp, 1 if center else 0, ptr(ws), wsb, stream_ptr(dev))
        else:
            rc = lib.pn2_sa_layer_msg_device_ragged(b, n, npoint, k, radii, nsamples, ptr(xyz.detach()), ptr(lens), ptr(fps_idx),
                                                    ptr(new_xyz), pidx, pcnt, pgrp, 1 if center else 0, ptr(ws), wsb,
                                                    stream_ptr(dev))
    _lib.check(rc, "pn2_sa_layer_msg_device")
    return fps_idx, new_xyz, idx, cnt, grouped


KNN_MAX_K = 128  # pn2_sa_knn_layer_device's (and pn2_knn_point's) largest k


def sample_knn(npoint: int, k: int, xyz: torch.Tensor, center: bool = True, want_grouped: bool = True,
               want_dist: bool = False, *, lengths=None):
    """FPS + gather_point + knn_point(k, xyz, new_xyz) + group_point(xyz) [- new_xyz] in one call.

    Returns (fps_idx (b,npoint) i32, new_xyz (b,npoint,3), idx (b,npoint,k) i32, dist (b,npoint,k) f32 or None,
    grouped_xyz (b,npoint,k,3) or None).  ``dist`` is knn_point's ``val`` (squared distances, ascending);
    ``center=True`` subtracts the centroid.  Bit-identical to the separate ops; no gradients.  Needs
    1 <= k <= min(n, 128) (ValueError otherwise: larger k keep knn_point's composite path).
    ``lengths`` (b,) integers, optional: cloud i is ``xyz[i, :lengths[i]]``.  Its fps_idx and new_xyz are what the
    sampling returns for it alone; idx, dist and grouped_xyz are ``knn_point(k, xyz, new_xyz, lengths=lengths)`` and
    its gather, so a cloud shorter than k repeats its nearest neighbour (column 0) in columns [lengths[i], k).  Every
    index is below its length.  A device tensor is never read on the host, so the call can be captured in a CUDA graph
    and replayed with new lengths written into the same tensor."""
    npoint, k = int(npoint), int(k)
    if npoint <= 0:
        raise ValueError("FarthestPointSample expects positive npoint")
    if k <= 0:
        raise ValueError("knn_point expects positive k")
    xyz = require_cuda(xyz, "xyz", torch.float32)
    if xyz.dim() != 3 or xyz.shape[2] != 3:
        raise ValueError(f"expected (batch_size, ndataset, 3) xyz shape, got {tuple(xyz.shape)}")
    b, n, _ = xyz.shape
    if n <= 0:
        raise ValueError("FarthestPointSample expects at least one point per batch entry")
    if k > n:
        raise ValueError(f"knn_point expects k <= ndataset (the reference slices k columns of an n-column matrix), got k={k}, n={n}")
    if k > KNN_MAX_K:
        raise ValueError(f"sample_knn expects k <= {KNN_MAX_K}, got k={k}")
    dev = xyz.device
    lens = device_lengths(lengths, b, n, dev, "sample_knn")
    if torch.compiler.is_compiling():
        fps_idx, new_xyz, idx, dist, grouped = torch.ops.pn2.sample_knn(npoint, k, xyz.detach(), bool(center),
                                                                        bool(want_grouped), bool(want_dist), lens)
        return fps_idx, new_xyz, idx, dist if want_dist else None, grouped if want_grouped else None
    return sample_knn_launch(npoint, k, xyz, center, want_grouped, want_dist, lens)


def sample_knn_launch(npoint: int, k: int, xyz: torch.Tensor, center: bool, want_grouped: bool, want_dist: bool, lens):
    b, n, _ = xyz.shape
    dev = xyz.device
    fps_idx = torch.empty((b, npoint), dtype=torch.int32, device=dev)
    new_xyz = torch.empty((b, npoint, 3), dtype=torch.float32, device=dev)
    idx = torch.empty((b, npoint, k), dtype=torch.int32, device=dev)
    dist = torch.empty((b, npoint, k), dtype=torch.float32, device=dev) if want_dist else None
    grouped = torch.empty((b, npoint, k, 3), dtype=torch.float32, device=dev) if want_grouped else None
    if b == 0:
        return fps_idx, new_xyz, idx, dist, grouped
    lib = _lib.load()
    with on_device(xyz):
        wsb = int(lib.pn2_sa_knn_layer_workspace_bytes(b, n, npoint, k))
        ws = torch.empty(wsb, dtype=torch.uint8, device=dev) if wsb else None
        if lens is None:
            rc = lib.pn2_sa_knn_layer_device(b, n, npoint, k, ptr(xyz.detach()), ptr(fps_idx), ptr(new_xyz), ptr(idx), ptr(dist),
                                             ptr(grouped), 1 if center else 0, ptr(ws), wsb, stream_ptr(dev))
        else:
            rc = lib.pn2_sa_knn_layer_device_ragged(b, n, npoint, k, ptr(xyz.detach()), ptr(lens), ptr(fps_idx), ptr(new_xyz),
                                                    ptr(idx), ptr(dist), ptr(grouped), 1 if center else 0, ptr(ws), wsb,
                                                    stream_ptr(dev))
    _lib.check(rc, "pn2_sa_knn_layer_device")
    return fps_idx, new_xyz, idx, dist, grouped


def ball_group(radius: float, nsample: int, xyz1: torch.Tensor, xyz2: torch.Tensor, center: bool = True,
               want_grouped: bool = True):
    """query_ball_point(radius, nsample, xyz1, xyz2) + group_point(xyz1, idx) [- xyz2] in one launch.

    Returns (idx, pts_cnt, grouped_xyz or None).  Falls back to the separate ops when the cloud does
    not fit the kernel's shared-memory grid (n > 9700)."""
    radius, nsample = float(radius), int(nsample)
    if not radius > 0:
        raise ValueError("QueryBallPoint expects positive radius")
    if nsample <= 0:
        raise ValueError("QueryBallPoint expects positive nsample")
    xyz1 = require_cuda(xyz1, "xyz1", torch.float32)
    xyz2 = require_cuda(xyz2, "xyz2", torch.float32)
    same_device(xyz1, xyz2)
    if xyz1.dim() != 3 or xyz1.shape[2] != 3 or xyz2.dim() != 3 or xyz2.shape[2] != 3 or xyz1.shape[0] != xyz2.shape[0]:
        raise ValueError("QueryBallPoint expects (batch_size, ndataset, 3) xyz1 and (batch_size, npoint, 3) xyz2")
    if torch.compiler.is_compiling():
        idx, cnt, g = torch.ops.pn2.ball_group(radius, nsample, xyz1.detach(), xyz2.detach(), bool(center), bool(want_grouped))
        return idx, cnt, g if want_grouped else None
    return ball_group_launch(radius, nsample, xyz1, xyz2, center, want_grouped)


def ball_group_launch(radius: float, nsample: int, xyz1: torch.Tensor, xyz2: torch.Tensor, center: bool, want_grouped: bool):
    b, n, _ = xyz1.shape
    m = xyz2.shape[1]
    lib = _lib.load()
    if n <= 0 or not lib.pn2_ball_group_fits(n):
        from .tf_grouping import group_point, query_ball_point
        idx, cnt = query_ball_point(radius, nsample, xyz1, xyz2)
        g = None
        if want_grouped:
            g = group_point(xyz1.detach(), idx)
            if center:
                g = g - xyz2.unsqueeze(2)
        return idx, cnt, g
    dev = xyz1.device
    idx = torch.empty((b, m, nsample), dtype=torch.int32, device=dev)
    cnt = torch.empty((b, m), dtype=torch.int32, device=dev)
    g = torch.empty((b, m, nsample, 3), dtype=torch.float32, device=dev) if want_grouped else None
    if b * m:
        with on_device(xyz1):
            rc = lib.pn2_ball_group(b, n, m, radius, nsample, ptr(xyz1.detach()), ptr(xyz2.detach()), ptr(idx), ptr(cnt), ptr(g),
                                    1 if center else 0, stream_ptr(dev))
        _lib.check(rc, "pn2_ball_group")
    return idx, cnt, g


class SetAbstractionDevice:
    """``depth`` independent batches of one SA sampling+grouping layer in flight on private streams.

    Usage::
        sa = SetAbstractionDevice(b, n, npoint, radius, nsample, depth=2)
        for xyz in device_batches:                 # (b,n,3) float32 CUDA tensors
            if sa.full():
                fps_idx, new_xyz, idx, pts_cnt, grouped = sa.collect()   # oldest batch, in order
            sa.submit(xyz)
        while sa.pending():
            ... = sa.collect()

    ``submit`` never blocks; the tensors ``collect`` returns belong to the slot and stay valid until
    the slot is reused (``depth`` submits later).  ``collect`` makes the caller's current stream wait
    for the batch (no host synchronisation unless ``sync=True``).

    ``submit(xyz, lengths)`` takes a padded batch of variable-size clouds (``lengths`` as for ``sample_group``:
    a device tensor is never read back, so ``enqueue`` with one can be captured in a CUDA graph and replayed
    with new lengths written into it).
    """

    def __init__(self, b, n, npoint, radius, nsample, depth: int = 2, center: bool = False, want_grouped: bool = True,
                 device=None):
        if depth < 1:
            raise ValueError("SetAbstractionDevice expects depth >= 1")
        if not torch.cuda.is_available():
            raise RuntimeError("SetAbstractionDevice needs a CUDA device: pointnet2_b200 has no CPU path")
        self.b, self.n, self.m, self.radius, self.s = int(b), int(n), int(npoint), float(radius), int(nsample)
        self.center = bool(center)
        self.device = torch.device(device if device is not None else f"cuda:{torch.cuda.current_device()}")
        self.lib = _lib.load()
        dev = self.device
        wsb = int(self.lib.pn2_sa_layer_device_workspace_bytes(self.b, self.n, self.m, self.s))
        self.slots = []
        for _ in range(int(depth)):
            self.slots.append(dict(
                fps_idx=torch.empty((self.b, self.m), dtype=torch.int32, device=dev),
                new_xyz=torch.empty((self.b, self.m, 3), dtype=torch.float32, device=dev),
                idx=torch.empty((self.b, self.m, self.s), dtype=torch.int32, device=dev),
                pts_cnt=torch.empty((self.b, self.m), dtype=torch.int32, device=dev),
                grouped=torch.empty((self.b, self.m, self.s, 3), dtype=torch.float32, device=dev) if want_grouped else None,
                ws=torch.empty(wsb, dtype=torch.uint8, device=dev) if wsb else None, wsb=wsb, xyz=None, lengths=None,
                stream=torch.cuda.Stream(dev), done=torch.cuda.Event()))
        self._next = 0
        self._inflight: collections.deque[int] = collections.deque()

    @property
    def depth(self) -> int:
        return len(self.slots)

    def pending(self) -> int:
        return len(self._inflight)

    def full(self) -> bool:
        return len(self._inflight) == len(self.slots)

    def enqueue(self, slot: dict, xyz: torch.Tensor, stream: torch.cuda.Stream, lengths: torch.Tensor | None = None) -> None:
        """Issue the layer for ``xyz`` into ``slot``'s buffers on ``stream`` (capturable in a CUDA graph).
        ``lengths``: None, or the (b,) int32 device tensor of per-cloud lengths."""
        with torch.cuda.device(self.device):
            if lengths is None:
                rc = self.lib.pn2_sa_layer_device(self.b, self.n, self.m, self.radius, self.s, ptr(xyz), ptr(slot["fps_idx"]),
                                                  ptr(slot["new_xyz"]), ptr(slot["idx"]), ptr(slot["pts_cnt"]), ptr(slot["grouped"]),
                                                  1 if self.center else 0, ptr(slot["ws"]), slot["wsb"], stream.cuda_stream)
            else:
                rc = self.lib.pn2_sa_layer_device_ragged(self.b, self.n, self.m, self.radius, self.s, ptr(xyz), ptr(lengths),
                                                         ptr(slot["fps_idx"]), ptr(slot["new_xyz"]), ptr(slot["idx"]),
                                                         ptr(slot["pts_cnt"]), ptr(slot["grouped"]), 1 if self.center else 0,
                                                         ptr(slot["ws"]), slot["wsb"], stream.cuda_stream)
        _lib.check(rc, "pn2_sa_layer_device")

    def submit(self, xyz: torch.Tensor, lengths=None) -> int:
        if self.full():
            raise RuntimeError("SetAbstractionDevice is full: collect() the oldest batch first")
        xyz = require_cuda(xyz, "xyz", torch.float32)
        if tuple(xyz.shape) != (self.b, self.n, 3):
            raise ValueError(f"expected xyz of shape {(self.b, self.n, 3)}, got {tuple(xyz.shape)}")
        lens = device_lengths(lengths, self.b, self.n, self.device, "SetAbstractionDevice")
        i = self._next
        slot = self.slots[i]
        slot["xyz"], slot["lengths"] = xyz, lens  # keep the inputs alive while the kernels read them
        st = slot["stream"]
        st.wait_stream(torch.cuda.current_stream(self.device))  # xyz (and lengths) were produced on the caller's stream
        self.enqueue(slot, xyz, st, lens)
        slot["done"].record(st)
        self._inflight.append(i)
        self._next = (i + 1) % len(self.slots)
        return i

    def collect(self, sync: bool = False):
        if not self._inflight:
            raise RuntimeError("SetAbstractionDevice.collect() with nothing submitted")
        i = self._inflight.popleft()
        s = self.slots[i]
        if sync:
            s["done"].synchronize()
        else:
            torch.cuda.current_stream(self.device).wait_event(s["done"])
        return s["fps_idx"], s["new_xyz"], s["idx"], s["pts_cnt"], s["grouped"]
