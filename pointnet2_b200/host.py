"""Host-buffer entry to the set-abstraction path.

The reference is driven from numpy through ``sess.run(feed_dict=...)`` (train.py:226-231): inputs
start in host memory and results come back to host memory.  ``SetAbstractionHost`` is that call
for one SSG sampling+grouping layer (farthest_point_sample + gather_point + query_ball_point +
group_point(xyz), utils/pointnet_util.py:40-45): it owns pinned host staging buffers and a device
workspace, and each ``run`` issues H2D copy -> the overlapped sampling + grouping kernels (sa_fused.cu) -> D2H copies on one
stream through the C-ABI ``pn2_sa_layer_host``.

``SetAbstractionPipeline`` is the same call for a STREAM of batches (the reference's training loop
feeds one batch per ``sess.run`` while its input queue prepares the next, train.py:207-231): a ring
of ``depth`` such sessions, each on its own CUDA stream, so batch k+1's copy-in and sampling overlap
batch k's grouping and copy-out.  One FPS launch occupies one SM per cloud (32 of 132 at the
benchmark's batch size), so consecutive batches really do run side by side.

``ragged=True`` takes batches of differently sized clouds (a ``feed_dict`` of numpy clouds of their own
lengths) through ``pn2_sa_layer_host_ragged``: the clouds are packed back to back into one pinned buffer,
only their real rows cross PCIe, and the device layer runs at the stride of the longest cloud of the
batch rather than at the capacity ``n``.  Each cloud gets bit for bit what the dense layer computes for it
alone (DESIGN.md §6.8).

``radius`` and ``nsample`` given as equal-length sequences make either class the multi-scale layer
(pointnet_sa_module_msg, utils/pointnet_util.py:156-196) through ``pn2_sa_layer_msg_host`` /
``pn2_sa_layer_msg_host_ragged``: ONE sampling chain and one copy-in for every scale, each scale's ball query
overlapping the chain as in ``sa_layer.sample_group_msg``, whose results it returns.
"""
from __future__ import annotations

import collections
import collections.abc
import ctypes

import numpy as np
import torch

from . import _lib, numa


def pack_clouds(clouds, n: int, xyz: np.ndarray, lengths: np.ndarray) -> int:
    """Copy ``clouds`` (a sequence of len(lengths) float32 (len_i, 3) arrays, 1 <= len_i <= n) back to back into
    the packed (>= sum len_i, 3) float32 array ``xyz`` and their lengths into the int32 array ``lengths``.
    Returns the number of rows written.  ValueError / TypeError before anything is written."""
    b = lengths.shape[0]
    if isinstance(clouds, np.ndarray) or len(clouds) != b:
        raise ValueError(f"expected a list of {b} clouds, got {type(clouds).__name__} of length {len(clouds)}")
    for i, c in enumerate(clouds):
        if not isinstance(c, np.ndarray) or c.dtype != np.float32:
            raise TypeError(f"cloud {i}: expected a float32 numpy array, got {getattr(c, 'dtype', type(c).__name__)}")
        if c.ndim != 2 or c.shape[1] != 3:
            raise ValueError(f"cloud {i}: expected shape (len, 3), got {c.shape}")
        if not 1 <= c.shape[0] <= n:
            raise ValueError(f"cloud {i}: expected 1 <= len <= {n} (the capacity) points, got {c.shape[0]}")
    off = 0
    for i, c in enumerate(clouds):
        xyz[off:off + c.shape[0]] = c
        lengths[i] = c.shape[0]
        off += c.shape[0]
    return off


def _pointers(tensors):
    """a C array of the tensors' data pointers, NULL for None"""
    return (ctypes.c_void_p * len(tensors))(*[t.data_ptr() if t is not None else None for t in tensors])


def check_lengths(lengths, b: int, n: int) -> np.ndarray:
    """Host lengths of a ragged batch as a (b,) int64 array; ValueError unless 1 <= l <= n for each."""
    arr = np.asarray(lengths)
    if arr.shape != (b,) or (arr.size and not np.issubdtype(arr.dtype, np.integer)):
        raise ValueError(f"expected ({b},) integer lengths, got {arr.dtype} {arr.shape}")
    if b and (int(arr.min()) < 1 or int(arr.max()) > n):
        raise ValueError(f"expected 1 <= lengths <= {n} (the capacity), got {arr.tolist()}")
    return arr.astype(np.int64)


MAX_SCALES = 16  # pn2_sa_layer_msg_host's


def _is_sequence(v) -> bool:
    if isinstance(v, np.ndarray):
        return v.ndim > 0
    return isinstance(v, collections.abc.Sequence) and not isinstance(v, (str, bytes))


def layer_scales(radius, nsample, want_grouped=True):
    """The scales of a host-buffer layer.  None for the single-scale form (radius and nsample scalars, want_grouped a
    bool); for the multi-scale form (radius and nsample equal-length sequences) the tuples (radii, nsamples, wants),
    want_grouped being a bool for every scale or a sequence of one bool per scale.  ValueError for empty or unequal
    sequences, a scalar mixed with a sequence, more than MAX_SCALES scales, or a non-positive radius or nsample."""
    if not _is_sequence(radius) and not _is_sequence(nsample):
        if _is_sequence(want_grouped):
            raise ValueError("a per-scale want_grouped needs radius and nsample sequences")
        return None
    if not (_is_sequence(radius) and _is_sequence(nsample)) or len(radius) != len(nsample) or not len(radius):
        raise ValueError("radius and nsample must be non-empty sequences of equal length")
    if len(radius) > MAX_SCALES:
        raise ValueError(f"at most {MAX_SCALES} scales, got {len(radius)}")
    radii, nsamples = tuple(float(r) for r in radius), tuple(int(v) for v in nsample)
    if not all(r > 0 for r in radii):
        raise ValueError(f"QueryBallPoint expects positive radii, got {list(radii)}")
    if min(nsamples) <= 0:
        raise ValueError(f"QueryBallPoint expects positive nsample, got {list(nsamples)}")
    if _is_sequence(want_grouped):
        if len(want_grouped) != len(radii):
            raise ValueError(f"want_grouped has {len(want_grouped)} entries for {len(radii)} scales")
        wants = tuple(bool(w) for w in want_grouped)
    else:
        wants = (bool(want_grouped),) * len(radii)
    return radii, nsamples, wants


class SetAbstractionHost:
    """One SSG sampling+grouping layer fed from and returning to pinned host memory.

    ``ragged=False``: ``h_xyz`` is a (b, n, 3) batch.  ``ragged=True``: ``h_xyz`` is a packed (b*n, 3) buffer whose
    first sum(lengths) rows hold the clouds back to back and ``h_lengths`` the (b,) lengths; ``run`` / ``pack`` take a
    list of b float32 (len_i, 3) arrays, 1 <= len_i <= n.  ``h2d_bytes`` is what the last launch copied to the device,
    ``d2h_bytes`` what each launch copies back.

    ``radius`` and ``nsample`` as equal-length sequences (see ``layer_scales``): the multi-scale layer.  ``h_idx`` and
    ``h_pts_cnt`` are then lists of one buffer per scale and ``h_grouped_xyz`` a list (None for a scale whose
    grouped_xyz is not wanted, which is then neither computed nor copied back) or None when no scale wants it.
    """

    def __init__(self, b: int, n: int, npoint: int, radius, nsample, device=None, want_grouped=True,
                 ragged: bool = False):
        scales = layer_scales(radius, nsample, want_grouped)
        if not torch.cuda.is_available():
            raise RuntimeError("SetAbstractionHost needs a CUDA device: pointnet2_b200 has no CPU path")
        self.b, self.n, self.m = int(b), int(n), int(npoint)
        self.msg = scales is not None
        if self.msg:
            self.radii, self.nsamples, wants = scales
            k = len(self.radii)
            self._c_radii = (ctypes.c_float * k)(*self.radii)
            self._c_nsamples = (ctypes.c_int * k)(*self.nsamples)
        else:
            self.radius, self.s = float(radius), int(nsample)
        self.ragged = bool(ragged)
        self.device = torch.device(device if device is not None else f"cuda:{torch.cuda.current_device()}")
        self.lib = _lib.load()
        if self.msg:
            ws_fn = (self.lib.pn2_sa_layer_msg_host_ragged_workspace_bytes if self.ragged
                     else self.lib.pn2_sa_layer_msg_host_workspace_bytes)
            ws = int(ws_fn(self.b, self.n, self.m, k, self._c_nsamples))
        else:
            ws_fn = self.lib.pn2_sa_layer_host_ragged_workspace_bytes if self.ragged else self.lib.pn2_sa_layer_workspace_bytes
            ws = int(ws_fn(self.b, self.n, self.m, self.s))
        if ws <= 0:
            raise ValueError("SetAbstractionHost expects positive b, n, npoint, nsample")
        self.workspace = torch.empty(ws, dtype=torch.uint8, device=self.device)
        pin = dict(pin_memory=True)
        # pinned staging buffers are placed on the NUMA node the GPU hangs off (the copies of a rank
        # whose buffers sit on the other socket cross the inter-socket link and do not scale)
        with numa.prefer_node_of(self.device):
            self.h_xyz = torch.empty((self.b * self.n, 3) if self.ragged else (self.b, self.n, 3), dtype=torch.float32, **pin)
            self.h_lengths = torch.full((self.b,), self.n, dtype=torch.int32, **pin) if self.ragged else None
            self.h_new_xyz = torch.empty((self.b, self.m, 3), dtype=torch.float32, **pin)
            if self.msg:
                i32, f32 = dict(dtype=torch.int32, **pin), dict(dtype=torch.float32, **pin)
                self.h_idx = [torch.empty((self.b, self.m, s), **i32) for s in self.nsamples]
                self.h_pts_cnt = [torch.empty((self.b, self.m), **i32) for _ in self.nsamples]
                self.h_grouped_xyz = ([torch.empty((self.b, self.m, s, 3), **f32) if w else None
                                       for s, w in zip(self.nsamples, wants)] if any(wants) else None)
            else:
                self.h_idx = torch.empty((self.b, self.m, self.s), dtype=torch.int32, **pin)
                self.h_pts_cnt = torch.empty((self.b, self.m), dtype=torch.int32, **pin)
                # want_grouped=False: grouped_xyz is neither computed nor copied back (it is xyz[idx], which a
                # host-side caller can regroup itself) — 3/4 of the device-to-host bytes of the layer
                self.h_grouped_xyz = (torch.empty((self.b, self.m, self.s, 3), dtype=torch.float32, **pin)
                                      if want_grouped else None)
            outs = [t for v in (self.h_new_xyz, self.h_idx, self.h_pts_cnt, self.h_grouped_xyz)
                    for t in (v if isinstance(v, list) else [v]) if t is not None]
            for t in [self.h_xyz] + outs:
                t.zero_()  # first touch under the NUMA preference
        if self.msg:  # the host pointer arrays the multi-scale entries take
            self._c_idx, self._c_cnt = _pointers(self.h_idx), _pointers(self.h_pts_cnt)
            self._c_grp = _pointers(self.h_grouped_xyz) if self.h_grouped_xyz is not None else None
        self.h2d_bytes = self.h_xyz.numel() * 4
        self.d2h_bytes = 4 * sum(t.numel() for t in outs)

    def pack(self, clouds) -> None:
        """ragged=True: write a list of b float32 (len_i, 3) arrays into the pinned packed input and lengths."""
        if not self.ragged:
            raise RuntimeError("SetAbstractionHost.pack needs ragged=True")
        pack_clouds(clouds, self.n, self.h_xyz.numpy(), self.h_lengths.numpy())

    def set_lengths(self, lengths) -> None:
        """ragged=True: the lengths of clouds already written back to back into ``h_xyz``."""
        if not self.ragged:
            raise RuntimeError("SetAbstractionHost.set_lengths needs ragged=True")
        self.h_lengths.numpy()[...] = check_lengths(lengths, self.b, self.n)

    def launch(self, stream: torch.cuda.Stream | None = None) -> None:
        """Enqueue copy-in, the kernels and copy-out for whatever is in ``self.h_xyz`` (and ``self.h_lengths``)."""
        vp = ctypes.c_void_p
        with torch.cuda.device(self.device):
            st = stream if stream is not None else torch.cuda.current_stream(self.device)
            inp = [vp(self.h_xyz.data_ptr())] + ([vp(self.h_lengths.data_ptr())] if self.ragged else [])
            tail = (vp(self.workspace.data_ptr()), ctypes.c_size_t(self.workspace.numel()), vp(st.cuda_stream))
            if self.msg:
                name = "pn2_sa_layer_msg_host_ragged" if self.ragged else "pn2_sa_layer_msg_host"
                rc = getattr(self.lib, name)(self.b, self.n, self.m, len(self.radii), self._c_radii, self._c_nsamples, *inp,
                                             vp(self.h_new_xyz.data_ptr()), self._c_idx, self._c_cnt, self._c_grp, *tail)
            else:
                name = "pn2_sa_layer_host_ragged" if self.ragged else "pn2_sa_layer_host"
                rc = getattr(self.lib, name)(
                    self.b, self.n, self.m, self.radius, self.s, *inp,
                    vp(self.h_new_xyz.data_ptr()), vp(self.h_idx.data_ptr()), vp(self.h_pts_cnt.data_ptr()),
                    vp(self.h_grouped_xyz.data_ptr() if self.h_grouped_xyz is not None else 0), *tail)
        _lib.check(rc, name)
        if self.ragged:
            # read after the call succeeded, as the entry read them: the lengths copy and the packed rows
            self.h2d_bytes = 4 * self.b + 12 * int(self.h_lengths.numpy().sum(dtype=np.int64))

    def outputs(self, copy: bool = False):
        """(new_xyz, idx, pts_cnt, grouped_xyz) as numpy views of the pinned outputs, or copies.  Multi-scale: idx and
        pts_cnt are lists of one array per scale, grouped_xyz a list (None for a scale not wanted) or None."""
        one = lambda t: None if t is None else (t.numpy().copy() if copy else t.numpy())  # noqa: E731
        each = lambda v: [one(t) for t in v] if isinstance(v, list) else one(v)  # noqa: E731
        return one(self.h_new_xyz), each(self.h_idx), each(self.h_pts_cnt), each(self.h_grouped_xyz)

    def run(self, xyz):
        """xyz: (b,n,3) float32 numpy array, or with ragged=True a list of b float32 (len_i, 3) arrays.
        Returns numpy (new_xyz, idx, pts_cnt, grouped_xyz), with lists for the multi-scale layer (see ``outputs``)."""
        if self.ragged:
            self.pack(xyz)
        else:
            xyz = np.ascontiguousarray(xyz, dtype=np.float32)
            if xyz.shape != (self.b, self.n, 3):
                raise ValueError(f"expected xyz of shape {(self.b, self.n, 3)}, got {xyz.shape}")
            self.h_xyz.numpy()[...] = xyz
        self.launch()
        torch.cuda.current_stream(self.device).synchronize()
        return self.outputs(copy=True)


class SetAbstractionPipeline:
    """A ring of ``depth`` SetAbstractionHost sessions on private streams.

    Usage::
        pipe = SetAbstractionPipeline(b, n, npoint, radius, nsample, depth=2)
        for batch in batches:
            if pipe.full():
                new_xyz, idx, pts_cnt, grouped_xyz = pipe.collect()   # oldest batch, in order
            pipe.input_buffer()[...] = batch                          # fill the pinned slot
            pipe.submit()
        while pipe.pending():
            ... = pipe.collect()

    ``collect`` returns numpy views of the slot's pinned output buffers; they stay valid until the
    next ``submit`` that reuses the slot (``depth`` submits later).

    ``ragged=True``: ``submit(clouds)`` takes a list of b float32 (len_i, 3) arrays; or fill the first
    sum(lengths) rows of the packed ``input_buffer()`` with the clouds back to back and ``submit(lengths=...)``.
    ``h2d_bytes`` is what the last submitted batch copied to the device.

    ``radius`` and ``nsample`` as equal-length sequences: the multi-scale layer, whose ``collect`` returns
    (new_xyz, [idx_k], [pts_cnt_k], [grouped_xyz_k] or None) as ``SetAbstractionHost.outputs`` does.
    """

    def __init__(self, b: int, n: int, npoint: int, radius, nsample, depth: int = 2, device=None,
                 want_grouped=True, ragged: bool = False):
        if depth < 1:
            raise ValueError("SetAbstractionPipeline expects depth >= 1")
        self.ragged = bool(ragged)
        self.slots = [SetAbstractionHost(b, n, npoint, radius, nsample, device=device, want_grouped=want_grouped,
                                         ragged=self.ragged)
                      for _ in range(int(depth))]
        self.device = self.slots[0].device
        self.streams = [torch.cuda.Stream(self.device) for _ in self.slots]
        self.done = [torch.cuda.Event() for _ in self.slots]
        self._next = 0
        self._inflight: collections.deque[int] = collections.deque()
        self.h2d_bytes, self.d2h_bytes = self.slots[0].h2d_bytes, self.slots[0].d2h_bytes

    @property
    def depth(self) -> int:
        return len(self.slots)

    def pending(self) -> int:
        return len(self._inflight)

    def full(self) -> bool:
        return len(self._inflight) == len(self.slots)

    def input_buffer(self) -> np.ndarray:
        """The pinned (b,n,3) float32 input of the slot the next ``submit`` will use; (b*n,3) packed with ragged=True."""
        if self.full():
            raise RuntimeError("SetAbstractionPipeline is full: collect() the oldest batch first")
        return self.slots[self._next].h_xyz.numpy()

    def submit(self, xyz=None, after: torch.cuda.Event | None = None, *, lengths=None) -> int:
        """Enqueue one batch (``xyz`` is copied into the slot's pinned input when given; otherwise
        whatever ``input_buffer()`` holds is used, with ``lengths`` when ragged). Returns the slot index. Never blocks."""
        if self.full():
            raise RuntimeError("SetAbstractionPipeline is full: collect() the oldest batch first")
        i = self._next
        slot = self.slots[i]
        if self.ragged:
            if (xyz is None) == (lengths is None):
                raise ValueError("a ragged SetAbstractionPipeline.submit takes either a list of clouds or lengths")
            if xyz is not None:
                slot.pack(xyz)
            else:
                slot.set_lengths(lengths)
        elif lengths is not None:
            raise ValueError("lengths need SetAbstractionPipeline(..., ragged=True)")
        elif xyz is not None:
            xyz = np.ascontiguousarray(xyz, dtype=np.float32)
            if xyz.shape != (slot.b, slot.n, 3):
                raise ValueError(f"expected xyz of shape {(slot.b, slot.n, 3)}, got {xyz.shape}")
            slot.h_xyz.numpy()[...] = xyz
        if after is not None:
            self.streams[i].wait_event(after)
        slot.launch(self.streams[i])
        self.h2d_bytes = slot.h2d_bytes
        self.done[i].record(self.streams[i])
        self._inflight.append(i)
        self._next = (i + 1) % len(self.slots)
        return i

    def collect(self):
        """Wait for the OLDEST submitted batch; returns (new_xyz, idx, pts_cnt, grouped_xyz) views."""
        if not self._inflight:
            raise RuntimeError("SetAbstractionPipeline.collect() with nothing submitted")
        i = self._inflight.popleft()
        self.done[i].synchronize()
        return self.slots[i].outputs()
