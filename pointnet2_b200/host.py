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
"""
from __future__ import annotations

import collections
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


def check_lengths(lengths, b: int, n: int) -> np.ndarray:
    """Host lengths of a ragged batch as a (b,) int64 array; ValueError unless 1 <= l <= n for each."""
    arr = np.asarray(lengths)
    if arr.shape != (b,) or (arr.size and not np.issubdtype(arr.dtype, np.integer)):
        raise ValueError(f"expected ({b},) integer lengths, got {arr.dtype} {arr.shape}")
    if b and (int(arr.min()) < 1 or int(arr.max()) > n):
        raise ValueError(f"expected 1 <= lengths <= {n} (the capacity), got {arr.tolist()}")
    return arr.astype(np.int64)


class SetAbstractionHost:
    """One SSG sampling+grouping layer fed from and returning to pinned host memory.

    ``ragged=False``: ``h_xyz`` is a (b, n, 3) batch.  ``ragged=True``: ``h_xyz`` is a packed (b*n, 3) buffer whose
    first sum(lengths) rows hold the clouds back to back and ``h_lengths`` the (b,) lengths; ``run`` / ``pack`` take a
    list of b float32 (len_i, 3) arrays, 1 <= len_i <= n.  ``h2d_bytes`` is what the last launch copied to the device.
    """

    def __init__(self, b: int, n: int, npoint: int, radius: float, nsample: int, device=None, want_grouped: bool = True,
                 ragged: bool = False):
        if not torch.cuda.is_available():
            raise RuntimeError("SetAbstractionHost needs a CUDA device: pointnet2_b200 has no CPU path")
        self.b, self.n, self.m, self.radius, self.s = int(b), int(n), int(npoint), float(radius), int(nsample)
        self.ragged = bool(ragged)
        self.device = torch.device(device if device is not None else f"cuda:{torch.cuda.current_device()}")
        self.lib = _lib.load()
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
            self.h_idx = torch.empty((self.b, self.m, self.s), dtype=torch.int32, **pin)
            self.h_pts_cnt = torch.empty((self.b, self.m), dtype=torch.int32, **pin)
            # want_grouped=False: grouped_xyz is neither computed nor copied back (it is xyz[idx], which a
            # host-side caller can regroup itself) — 3/4 of the device-to-host bytes of the layer
            self.h_grouped_xyz = (torch.empty((self.b, self.m, self.s, 3), dtype=torch.float32, **pin)
                                  if want_grouped else None)
            for t in (self.h_xyz, self.h_new_xyz, self.h_idx, self.h_pts_cnt, self.h_grouped_xyz):
                if t is not None:
                    t.zero_()  # first touch under the NUMA preference
        self.h2d_bytes = self.h_xyz.numel() * 4
        self.d2h_bytes = 4 * (self.h_new_xyz.numel() + self.h_idx.numel() + self.h_pts_cnt.numel()
                              + (self.h_grouped_xyz.numel() if want_grouped else 0))

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
        with torch.cuda.device(self.device):
            st = stream if stream is not None else torch.cuda.current_stream(self.device)
            if self.ragged:
                rc = self.lib.pn2_sa_layer_host_ragged(
                    self.b, self.n, self.m, self.radius, self.s,
                    ctypes.c_void_p(self.h_xyz.data_ptr()), ctypes.c_void_p(self.h_lengths.data_ptr()),
                    ctypes.c_void_p(self.h_new_xyz.data_ptr()), ctypes.c_void_p(self.h_idx.data_ptr()),
                    ctypes.c_void_p(self.h_pts_cnt.data_ptr()),
                    ctypes.c_void_p(self.h_grouped_xyz.data_ptr() if self.h_grouped_xyz is not None else 0),
                    ctypes.c_void_p(self.workspace.data_ptr()),
                    ctypes.c_size_t(self.workspace.numel()), ctypes.c_void_p(st.cuda_stream))
                _lib.check(rc, "pn2_sa_layer_host_ragged")
                # read after the call succeeded, as the entry read them: the lengths copy and the packed rows
                self.h2d_bytes = 4 * self.b + 12 * int(self.h_lengths.numpy().sum(dtype=np.int64))
                return
            rc = self.lib.pn2_sa_layer_host(
                self.b, self.n, self.m, self.radius, self.s,
                ctypes.c_void_p(self.h_xyz.data_ptr()), ctypes.c_void_p(self.h_new_xyz.data_ptr()),
                ctypes.c_void_p(self.h_idx.data_ptr()), ctypes.c_void_p(self.h_pts_cnt.data_ptr()),
                ctypes.c_void_p(self.h_grouped_xyz.data_ptr() if self.h_grouped_xyz is not None else 0),
                ctypes.c_void_p(self.workspace.data_ptr()),
                ctypes.c_size_t(self.workspace.numel()), ctypes.c_void_p(st.cuda_stream))
        _lib.check(rc, "pn2_sa_layer_host")

    def run(self, xyz):
        """xyz: (b,n,3) float32 numpy array, or with ragged=True a list of b float32 (len_i, 3) arrays.
        Returns numpy (new_xyz, idx, pts_cnt, grouped_xyz)."""
        if self.ragged:
            self.pack(xyz)
        else:
            xyz = np.ascontiguousarray(xyz, dtype=np.float32)
            if xyz.shape != (self.b, self.n, 3):
                raise ValueError(f"expected xyz of shape {(self.b, self.n, 3)}, got {xyz.shape}")
            self.h_xyz.numpy()[...] = xyz
        self.launch()
        torch.cuda.current_stream(self.device).synchronize()
        return (self.h_new_xyz.numpy().copy(), self.h_idx.numpy().copy(), self.h_pts_cnt.numpy().copy(),
                self.h_grouped_xyz.numpy().copy() if self.h_grouped_xyz is not None else None)


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
    """

    def __init__(self, b: int, n: int, npoint: int, radius: float, nsample: int, depth: int = 2, device=None,
                 want_grouped: bool = True, ragged: bool = False):
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
        s = self.slots[i]
        return (s.h_new_xyz.numpy(), s.h_idx.numpy(), s.h_pts_cnt.numpy(),
                s.h_grouped_xyz.numpy() if s.h_grouped_xyz is not None else None)
