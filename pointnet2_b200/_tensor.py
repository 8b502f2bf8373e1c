"""Argument checking shared by the op wrappers.

Mirrors the reference OpKernels' OP_REQUIRES checks (tf_ops/sampling/tf_sampling.cpp:99,105,131,135;
tf_ops/grouping/tf_grouping.cpp:71-84,90,96; tf_ops/3d_interpolation/tf_interpolate.cpp:163-168,
197-206): shape / attribute violations raise ValueError (TensorFlow: InvalidArgument), wrong dtypes
raise TypeError.  Tensors must live on a CUDA device: there is no CPU path.  The seeded samplers (scene.py, shapes.py)
share their set packing and their seed, index and npoints checks here.
"""
from __future__ import annotations

import ctypes
from contextlib import contextmanager

import numpy as np
import torch


# Feature tensors may be float32, bfloat16 or float16 (the kernels compute in float32 and round once); coordinates,
# weights and indices have a single dtype.
FEATURE_DTYPES = (torch.float32, torch.bfloat16, torch.float16)

# dtype codes of the typed entry points (include/pn2_api.h: PN2_F32, PN2_BF16, PN2_F16)
DTYPE_CODES = {torch.float32: 0, torch.bfloat16: 1, torch.float16: 2}


def require_cuda(t: torch.Tensor, name: str, dtype) -> torch.Tensor:
    """``dtype``: one torch.dtype or a tuple of the allowed ones."""
    if not isinstance(t, torch.Tensor):
        raise TypeError(f"{name} must be a torch.Tensor, got {type(t).__name__}")
    allowed = dtype if isinstance(dtype, tuple) else (dtype,)
    if t.dtype not in allowed:
        want = allowed[0] if len(allowed) == 1 else " or ".join(str(d) for d in allowed)
        raise TypeError(f"{name} must be {want}, got {t.dtype}")
    if not t.is_cuda:
        raise RuntimeError(f"{name} must be a CUDA tensor: pointnet2_b200 has no CPU path "
                           f"(got device {t.device})")
    return t if t.is_contiguous() else t.contiguous()


_INT_DTYPES = (torch.int8, torch.int16, torch.int32, torch.int64, torch.uint8)


def device_lengths(lengths, b: int, n: int, device: torch.device, op: str):
    """Per-cloud lengths of a padded (b, n, 3) batch as the (b,) int32 tensor on ``device`` the ragged entries take,
    or None for ``lengths=None`` (every cloud has n points).

    A tensor on ``device`` is used as is (another integer dtype is converted on the device) and never read back: the
    kernels clamp its values to [1, n], so the call stays asynchronous and capturable in a CUDA graph.  A CPU tensor, a
    numpy array or a Python sequence is checked here — shape (b,), 1 <= l <= n, else ValueError, as the reference's
    OP_REQUIRES would — and then copied to the device."""
    if lengths is None:
        return None
    if isinstance(lengths, torch.Tensor) and lengths.is_cuda:
        if lengths.device != device:
            raise RuntimeError(f"all tensors must be on the same device ({device} vs {lengths.device})")
        if lengths.dtype not in _INT_DTYPES:
            raise TypeError(f"{op} expects integer lengths, got {lengths.dtype}")
        if tuple(lengths.shape) != (b,):
            raise ValueError(f"{op} expects (batch_size,) lengths shape ({b},), got {tuple(lengths.shape)}")
        return lengths.to(torch.int32).contiguous()
    if not isinstance(lengths, torch.Tensor) and torch.compiler.is_compiling():
        # traced (torch.export): a host sequence is checked here, in Python, and enters the graph as a constant
        arr = np.asarray(lengths)
        if arr.size and not np.issubdtype(arr.dtype, np.integer):
            raise TypeError(f"{op} expects integer lengths, got {arr.dtype}")
        if tuple(arr.shape) != (b,):
            raise ValueError(f"{op} expects (batch_size,) lengths shape ({b},), got {tuple(arr.shape)}")
        vals = [int(v) for v in arr.tolist()]
        if b and (min(vals) < 1 or max(vals) > n):
            raise ValueError(f"{op} expects 1 <= lengths <= {n} (the padded number of points), got {vals}")
        return torch.tensor(vals, dtype=torch.int32, device=device)
    if isinstance(lengths, torch.Tensor):
        if lengths.dtype not in _INT_DTYPES:
            raise TypeError(f"{op} expects integer lengths, got {lengths.dtype}")
        host = lengths.detach().to(torch.int64)
    else:
        arr = np.asarray(lengths)
        if arr.size and not np.issubdtype(arr.dtype, np.integer):
            raise TypeError(f"{op} expects integer lengths, got {arr.dtype}")
        host = torch.from_numpy(arr.astype(np.int64).reshape(arr.shape))
    if tuple(host.shape) != (b,):
        raise ValueError(f"{op} expects (batch_size,) lengths shape ({b},), got {tuple(host.shape)}")
    if b and (int(host.min()) < 1 or int(host.max()) > n):
        raise ValueError(f"{op} expects 1 <= lengths <= {n} (the padded number of points), got {host.tolist()}")
    return host.to(torch.int32).to(device)


def as_int(v, name: str, op: str) -> int:
    """``v`` as a Python int; TypeError for anything but an int or a numpy integer (bool included)."""
    if isinstance(v, bool) or not isinstance(v, (int, np.integer)):
        raise TypeError(f"{op} expects an integer {name}, got {type(v).__name__}")
    return int(v)


def device_lengths0(lengths, b: int, n: int, device: torch.device, op: str):
    """(b,) int32 lengths on ``device`` or None.  A CUDA tensor is used as is (the kernels clamp to [0, n]); a host
    value is checked here (0 <= l <= n) and copied."""
    if lengths is None:
        return None
    if isinstance(lengths, torch.Tensor) and lengths.is_cuda:
        if lengths.device != device:
            raise RuntimeError(f"all tensors must be on the same device ({device} vs {lengths.device})")
        if lengths.dtype not in _INT_DTYPES:
            raise TypeError(f"{op} expects integer lengths, got {lengths.dtype}")
        if tuple(lengths.shape) != (b,):
            raise ValueError(f"{op} expects (batch_size,) lengths shape ({b},), got {tuple(lengths.shape)}")
        return lengths.to(torch.int32).contiguous()
    host = np.asarray(lengths.cpu() if isinstance(lengths, torch.Tensor) else lengths)
    if host.size and not np.issubdtype(host.dtype, np.integer):
        raise TypeError(f"{op} expects integer lengths, got {host.dtype}")
    if host.shape != (b,):
        raise ValueError(f"{op} expects (batch_size,) lengths shape ({b},), got {host.shape}")
    if b and (host.min() < 0 or host.max() > n):
        raise ValueError(f"{op} expects 0 <= lengths <= {n} (the padded number of points), got {host.tolist()}")
    return torch.from_numpy(host.astype(np.int32)).to(device)


I31 = 2 ** 31
SELECT_MAX_ROWS = 16384  # npoints cap of the samplers: their row sort is npoints x 8 bytes of shared memory


def to_host(a) -> np.ndarray:
    if isinstance(a, torch.Tensor):
        return a.detach().cpu().numpy()
    return np.asarray(a)


def pack_offsets(arrays, owner: str, device):
    """(sizes, offsets) of a set packed from ``arrays``: sizes (S,) numpy int64, kept on the host, and offsets (S + 1,)
    int64 on ``device`` (default: the current CUDA device), member k holding rows offsets[k] .. offsets[k + 1] - 1.
    Refuses 2^31 - 1 rows or more in all: rows and their ends are int32 in the kernels."""
    sizes = np.array([len(a) for a in arrays], np.int64)
    if int(sizes.sum()) >= I31 - 1:
        raise ValueError(f"{owner} takes fewer than 2^31 - 1 points in all, got {int(sizes.sum())}")
    dev = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
    return sizes, torch.from_numpy(np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)).to(dev)


def on_set_device(t: torch.Tensor, name: str, dev: torch.device) -> None:
    if t.device != dev:
        raise RuntimeError(f"{name} must be on the set's device {dev}, got {t.device}")


def check_npoints(npoints, op: str) -> None:
    if isinstance(npoints, bool) or not isinstance(npoints, int):
        raise TypeError(f"{op} expects an integer npoints, got {type(npoints).__name__}")
    if not 1 <= npoints <= SELECT_MAX_ROWS:
        raise ValueError(f"{op} expects 1 <= npoints <= {SELECT_MAX_ROWS} (the shared-memory sort), got {npoints}")


def check_dropout(max_dropout, op: str) -> None:
    if isinstance(max_dropout, bool) or not isinstance(max_dropout, (int, float)):
        raise TypeError(f"{op} expects a number for max_dropout, got {type(max_dropout).__name__}")
    if not 0.0 <= max_dropout <= 1.0:
        raise ValueError(f"{op} expects 0 <= max_dropout <= 1, got {max_dropout}")


def index_tensors(op: str, dev: torch.device, max_batch=None, **named) -> tuple:
    """The (B,) integer CUDA tensors that give each of a call's B entries its set member (and mode), 1 <= B (<=
    max_batch), on the set's device ``dev``, as the contiguous int64 tensors the kernels read.  Their values are not read
    back: the kernels turn a member index outside the set into an empty entry."""
    for name, t in named.items():
        if not isinstance(t, torch.Tensor):
            raise TypeError(f"{name} must be a torch.Tensor, got {type(t).__name__}")
        if t.dtype.is_floating_point or t.dtype.is_complex or t.dtype == torch.bool:
            raise TypeError(f"{name} must be an integer tensor, got {t.dtype}")
        if t.dim() != 1 or t.shape[0] < 1 or (max_batch is not None and t.shape[0] > max_batch):
            bound = "B >= 1" if max_batch is None else f"1 <= B <= {max_batch}"
            raise ValueError(f"{op} expects a (B,) {name} with {bound}, got {tuple(t.shape)}")
    (first, t0), *rest = named.items()
    for name, t in rest:
        if t.shape[0] != t0.shape[0]:
            raise ValueError(f"{op} expects one {name} per {first}, got {t.shape[0]} and {t0.shape[0]}")
    for name, t in named.items():
        if not t.is_cuda:
            raise RuntimeError(f"{name} must be a CUDA tensor: pointnet2_b200 has no CPU path (got device {t.device})")
        on_set_device(t, name, dev)
    return tuple(t.to(torch.int64).contiguous() for t in named.values())


def seed_args(seed, op: str, dev: torch.device):
    """(value, tensor or None) of a sampler's seed: a Python int as its 64 bits (signed), or a (1,) int64 CUDA tensor
    on the set's device ``dev``, which the kernels read on the device."""
    if isinstance(seed, torch.Tensor):
        if seed.dtype != torch.int64 or tuple(seed.shape) != (1,):
            raise TypeError(f"a tensor seed must be a (1,) int64 tensor, got {seed.dtype} {tuple(seed.shape)}")
        if not seed.is_cuda:
            raise RuntimeError(f"a tensor seed must be a CUDA tensor (got device {seed.device})")
        on_set_device(seed, "seed", dev)
        return 0, seed
    if isinstance(seed, bool) or not isinstance(seed, (int, np.integer)):
        raise TypeError(f"{op} expects an int or a (1,) int64 CUDA tensor seed, got {type(seed).__name__}")
    seed = int(seed)
    if not -2 ** 63 <= seed < 2 ** 64:
        raise ValueError(f"{op} expects a 64-bit seed, got {seed}")
    return (seed - 2 ** 64 if seed >= 2 ** 63 else seed), None


def same_device(*ts: torch.Tensor) -> None:
    dev = ts[0].device
    for t in ts[1:]:
        if t.device != dev:
            raise RuntimeError(f"all tensors must be on the same device ({dev} vs {t.device})")


def ptr(t) -> ctypes.c_void_p:
    return ctypes.c_void_p(t.data_ptr() if t is not None else 0)


def stream_ptr(device) -> ctypes.c_void_p:
    return ctypes.c_void_p(torch.cuda.current_stream(device).cuda_stream)


@contextmanager
def on_device(t: torch.Tensor):
    with torch.cuda.device(t.device):
        yield
