"""Argument checking shared by the op wrappers.

Mirrors the reference OpKernels' OP_REQUIRES checks (tf_ops/sampling/tf_sampling.cpp:99,105,131,135;
tf_ops/grouping/tf_grouping.cpp:71-84,90,96; tf_ops/3d_interpolation/tf_interpolate.cpp:163-168,
197-206): shape / attribute violations raise ValueError (TensorFlow: InvalidArgument), wrong dtypes
raise TypeError.  Tensors must live on a CUDA device: there is no CPU path.
"""
from __future__ import annotations

import ctypes
from contextlib import contextmanager

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
    if isinstance(lengths, torch.Tensor):
        if lengths.dtype not in _INT_DTYPES:
            raise TypeError(f"{op} expects integer lengths, got {lengths.dtype}")
        host = lengths.detach().to(torch.int64)
    else:
        import numpy as np
        arr = np.asarray(lengths)
        if arr.size and not np.issubdtype(arr.dtype, np.integer):
            raise TypeError(f"{op} expects integer lengths, got {arr.dtype}")
        host = torch.from_numpy(arr.astype(np.int64).reshape(arr.shape))
    if tuple(host.shape) != (b,):
        raise ValueError(f"{op} expects (batch_size,) lengths shape ({b},), got {tuple(host.shape)}")
    if b and (int(host.min()) < 1 or int(host.max()) > n):
        raise ValueError(f"{op} expects 1 <= lengths <= {n} (the padded number of points), got {host.tolist()}")
    return host.to(torch.int32).to(device)


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
