"""Point-cloud rendering on the GPU: the reference's viewer (utils/show3d_balls.py showpoints driving
utils/render_balls_so.cpp render_ball) on a padded ragged batch of clouds and any number of views.

    img = render_balls(ixyz, colors, 800, 800, 10)          # (B, H, W, 3) uint8, render_ball on every cloud
    ixyz = project_points(xyz, xangle=[0.0, 0.5])           # (B, V, N, 3) int32, showpoints' view transform
    img = show_points(xyz, palette[labels], ballradius=8)   # (B, V, 800, 800, 3) uint8, the non-interactive viewer

Image b of render_balls is bit for bit what render_ball writes for cloud b alone on a canvas filled with the background
(csrc/render.cu, DESIGN.md §6.16).  Per-cloud ``lengths`` are clamped to [0, N] on the device and never read back, so
every call is asynchronous and can be captured in a CUDA graph; a cloud of length 0 renders as background.
"""
from __future__ import annotations

import numpy as np
import torch

from . import _lib
from ._tensor import as_int as _int, device_lengths0 as _lengths, on_device, ptr, require_cuda, stream_ptr

MAX_RADIUS = 4096     # pn2_api.h: r <= 4096
MAX_IMAGES = 65535    # images per call (B, or B * V for show_points)


def _background(background, op: str) -> np.ndarray:
    bg = np.asarray(background)
    if bg.shape != (3,) or not np.issubdtype(bg.dtype, np.integer) or bg.min() < 0 or bg.max() > 255:
        raise ValueError(f"{op} expects a background of 3 integers in [0, 255], got {background!r}")
    return np.ascontiguousarray(bg.astype(np.uint8))


def render_balls(ixyz: torch.Tensor, colors, height: int, width: int, radius: int, background=(0, 0, 0), *,
                 lengths=None) -> torch.Tensor:
    """render_ball on each cloud of a batch.  ixyz (B, N, 3) int32 CUDA (x indexes rows, y columns, z is depth);
    colors (B, N, 3) float32 = (c0, c1, c2) per point, or None for 255 everywhere; lengths (B,) or None.  Returns
    (B, height, width, 3) uint8: channel 0 from c2, 1 from c0, 2 from c1, shaded by the ball's height and the point's
    depth, and ``background`` where no ball reaches.  Real points need |x|, |y|, |z| <= 2^30."""
    op = "render_balls"
    ixyz = require_cuda(ixyz, "ixyz", torch.int32)
    if ixyz.dim() != 3 or ixyz.shape[2] != 3:
        raise ValueError(f"{op} expects ixyz of shape (B, N, 3), got {tuple(ixyz.shape)}")
    b, n, _ = ixyz.shape
    height, width, radius = _int(height, "height", op), _int(width, "width", op), _int(radius, "radius", op)
    if height < 1 or width < 1 or height * width >= 2 ** 31:
        raise ValueError(f"{op} expects height, width >= 1 and height * width < 2^31, got {height} x {width}")
    if radius > MAX_RADIUS:
        raise ValueError(f"{op} expects radius <= {MAX_RADIUS}, got {radius}")
    if b > MAX_IMAGES:
        raise ValueError(f"{op} renders at most {MAX_IMAGES} images per call, got {b}")
    if n >= 2 ** 30 // 3:
        raise ValueError(f"{op} expects N < 2^30 / 3, got {n}")
    if colors is not None:
        colors = require_cuda(colors, "colors", torch.float32)
        if tuple(colors.shape) != (b, n, 3):
            raise ValueError(f"{op} expects colors of shape {(b, n, 3)}, got {tuple(colors.shape)}")
        if colors.device != ixyz.device:
            raise RuntimeError(f"all tensors must be on the same device ({ixyz.device} vs {colors.device})")
    bg = _background(background, op)
    lens = _lengths(lengths, b, n, ixyz.device, op)
    out = torch.empty((b, height, width, 3), dtype=torch.uint8, device=ixyz.device)
    if b == 0:
        return out
    lib = _lib.load()
    with on_device(ixyz):
        wsb = int(lib.pn2_render_balls_workspace_bytes(b, height, width))
        ws = torch.empty(wsb, dtype=torch.uint8, device=ixyz.device)
        rc = lib.pn2_render_balls(b, n, height, width, ptr(ixyz), ptr(colors), ptr(lens), radius,
                                  bg.ctypes.data_as(_lib.c_void_p), ptr(ws), wsb, ptr(out), stream_ptr(ixyz.device))
    _lib.check(rc, "pn2_render_balls")
    return out


def _views(xangle, yangle, zoom) -> np.ndarray:
    """(V, 3, 3) float64: showpoints' eye(3).dot(Rx(xangle)).dot(Ry(yangle)) * zoom for every view, broadcasting
    scalars and length-1 sequences against length-V ones."""
    xa, ya, zm = (np.atleast_1d(np.asarray(a, np.float64)) for a in (xangle, yangle, zoom))
    for name, a in (("xangle", xa), ("yangle", ya), ("zoom", zm)):
        if a.ndim != 1 or a.size < 1:
            raise ValueError(f"project_points expects a scalar or a 1-D sequence for {name}, got shape {a.shape}")
    v = max(xa.size, ya.size, zm.size)
    if any(a.size not in (1, v) for a in (xa, ya, zm)):
        raise ValueError(f"project_points expects xangle, yangle and zoom of one length V or 1, got "
                         f"{xa.size}, {ya.size}, {zm.size}")
    xa, ya, zm = (np.broadcast_to(a, (v,)) for a in (xa, ya, zm))
    rots = np.empty((v, 3, 3), np.float64)
    for k in range(v):
        rot = np.eye(3)
        rot = rot.dot(np.array([[1.0, 0.0, 0.0],
                                [0.0, np.cos(xa[k]), -np.sin(xa[k])],
                                [0.0, np.sin(xa[k]), np.cos(xa[k])]]))
        rot = rot.dot(np.array([[np.cos(ya[k]), 0.0, -np.sin(ya[k])],
                                [0.0, 1.0, 0.0],
                                [np.sin(ya[k]), 0.0, np.cos(ya[k])]]))
        rots[k] = rot * zm[k]
    return rots


def project_points(xyz: torch.Tensor, size: int = 800, xangle=0.0, yangle=0.0, zoom=1.0, *,
                   lengths=None) -> torch.Tensor:
    """showpoints' view transform (show3d_balls.py:27-29, 52-74) with the angles given directly.  xyz (B, N, 3)
    float32 or float64 CUDA, taken as float64; every cloud is centred on the mean of its real points and scaled by
    (radius * 2.2) / size, radius the largest distance from that mean; then p Rx(xangle) Ry(yangle) zoom + (size/2,
    size/2, 0), truncated toward zero.  xangle, yangle, zoom: scalars or 1-D sequences of one length V.  Returns (B, V,
    N, 3) int32; padding rows are 0, coordinates are clamped to +-2^30 and a cloud whose points coincide maps to
    (size/2, size/2, 0)."""
    op = "project_points"
    xyz = require_cuda(xyz, "xyz", (torch.float64, torch.float32))
    if xyz.dim() != 3 or xyz.shape[2] != 3:
        raise ValueError(f"{op} expects xyz of shape (B, N, 3), got {tuple(xyz.shape)}")
    size = _int(size, "size", op)
    if size < 1:
        raise ValueError(f"{op} expects size >= 1, got {size}")
    b, n, _ = xyz.shape
    if b > MAX_IMAGES or n >= 2 ** 30 // 3:
        raise ValueError(f"{op} expects B <= {MAX_IMAGES} and N < 2^30 / 3, got {tuple(xyz.shape)}")
    rots = np.ascontiguousarray(_views(xangle, yangle, zoom))
    v = rots.shape[0]
    lens = _lengths(lengths, b, n, xyz.device, op)
    out = torch.empty((b, v, n, 3), dtype=torch.int32, device=xyz.device)
    if b == 0 or n == 0:
        return out.zero_()
    x64 = xyz.to(torch.float64).contiguous()
    ws = torch.empty((b, 4), dtype=torch.float64, device=xyz.device)
    lib = _lib.load()
    with on_device(xyz):
        rc = lib.pn2_project_points(b, n, v, ptr(x64), ptr(lens), rots.ctypes.data_as(_lib.c_void_p), size, ptr(ws),
                                    ws.numel() * 8, ptr(out), stream_ptr(xyz.device))
    _lib.check(rc, "pn2_project_points")
    return out


def magnify_blue_channel(img: torch.Tensor, level: int) -> torch.Tensor:
    """showpoints' magnifyBlue (show3d_balls.py:88-94) on channel 0 of (..., H, W, 3) uint8 images, in place: level 1
    takes the max with the pixel above and the pixel to the left, level 2 also with the ones below and to the right,
    each step on the previous step's result and with wrap-around edges (np.roll).  Returns img."""
    if level <= 0:
        return img
    c = img[..., 0]
    h, w = img.dim() - 3, img.dim() - 2
    c.copy_(torch.maximum(c, torch.roll(c, 1, dims=h)))
    if level >= 2:
        c.copy_(torch.maximum(c, torch.roll(c, -1, dims=h)))
    c.copy_(torch.maximum(c, torch.roll(c, 1, dims=w)))
    if level >= 2:
        c.copy_(torch.maximum(c, torch.roll(c, -1, dims=w)))
    return img


def show_points(xyz: torch.Tensor, colors=None, *, size: int = 800, xangle=0.0, yangle=0.0, zoom=1.0,
                ballradius: int = 10, background=(0, 0, 0), normalizecolor: bool = True, magnify_blue: int = 0,
                lengths=None) -> torch.Tensor:
    """The non-interactive showpoints (show3d_balls.py:25-94): every cloud of xyz (B, N, 3) from V views (see
    project_points) as (B, V, size, size, 3) uint8.  colors (B, N, 3) = (c0, c1, c2) per point, any float dtype, or
    None for white; normalizecolor divides each cloud's channel by (max + 1e-14) / 255 over its real points in float64
    and rounds once to float32.  For label colours pass ``palette[labels]``."""
    op = "show_points"
    ixyz = project_points(xyz, size, xangle, yangle, zoom, lengths=lengths)
    b, v, n, _ = ixyz.shape
    if b * v > MAX_IMAGES:
        raise ValueError(f"{op} renders at most {MAX_IMAGES} images per call, got {b} clouds x {v} views")
    lens = _lengths(lengths, b, n, xyz.device, op)
    if colors is not None:
        if not isinstance(colors, torch.Tensor) or not colors.dtype.is_floating_point:
            raise TypeError(f"{op} expects a floating-point colors tensor")
        if tuple(colors.shape) != (b, n, 3) or colors.device != xyz.device:
            raise ValueError(f"{op} expects colors of shape {(b, n, 3)} on {xyz.device}, got {tuple(colors.shape)} "
                             f"on {colors.device}")
        c = colors.to(torch.float64)
        if normalizecolor:
            rows = torch.arange(n, device=c.device)
            real = (rows[None, :] < lens[:, None])[..., None] if lens is not None else torch.ones_like(c, dtype=torch.bool)
            cmax = torch.where(real, c, torch.full_like(c, -torch.inf)).amax(dim=1, keepdim=True)
            c = c / ((cmax + 1e-14) / 255.0)
        colors = c.to(torch.float32)
        if v > 1:
            colors = colors[:, None].expand(b, v, n, 3).reshape(b * v, n, 3)
    # colors None: 255, which normalisation leaves at 255
    img = render_balls(ixyz.reshape(b * v, n, 3), colors, size, size, ballradius, background,
                       lengths=None if lens is None else lens.repeat_interleave(v))
    magnify_blue_channel(img, magnify_blue)
    return img.reshape(b, v, size, size, 3)
