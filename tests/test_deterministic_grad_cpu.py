"""CPU tests of the deterministic group_point / gather_point gradients: the workspace size, the argument checks of the
C entries (returned before any launch, so no device is needed) and which entry the autograd ops call, which follows
torch.are_deterministic_algorithms_enabled()."""
import ctypes
import os
import subprocess
import sys
from unittest import mock

import pytest
import torch

from pointnet2_b200 import _lib, pointnet_util, tf_grouping, tf_interpolate, tf_sampling

NEW = ["pn2_group_point_grad_det_workspace_bytes", "pn2_group_point_grad_det", "pn2_group_point_grad_det_typed",
       "pn2_gather_point_grad_det"]


def test_new_entries_are_declared_and_loaded():
    lib = _lib.load()
    for name in NEW:
        assert name in _lib.EXPORTED_SYMBOLS and hasattr(lib, name)


@pytest.mark.parametrize("b,n,m,s", [(1, 8, 2, 2), (32, 512, 128, 64), (16, 1024, 256, 32), (3, 100, 1, 1), (2, 7, 3000, 300)])
def test_workspace_size(b, n, m, s):
    lib = _lib.load()
    ne = m * s
    # offsets (b, n+1) + cursors (b, n) + entries (b, m*s) + the queue of lists longer than 256 entries, in ints
    want = 4 * (b * (n + 1) + b * n + b * ne + 1 + b * (ne // 257 + 1))
    assert lib.pn2_group_point_grad_det_workspace_bytes(b, n, m, s) == want
    # three_interpolate's gradient is the same structure with 3 entries per unknown point and the known points as targets
    assert lib.pn2_three_interpolate_grad_det_workspace_bytes(b, ne, n) == 4 * (b * (n + 1) + b * n + 3 * b * ne + 1 + b * (3 * ne // 257 + 1))
    for bad in [(0, n, m, s), (b, 0, m, s), (b, n, 0, s), (b, n, m, 0), (-1, n, m, s)]:
        assert lib.pn2_group_point_grad_det_workspace_bytes(*bad) == 0


def test_argument_errors_return_invalid_value_without_a_launch():
    lib = _lib.load()
    fake = ctypes.c_void_p(256)  # never dereferenced: every call below is refused first
    null = ctypes.c_void_p(0)
    ws = lib.pn2_group_point_grad_det_workspace_bytes(1, 8, 2, 2)
    before = _lib.launch_count()
    calls = [
        lib.pn2_group_point_grad_det(1, 8, 4, 2, 2, null, fake, fake, fake, ws, None),  # NULL grad_out
        lib.pn2_group_point_grad_det(1, 8, 4, 2, 2, fake, null, fake, fake, ws, None),  # NULL idx
        lib.pn2_group_point_grad_det(1, 8, 4, 2, 2, fake, fake, null, fake, ws, None),  # NULL grad_points
        lib.pn2_group_point_grad_det(1, 8, 4, 2, 2, fake, fake, fake, null, ws, None),  # NULL workspace
        lib.pn2_group_point_grad_det(1, 8, 4, 2, 2, fake, fake, fake, fake, ws - 1, None),  # workspace too small
        lib.pn2_group_point_grad_det(-1, 8, 4, 2, 2, fake, fake, fake, fake, ws, None),
        lib.pn2_group_point_grad_det(1, 0, 4, 2, 2, fake, fake, fake, fake, ws, None),
        lib.pn2_group_point_grad_det(1, 8, 4, 65536, 32768, fake, fake, fake, fake, 1 << 62, None),  # m*nsample = 2^31
        lib.pn2_group_point_grad_det_typed(3, 1, 8, 4, 2, 2, fake, fake, fake, fake, ws, None),  # unknown dtype
        lib.pn2_group_point_grad_det_typed(1, 1, 8, 4, 2, 2, fake, fake, fake, fake, ws - 1, None),
        lib.pn2_group_point_grad_det_typed(2, 1, 8, 4, 2, 2, fake, fake, null, fake, ws, None),
        lib.pn2_gather_point_grad_det(1, 8, 2, fake, fake, fake, fake, lib.pn2_group_point_grad_det_workspace_bytes(1, 8, 2, 1) - 1, None),
        lib.pn2_gather_point_grad_det(1, 8, 2, null, fake, fake, fake, 1 << 20, None),
    ]
    assert calls == [1] * len(calls)
    assert _lib.launch_count() == before
    # nothing to compute is not an error
    assert lib.pn2_group_point_grad_det(0, 8, 4, 2, 2, null, null, null, null, 0, None) == 0


class _Recorder:
    """stands in for the library: records the entry points called, returns 0 (success) from each"""

    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        def fn(*args):
            self.calls.append(name)
            return 64 if name.endswith("workspace_bytes") else 0
        return fn


@pytest.fixture
def recorder(monkeypatch):
    rec = _Recorder()
    monkeypatch.setattr(_lib, "load", lambda: rec)
    for mod in (tf_grouping, tf_sampling, tf_interpolate, pointnet_util):
        monkeypatch.setattr(mod, "on_device", lambda t: mock.MagicMock(), raising=False)
        monkeypatch.setattr(mod, "stream_ptr", lambda d: None, raising=False)
    yield rec
    torch.use_deterministic_algorithms(False)


@pytest.mark.parametrize("det", [False, True])
def test_routing_follows_torch_determinism(recorder, monkeypatch, det):
    torch.use_deterministic_algorithms(det)
    b, n, c, m, s = 2, 16, 5, 4, 3
    idx = torch.zeros((b, m, s), dtype=torch.int32)
    for dtype in (torch.float32, torch.bfloat16):
        recorder.calls.clear()
        tf_grouping.group_point_grad(torch.zeros((b, m, s, c), dtype=dtype), idx, (b, n, c))
        if det:
            assert recorder.calls == ["pn2_group_point_grad_det_workspace_bytes", "pn2_group_point_grad_det_typed"]
        else:
            assert recorder.calls == ["pn2_group_point_grad" if dtype == torch.float32 else "pn2_group_point_grad_typed"]
    ctx = mock.MagicMock(saved_tensors=(torch.zeros((b, m), dtype=torch.int32),), n=n)
    recorder.calls.clear()
    tf_sampling._GatherPoint.backward(ctx, torch.zeros((b, m, 3)))
    assert recorder.calls[-1] == ("pn2_gather_point_grad_det" if det else "pn2_gather_point_grad")
    # three_interpolate: the module flag off, torch's determinism decides
    monkeypatch.setattr(tf_interpolate, "DETERMINISTIC_GRAD", False)
    ctx = mock.MagicMock(saved_tensors=(torch.zeros((b, n, 3), dtype=torch.int32), torch.zeros((b, n, 3))), shape=(b, m, c),
                         dtype=torch.float32)
    recorder.calls.clear()
    tf_interpolate._ThreeInterpolate.backward(ctx, torch.zeros((b, n, c)))
    assert recorder.calls[-1] == ("pn2_three_interpolate_grad_det" if det else "pn2_three_interpolate_grad")


@pytest.mark.parametrize("needs_xyz", [False, True])
def test_group_concat_backward_scatters_coordinates_only_when_needed(recorder, needs_xyz):
    b, n, c, m, s = 2, 16, 5, 4, 3
    ctx = mock.MagicMock(saved_tensors=(torch.zeros((b, m, s), dtype=torch.int32),), meta=(b, n, c, m, s, False, True),
                         dtype=torch.float32, needs_input_grad=(needs_xyz, False, True, False, False))
    g_xyz, g_new_xyz, g_points, _, _ = pointnet_util._GroupConcat.backward(ctx, torch.zeros((b, m, s, c + 3)), None)
    assert recorder.calls == ["pn2_group_point_grad"] * (2 if needs_xyz else 1)
    assert (g_xyz is not None) == needs_xyz and g_new_xyz is None and g_points is not None


def test_demo_accepts_deterministic_flag():
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    out = subprocess.run([sys.executable, os.path.join(root, "tools", "train_ddp_demo.py"), "--help"], capture_output=True, text=True)
    assert out.returncode == 0 and "--deterministic" in out.stdout
