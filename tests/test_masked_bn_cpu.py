"""CPU tests of the fused masked batch norm + ReLU: the C entries are declared and refuse bad arguments before any launch,
and a CPU SharedMLP never reaches them (no device needed)."""
import ctypes
from unittest import mock

import pytest
import torch

from pointnet2_b200 import _lib, layers
from pointnet2_b200.layers import SharedMLP, row_mask

ENTRIES = ["pn2_masked_bn_workspace_bytes", "pn2_masked_bn_relu_forward_typed", "pn2_masked_bn_relu_backward_typed"]
P = ctypes.c_void_p
FAKE = P(256)  # never dereferenced: every call below is refused first


def test_entries_are_declared_and_loaded():
    lib = _lib.load()
    for name in ENTRIES:
        assert name in _lib.EXPORTED_SYMBOLS and hasattr(lib, name)
    for name in ENTRIES[1:]:
        assert _lib._SIGNATURES[name][1][0] is ctypes.c_int  # the dtype code comes first


def test_workspace_bytes_cover_the_partials():
    lib = _lib.load()
    assert lib.pn2_masked_bn_workspace_bytes(0, 128) == 0
    assert lib.pn2_masked_bn_workspace_bytes(10, 0) == 0
    # (rows, c) = (65536, 128): 256-row chunks, two floats per chunk and column
    assert lib.pn2_masked_bn_workspace_bytes(65536, 128) >= 2 * 4 * 256 * 128
    assert lib.pn2_masked_bn_workspace_bytes(65536, 128) <= lib.pn2_masked_bn_workspace_bytes(65537, 128)


def _fwd(lib, dtype=0, rows=64, c=8, x=FAKE, keep=FAKE, y=FAKE, sm=FAKE, si=FAKE, rm=None, rv=None, nbt=None,
         momentum=0.1, ws=FAKE, wsb=1 << 20):
    return lib.pn2_masked_bn_relu_forward_typed(dtype, rows, c, x, keep, None, None, 1e-5, momentum, nbt, rm, rv, y, sm, si,
                                                ws, wsb, None)


def _bwd(lib, dtype=0, rows=64, c=8, dy=FAKE, x=FAKE, y=FAKE, keep=FAKE, sm=FAKE, si=FAKE, dx=FAKE, ws=FAKE, wsb=1 << 20):
    return lib.pn2_masked_bn_relu_backward_typed(dtype, rows, c, dy, x, y, keep, None, sm, si, dx, None, None, ws, wsb, None)


@pytest.mark.parametrize("case", [
    dict(dtype=-1), dict(dtype=3), dict(c=0), dict(c=-4), dict(rows=-1),
    dict(x=None), dict(keep=None), dict(y=None), dict(sm=None), dict(si=None),
    dict(ws=None), dict(wsb=16),  # short workspace
    dict(rm=FAKE),  # running_mean without running_var
    dict(rm=FAKE, rv=FAKE, momentum=-1.0),  # cumulative average without num_batches_tracked
])
def test_forward_argument_errors_launch_nothing(case):
    lib = _lib.load()
    before = _lib.launch_count()
    assert _fwd(lib, **case) == 1, case
    assert _lib.launch_count() == before


@pytest.mark.parametrize("case", [
    dict(dtype=-1), dict(dtype=99), dict(c=0), dict(rows=-1),
    dict(dy=None), dict(x=None), dict(y=None), dict(keep=None), dict(sm=None), dict(si=None), dict(dx=None),
    dict(ws=None), dict(wsb=16),
])
def test_backward_argument_errors_launch_nothing(case):
    lib = _lib.load()
    before = _lib.launch_count()
    assert _bwd(lib, **case) == 1, case
    assert _lib.launch_count() == before


def test_empty_batch_is_a_no_op():
    lib = _lib.load()
    before = _lib.launch_count()
    assert _fwd(lib, rows=0, ws=None, wsb=0) == 0
    assert _bwd(lib, rows=0, ws=None, wsb=0) == 0
    assert _lib.launch_count() == before


def test_cpu_shared_mlp_never_calls_the_fused_entries():
    torch.manual_seed(0)
    m = SharedMLP(6, [16, 8]).train()
    t = torch.randn(2, 20, 6)
    mask = row_mask(torch.tensor([20, 7]), 20)
    with mock.patch.object(_lib, "load", side_effect=AssertionError("the library was loaded")):
        out = m(t, mask)
        out.sum().backward()
        assert not layers.fused_bn_applies(m.body[1], torch.zeros(4, 16))
    assert torch.equal(out[~mask], torch.zeros_like(out[~mask]))


def test_routing_predicate():
    bn = torch.nn.BatchNorm1d(4)
    meta = torch.empty(8, 4, device="meta")
    assert not layers.fused_bn_applies(bn, torch.zeros(8, 4))  # CPU
    assert not layers.fused_bn_applies(bn, meta)  # not CUDA

    def cuda_like(dtype=torch.float32, rows=8):
        # the predicate compares the module's device with x's: a CPU module stands for one on x's GPU
        return mock.Mock(is_cuda=True, dtype=dtype, shape=(rows, 4), device=torch.device("cpu"))

    assert layers.fused_bn_applies(bn.train(), cuda_like())
    assert layers.fused_bn_applies(bn.train(), cuda_like(torch.bfloat16))
    assert not layers.fused_bn_applies(bn.eval(), cuda_like())  # eval with running statistics: bn(x)
    assert layers.fused_bn_applies(torch.nn.BatchNorm1d(4, track_running_stats=False).eval(), cuda_like())
    assert layers.fused_bn_applies(torch.nn.BatchNorm1d(4, affine=False).train(), cuda_like())
    assert not layers.fused_bn_applies(bn.train(), cuda_like(torch.float64))
    assert not layers.fused_bn_applies(bn.train(), cuda_like(rows=0))
    # a module converted to 16 bits keeps the torch path: the kernels take float32 parameters and buffers
    for dtype in (torch.float16, torch.bfloat16):
        assert not layers.fused_bn_applies(torch.nn.BatchNorm1d(4).to(dtype).train(), cuda_like(dtype))
    other = mock.Mock(is_cuda=True, dtype=torch.float32, shape=(8, 4), device=torch.device("cuda:1"))
    assert not layers.fused_bn_applies(bn.train(), other)  # module on another device


def test_bn_followed_by_something_else_keeps_the_torch_path():
    """the fused op is BatchNorm1d + ReLU: a batch norm not followed by a ReLU is never fused"""
    bn = torch.nn.BatchNorm1d(4)
    x = mock.Mock(is_cuda=True, dtype=torch.float32, shape=(8, 4), device=torch.device("cpu"))
    assert layers._fuses_at([bn, torch.nn.ReLU()], 0, x)
    assert not layers._fuses_at([bn], 0, x)
    assert not layers._fuses_at([bn, torch.nn.Identity(), torch.nn.ReLU()], 0, x)
    assert not layers._fuses_at([torch.nn.Linear(4, 4), torch.nn.ReLU()], 0, x)
