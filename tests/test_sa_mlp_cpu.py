"""layers.sa_mlp_applies / layers.sa_mlp_max without a device: when the set-abstraction modules take the kernel, the
argument errors that need no launch, and the agreement of the header, the ctypes table and the build list."""
import os
import re

import pytest
import torch
from torch import nn

from pointnet2_b200 import _build, _lib, layers
from pointnet2_b200.layers import SharedMLP, sa_mlp_applies, sa_mlp_max

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


class _OnCuda:
    """a stand-in for a CUDA tensor: sa_mlp_applies looks at the device and the dtype only"""
    is_cuda = True
    requires_grad = False

    def __init__(self, dtype=torch.float32, device="cpu"):
        self.dtype, self.device = dtype, torch.device(device)


def test_applies_truth_table():
    mlp = SharedMLP(6, [8, 16]).eval()
    xyz = _OnCuda()
    with torch.no_grad():
        assert sa_mlp_applies(mlp, xyz)                      # (parameters on xyz's "device")
        assert sa_mlp_applies(mlp, xyz, _OnCuda(torch.bfloat16))
        assert not sa_mlp_applies(mlp, xyz, pooling="avg")
        assert not sa_mlp_applies(mlp, xyz, _OnCuda(torch.float64))
        assert not sa_mlp_applies(mlp, torch.zeros(1, 4, 3))  # CPU tensors
        assert not sa_mlp_applies(lambda t: t, xyz)           # not a SharedMLP
        assert not sa_mlp_applies(nn.Sequential(nn.Linear(6, 8)), xyz)
        assert not sa_mlp_applies(SharedMLP(6, [8] * 5).eval(), xyz)
        assert sa_mlp_applies(SharedMLP(6, [8] * 4).eval(), xyz)
        assert not sa_mlp_applies(SharedMLP(6, [2048]).eval(), xyz)
        assert sa_mlp_applies(SharedMLP(1027, [256]).eval(), xyz)
        assert sa_mlp_applies(SharedMLP(259, [256, 256, 512]).eval(), xyz)
        assert not sa_mlp_applies(SharedMLP(259, [256, 512, 1024]).eval(), xyz)  # cuBLAS is faster: layers.SA_MLP_MAX_MACS
        assert not sa_mlp_applies(SharedMLP(1028, [8]).eval(), xyz)
        assert not sa_mlp_applies(SharedMLP(6, [8]).eval().to(torch.bfloat16), xyz)
        assert not sa_mlp_applies(SharedMLP(6, [8]).train(), xyz)
        assert sa_mlp_applies(SharedMLP(6, [8], bn=False).train(), xyz)  # no batch norm: nothing depends on the mode
        nostats = SharedMLP(6, [8]).eval()
        nostats.body[1] = nn.BatchNorm1d(8, track_running_stats=False)
        assert not sa_mlp_applies(nostats, xyz)
    assert not sa_mlp_applies(mlp, xyz)                      # grad mode on


def test_argument_errors_need_no_device():
    x = torch.zeros(1, 8, 3)
    idx = torch.zeros(1, 2, 4, dtype=torch.int32)
    with torch.no_grad():
        with pytest.raises(TypeError, match="SharedMLP"):
            sa_mlp_max(x, x[:, :2], None, idx, nn.Linear(3, 4))
        with pytest.raises(ValueError, match="training mode"):
            sa_mlp_max(x, x[:, :2], None, idx, SharedMLP(3, [4]).train())
        nostats = SharedMLP(3, [4]).eval()
        nostats.body[1] = nn.BatchNorm1d(4, track_running_stats=False)
        with pytest.raises(ValueError, match="running statistics"):
            sa_mlp_max(x, x[:, :2], None, idx, nostats)
        with pytest.raises(ValueError, match="at most 4 layers"):
            sa_mlp_max(x, x[:, :2], None, idx, SharedMLP(3, [4] * 5).eval())
        with pytest.raises(ValueError, match="at most 4 layers of at most 1024"):
            sa_mlp_max(x, x[:, :2], None, idx, SharedMLP(3, [2048]).eval())
        with pytest.raises(RuntimeError, match="no CPU path"):
            sa_mlp_max(x, x[:, :2], None, idx, SharedMLP(3, [4]).eval())
        with pytest.raises(TypeError):
            sa_mlp_max(x.double(), x[:, :2], None, idx, SharedMLP(3, [4]).eval())
    with pytest.raises(RuntimeError, match="no_grad"):
        sa_mlp_max(x, x[:, :2], None, idx, SharedMLP(3, [4]).eval())


def test_stack_parsing():
    m = SharedMLP(5, [7, 9], last_activation=False)
    (l0, b0, r0), (l1, b1, r1) = layers._mlp_stack(m)
    assert (l0.out_features, isinstance(b0, nn.BatchNorm1d), r0) == (7, True, True)
    assert (l1.out_features, b1, r1) == (9, None, False)
    m.body.append(nn.Dropout())
    assert layers._mlp_stack(m) is None


def test_header_ctypes_and_sources_agree():
    assert "sa_mlp.cu" in _build.SOURCES and os.path.exists(os.path.join(_build.CSRC, "sa_mlp.cu"))
    text = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "pn2_api.h")).read(), flags=re.S)
    proto = re.search(r"int\s+pn2_sa_mlp_max_typed\s*\((.*?)\)\s*;", text, flags=re.S).group(1)
    args = [a.strip() for a in proto.split(",")]
    res, argtypes = _lib._SIGNATURES["pn2_sa_mlp_max_typed"]
    assert len(args) == len(argtypes)
    for a, t in zip(args, argtypes):
        want = _lib._P if "*" in a else {"int": _lib.c_int, "long long": _lib.c_longlong}[a.rsplit(" ", 1)[0]]
        assert t is want, (a, t)
    lib = _lib.load()
    null = _lib._P(0)
    before = _lib.launch_count()
    call = lambda dtype, nl: lib.pn2_sa_mlp_max_typed(dtype, 1, 8, 0, 2, 4, null, null, null, null, 1, 1, nl, null, null, null,
                                                      null, null, null, null, null, null, null, 4, null)
    assert call(0, 1) == 1 and call(7, 1) == 1 and call(0, 5) == 1  # null arrays, unknown dtype, five layers
    assert _lib.launch_count() == before
