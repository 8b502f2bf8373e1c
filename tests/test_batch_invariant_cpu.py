"""layers.batch_invariant / fp_mlp / mlp_rows without a device: the routing with the mode on and off, the errors
raised instead of a fall-back to the torch layers, the argument errors that need no launch, the context manager, and
the agreement of the header, the ctypes table and the build list."""
import os
import re

import pytest
import torch
from torch import nn

import pointnet2_b200
from pointnet2_b200 import _build, _lib, layers, pointnet_util
from pointnet2_b200.layers import SharedMLP, batch_invariant, fp_mlp, is_batch_invariant, mlp_rows, sa_mlp_applies

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


class _OnCuda:
    """a stand-in for a CUDA tensor: the routing looks at the device, the dtype and the shape only"""
    is_cuda = True
    requires_grad = False

    def __init__(self, shape=(4, 6), dtype=torch.float32, device="cpu"):
        self.shape, self.dtype, self.device = torch.Size(shape), dtype, torch.device(device)


class _Entered(Exception):
    pass


@pytest.fixture
def kernels_raise(monkeypatch):
    """fp_mlp / mlp_rows replaced by stand-ins that record the call and raise _Entered"""
    calls = []

    def enter(name):
        def f(*a, **k):
            calls.append(name)
            raise _Entered(name)
        return f

    monkeypatch.setattr(layers, "fp_mlp", enter("fp_mlp"))
    monkeypatch.setattr(layers, "mlp_rows", enter("mlp_rows"))
    return calls


def test_exported_and_off_by_default():
    assert pointnet2_b200.batch_invariant is batch_invariant
    assert pointnet2_b200.is_batch_invariant is is_batch_invariant
    assert not is_batch_invariant()


def test_context_manager_restores_the_previous_state():
    with batch_invariant():
        assert is_batch_invariant()
        with batch_invariant(False):
            assert not is_batch_invariant()
            with batch_invariant(True):
                assert is_batch_invariant()
            assert not is_batch_invariant()
        assert is_batch_invariant()
    assert not is_batch_invariant()
    with pytest.raises(KeyError):
        with batch_invariant():
            raise KeyError("x")
    assert not is_batch_invariant()


def test_invariant_applies_truth_table():
    mlp = SharedMLP(6, [8, 16]).eval()
    x = _OnCuda()
    with torch.no_grad():
        assert not layers.invariant_applies(mlp, x)            # mode off
        with batch_invariant():
            assert layers.invariant_applies(mlp, x)
            assert not layers.invariant_applies(mlp, torch.zeros(4, 6))          # CPU
            assert not layers.invariant_applies(SharedMLP(6, [8]).train(), x)     # batch statistics
            assert layers.invariant_applies(SharedMLP(6, [8], bn=False).train(), x)  # no batch norm: nothing to decide
            nostats = SharedMLP(6, [8]).eval()
            nostats.body[1] = nn.BatchNorm1d(8, track_running_stats=False)
            assert not layers.invariant_applies(nostats, x)
    with batch_invariant():
        assert not layers.invariant_applies(mlp, x)            # grad mode on


def test_sa_mlp_applies_ignores_the_width_rule_in_the_mode():
    wide = SharedMLP(259, [256, 512, 1024]).eval()
    with torch.no_grad():
        assert not sa_mlp_applies(wide, _OnCuda())
        with batch_invariant():
            assert sa_mlp_applies(wide, _OnCuda())
            assert not sa_mlp_applies(SharedMLP(6, [8] * 5).eval(), _OnCuda())
            assert not sa_mlp_applies(wide.train(), _OnCuda())
        assert sa_mlp_applies(SharedMLP(6, [8]).eval(), _OnCuda())


def test_shared_mlp_routing(kernels_raise):
    mlp = SharedMLP(6, [8]).eval()
    t = torch.randn(5, 6)
    with torch.no_grad():
        mlp(t)                                          # mode off: the torch layers
        with batch_invariant():
            mlp(t)                                      # CPU tensor: the torch layers
            orig = SharedMLP.forward
            # a CUDA stand-in reaches the kernel call (the stand-in raises before anything touches its data)
            with pytest.raises(_Entered):
                orig(mlp, _OnCuda((5, 6)))
            with pytest.raises(_Entered):
                orig(mlp, _OnCuda((5, 6)), torch.ones(5, dtype=torch.bool))
    with batch_invariant():
        mlp(t)                                          # grad mode: torch
    assert kernels_raise == ["mlp_rows", "mlp_rows"]


def test_mode_off_never_enters_the_kernels(kernels_raise):
    mlp = SharedMLP(6, [8]).eval()
    with torch.no_grad():
        SharedMLP.forward(mlp, torch.randn(4, 6))
        assert pointnet_util._fp_mlp_route(mlp, _OnCuda((1, 4, 3)), None, _OnCuda((1, 2, 6)), None, True, None, None) is None
    assert kernels_raise == []


def test_fp_route():
    mlp = SharedMLP(6, [8]).eval()
    xyz1, p2 = _OnCuda((1, 4, 3)), _OnCuda((1, 2, 6))
    route = lambda m: pointnet_util._fp_mlp_route(m, xyz1, None, p2, None, True, None, None)  # noqa: E731
    with torch.no_grad():
        assert route(mlp) is None
        with batch_invariant():
            assert route(mlp) is mlp
            assert route(lambda t: t) is None                    # another callable routes its own SharedMLP calls
            assert route(SharedMLP(6, [8]).train()) is None
    with batch_invariant():
        assert route(mlp) is None                                # grad mode


def test_raises_instead_of_falling_back():
    """an eval-mode, no-grad CUDA layer in the mode that the kernels cannot take is a RuntimeError (the cases that need
    no device; a module converted to 16 bits is checked on the GPU)"""
    for mlp in (SharedMLP(6, [8] * 5).eval(), SharedMLP(6, [2048]).eval(), SharedMLP(1537, [8]).eval()):
        with pytest.raises(RuntimeError, match="batch_invariant"):
            layers._invariant_call(mlp_rows, torch.randn(3, mlp.in_channels), mlp)
    with pytest.raises(RuntimeError, match="batch_invariant"):
        layers._invariant_call(fp_mlp, torch.zeros(1, 4, 3), torch.zeros(1, 2, 3), None, torch.zeros(1, 2, 6),
                               SharedMLP(6, [8] * 5).eval())


def test_argument_errors_need_no_device():
    xyz1, xyz2, p2 = torch.zeros(1, 8, 3), torch.zeros(1, 4, 3), torch.zeros(1, 4, 6)
    t = torch.zeros(8, 6)
    with torch.no_grad():
        for call in (lambda m: fp_mlp(xyz1, xyz2, None, p2, m), lambda m: mlp_rows(t, m)):
            with pytest.raises(TypeError, match="SharedMLP"):
                call(nn.Linear(6, 4))
            with pytest.raises(ValueError, match="training mode"):
                call(SharedMLP(6, [4]).train())
            nostats = SharedMLP(6, [4]).eval()
            nostats.body[1] = nn.BatchNorm1d(4, track_running_stats=False)
            with pytest.raises(ValueError, match="running statistics"):
                call(nostats)
            with pytest.raises(ValueError, match="at most 4 layers"):
                call(SharedMLP(6, [4] * 5).eval())
            with pytest.raises(ValueError, match="at most 4 layers of at most 1024"):
                call(SharedMLP(6, [2048]).eval())
            with pytest.raises(RuntimeError, match="no CPU path"):
                call(SharedMLP(6, [4]).eval())
        with pytest.raises(ValueError, match="1536 inputs"):
            mlp_rows(torch.zeros(2, 1537), SharedMLP(1537, [4]).eval())
    with pytest.raises(RuntimeError, match="no_grad"):
        mlp_rows(t, SharedMLP(6, [4]).eval())
    with pytest.raises(RuntimeError, match="no_grad"):
        fp_mlp(xyz1, xyz2, None, p2, SharedMLP(6, [4]).eval())


def _proto(text, name):
    proto = re.search(r"\b" + name + r"\s*\((.*?)\)\s*;", text, flags=re.S).group(1)
    return [a.strip() for a in proto.split(",")]


def test_header_ctypes_and_sources_agree():
    assert "fp_mlp.cu" in _build.SOURCES and os.path.exists(os.path.join(_build.CSRC, "fp_mlp.cu"))
    assert any(h.endswith("mlp_tile.cuh") for h in _build.HEADERS)
    text = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "pn2_api.h")).read(), flags=re.S)
    kinds = {"int": _lib.c_int, "long long": _lib.c_longlong, "size_t": _lib.c_size_t}
    for name in ("pn2_fp_mlp_typed", "pn2_mlp_rows_typed", "pn2_fp_mlp_workspace_bytes"):
        args = _proto(text, name)
        res, argtypes = _lib._SIGNATURES[name]
        assert len(args) == len(argtypes), name
        for a, t in zip(args, argtypes):
            want = _lib._P if "*" in a else kinds[a.rsplit(" ", 1)[0]]
            assert t is want, (name, a, t)
    lib = _lib.load()
    null = _lib._P(0)
    assert lib.pn2_api_version() == 2
    assert lib.pn2_fp_mlp_workspace_bytes(0, 5) == 0 and lib.pn2_fp_mlp_workspace_bytes(2, 100) >= 2 * 2 * 100 * 3 * 4
    before = _lib.launch_count()
    fp = lambda dtype, nl, c2=4: lib.pn2_fp_mlp_typed(dtype, 1, 8, 4, c2, 0, null, null, null, null, null, nl, null, null,  # noqa: E731
                                                      null, null, null, null, null, null, null, null, 8, null, 0, null)
    rows = lambda dtype, nl, c=6: lib.pn2_mlp_rows_typed(dtype, 8, c, null, null, nl, null, null, null, null, null,  # noqa: E731
                                                         null, null, null, null, null, 8, null)
    assert fp(0, 1) == 1 and fp(7, 1) == 1 and fp(0, 5) == 1 and fp(0, 1, c2=1537) == 1
    assert rows(0, 1) == 1 and rows(7, 1) == 1 and rows(0, 5) == 1 and rows(0, 1, c=1537) == 1
    # widths over the limit, with every array present
    import ctypes
    w = (ctypes.c_int * 1)(2048)
    ptrs = (ctypes.c_void_p * 1)(8)
    relu = (ctypes.c_int * 1)(1)
    assert lib.pn2_mlp_rows_typed(0, 8, 6, ptrs[0], null, 1, w, ptrs, ptrs, null, null, null, null, null, relu, ptrs[0],
                                  2048, null) == 1
    assert _lib.launch_count() == before
