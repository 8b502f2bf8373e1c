"""CPU tests of the 16-bit feature surface: which dtypes the ops accept, and the typed C entry points' argument checks
(no device needed: errors are returned before any launch)."""
import ctypes

import pytest
import torch

import pointnet2_b200
from pointnet2_b200 import _lib
from pointnet2_b200.pointnet_util import group_and_concat
from pointnet2_b200.tf_interpolate import fp_interpolate_concat, three_nn_interpolate

TYPED = ["pn2_group_point_typed", "pn2_group_point_grad_typed", "pn2_group_concat_typed", "pn2_three_interpolate_typed",
         "pn2_three_interpolate_grad_det_typed", "pn2_three_nn_interpolate_typed", "pn2_fp_interpolate_concat_typed"]


def test_typed_entries_are_declared_and_loaded():
    lib = _lib.load()
    for name in TYPED:
        assert name in _lib.EXPORTED_SYMBOLS and hasattr(lib, name)
        assert _lib._SIGNATURES[name][1][0] is ctypes.c_int  # the dtype code comes first


def _calls(dtype, null):
    """one call per typed entry with non-empty sizes; every tensor argument is `null`"""
    P = null
    return [
        ("pn2_group_point_typed", (dtype, 1, 8, 4, 2, 2, P, P, P, None)),
        ("pn2_group_point_grad_typed", (dtype, 1, 8, 4, 2, 2, P, P, P, P, None)),
        ("pn2_group_concat_typed", (dtype, 1, 8, 4, 2, 2, P, P, P, P, 1, P, P, None)),
        ("pn2_three_interpolate_typed", (dtype, 1, 8, 4, 2, P, P, P, P, None)),
        ("pn2_three_interpolate_grad_det_typed", (dtype, 1, 2, 4, 8, P, P, P, P, P, 1 << 20, None)),
        ("pn2_three_nn_interpolate_typed", (dtype, 1, 2, 8, 4, P, P, P, P, P, P, P, None)),
        ("pn2_fp_interpolate_concat_typed", (dtype, 1, 2, 8, 4, 4, P, P, P, P, P, None)),
    ]


@pytest.mark.parametrize("dtype", [-1, 3, 99])
def test_unknown_dtype_code_is_an_argument_error(dtype):
    lib = _lib.load()
    before = _lib.launch_count()
    for name, args in _calls(dtype, ctypes.c_void_p(0)):
        assert getattr(lib, name)(*args) == 1, name
    assert _lib.launch_count() == before


@pytest.mark.parametrize("dtype", [0, 1, 2])
def test_null_tensors_are_an_argument_error(dtype):
    lib = _lib.load()
    before = _lib.launch_count()
    for name, args in _calls(dtype, ctypes.c_void_p(0)):
        assert getattr(lib, name)(*args) == 1, name
    assert _lib.launch_count() == before


def test_16bit_accumulator_is_required():
    """a 16-bit group_point gradient needs the float32 accumulator; float32 does not"""
    lib = _lib.load()
    before = _lib.launch_count()
    fake = ctypes.c_void_p(256)  # never dereferenced: the call is refused first
    assert lib.pn2_group_point_grad_typed(1, 1, 8, 4, 2, 2, fake, fake, fake, None, None) == 1
    assert lib.pn2_group_point_grad_typed(2, 1, 8, 4, 2, 2, fake, fake, fake, None, None) == 1
    assert _lib.launch_count() == before


def test_feature_dtypes_and_coordinate_dtypes():
    """float64 / integer features and 16-bit coordinates raise TypeError before the device is looked at"""
    i3 = torch.zeros(1, 4, 3, dtype=torch.int32)
    w = torch.zeros(1, 4, 3)
    for bad in (torch.float64, torch.int32):
        with pytest.raises(TypeError, match="points must be"):
            pointnet2_b200.group_point(torch.zeros(1, 8, 5, dtype=bad), i3)
        with pytest.raises(TypeError, match="points must be"):
            pointnet2_b200.three_interpolate(torch.zeros(1, 8, 5, dtype=bad), i3, w)
    for half in (torch.float16, torch.bfloat16):
        x = torch.zeros(1, 8, 3, dtype=half)
        with pytest.raises(TypeError):
            pointnet2_b200.farthest_point_sample(4, x)
        with pytest.raises(TypeError, match="xyz1"):
            pointnet2_b200.query_ball_point(0.1, 4, x, x)
        with pytest.raises(TypeError, match="xyz1"):
            pointnet2_b200.three_nn(x, x)
        with pytest.raises(TypeError, match="xyz"):
            group_and_concat(x, x, torch.zeros(1, 8, 5, dtype=half), i3)
        with pytest.raises(TypeError, match="xyz1"):
            three_nn_interpolate(x, x, torch.zeros(1, 8, 5, dtype=half))
    # 16-bit features pass the dtype check and reach the device check
    with pytest.raises(RuntimeError, match="no CPU path"):
        pointnet2_b200.group_point(torch.zeros(1, 8, 5, dtype=torch.bfloat16), i3)


def test_fp_interpolate_concat_refuses_mixed_feature_dtypes():
    x = torch.zeros(1, 8, 3)
    with pytest.raises(TypeError, match="same dtype"):
        fp_interpolate_concat(x, x, torch.zeros(1, 8, 4, dtype=torch.bfloat16), torch.zeros(1, 8, 4))
    with pytest.raises(TypeError, match="same dtype"):
        fp_interpolate_concat(x, x, torch.zeros(1, 8, 4, dtype=torch.float16), torch.zeros(1, 8, 4, dtype=torch.bfloat16))


def test_demo_accepts_amp_flag():
    import os
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    out = subprocess.run([sys.executable, os.path.join(root, "tools", "train_ddp_demo.py"), "--help"], capture_output=True, text=True)
    assert out.returncode == 0 and "--amp" in out.stdout and "bf16" in out.stdout
