"""CPU tests of the variable-size-cloud surface: the `lengths` keyword on every op that takes it, the host-side
validation of lengths, and the ValueError where lengths are not supported (kNN grouping, group_all)."""
import inspect

import numpy as np
import pytest
import torch

from pointnet2_b200 import _lib, nets, pointnet_util, sa_layer, tf_grouping, tf_sampling
from pointnet2_b200._tensor import device_lengths


def test_lengths_is_a_keyword_after_the_reference_arguments():
    for fn, positional in ((tf_sampling.farthest_point_sample, ["npoint", "inp"]),
                           (tf_sampling.farthest_point_sample_and_gather, ["npoint", "inp"]),
                           (tf_grouping.query_ball_point, ["radius", "nsample", "xyz1", "xyz2"]),
                           (sa_layer.sample_group, ["npoint", "radius", "nsample", "xyz", "center", "want_grouped"]),
                           (sa_layer.sample_group_msg, ["npoint", "radius_list", "nsample_list", "xyz", "center", "want_grouped"])):
        params = inspect.signature(fn).parameters
        assert list(params)[:len(positional)] == positional, fn.__name__
        assert params["lengths"].kind == inspect.Parameter.KEYWORD_ONLY and params["lengths"].default is None, fn.__name__
    for fn in (pointnet_util.sample_and_group, pointnet_util.pointnet_sa_module, pointnet_util.pointnet_sa_module_msg,
               nets.PointNet2ClsSSG.forward, nets.PointNet2ClsMSG.forward):
        assert inspect.signature(fn).parameters["lengths"].default is None, fn.__qualname__


def test_ragged_entries_are_in_the_signature_table():
    for name in ("pn2_fps_gather_ragged", "pn2_query_ball_point_ragged", "pn2_sa_layer_device_ragged",
                 "pn2_sa_layer_msg_device_ragged"):
        assert name in _lib.EXPORTED_SYMBOLS
        assert hasattr(_lib.load(), name)


def test_host_lengths_are_checked_and_converted():
    cpu = torch.device("cpu")
    assert device_lengths(None, 3, 10, cpu, "op") is None
    for ok in ([1, 10, 5], (1, 10, 5), np.array([1, 10, 5], np.int16), torch.tensor([1, 10, 5])):
        got = device_lengths(ok, 3, 10, cpu, "op")
        assert got.dtype == torch.int32 and got.tolist() == [1, 10, 5]
    for bad in ([0, 1, 1], [1, 11, 1], [-2, 1, 1], [1, 1], [[1, 1, 1]], torch.tensor([1, 1, 1, 1]), np.zeros((3, 1), np.int32)):
        with pytest.raises(ValueError):
            device_lengths(bad, 3, 10, cpu, "op")
    for bad in ([1.0, 2.0, 3.0], torch.tensor([1.0, 2.0, 3.0]), np.array([True, True, True])):
        with pytest.raises(TypeError):
            device_lengths(bad, 3, 10, cpu, "op")
    assert device_lengths([], 0, 10, cpu, "op").numel() == 0


def test_lengths_are_refused_where_unsupported():
    x = torch.zeros(2, 16, 3)
    with pytest.raises(ValueError, match="knn"):
        pointnet_util.sample_and_group(4, 0.2, 4, x, None, knn=True, lengths=[16, 8])
    with pytest.raises(ValueError, match="group_all"):
        pointnet_util.pointnet_sa_module(x, None, None, None, None, group_all=True, lengths=[16, 8])
