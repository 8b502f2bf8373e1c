"""GPU tests of voxel and pillar grouping (csrc/voxel.cu, pointnet2_b200.pc_util): idx, count and grouped bit for bit
against tests/voxel_oracle.py on seeded batches (uniform, clustered and duplicate-heavy clouds, a cell of more than
16384 rows, NaN padding with lengths 0, 1 and N, every grid and nsample size class), the reference's own outputs
(tests/golden/pcutil_*.npz) through the three pc_util wrappers, run-to-run bits, a device seed replayed through a CUDA
graph, and group_point on the returned idx."""
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import voxel_oracle as VO  # noqa: E402

from pointnet2_b200 import _lib, group_point, pc_util  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _check(xyz, vsize, radius=1.0, nsample=128, seed=0, dims=3, lengths=None, dev_lengths=None):
    """voxel_group on the GPU against the oracle, every output bit for bit; returns the device outputs."""
    x = torch.from_numpy(xyz).to(DEV)
    lens = dev_lengths if dev_lengths is not None else lengths
    idx, count, grouped = pc_util.voxel_group(x, vsize, radius, nsample, seed, dims=dims, lengths=lens)
    w_idx, w_count, w_grouped = VO.oracle_voxel_group(xyz, vsize, radius, nsample, seed, dims, lengths)
    np.testing.assert_array_equal(count.cpu().numpy(), w_count)
    np.testing.assert_array_equal(idx.cpu().numpy(), w_idx)
    g = grouped.cpu().numpy()
    assert np.array_equal(np.isnan(g), np.isnan(w_grouped))
    np.testing.assert_array_equal(np.nan_to_num(g), np.nan_to_num(w_grouped))
    return idx, count, grouped


def _uniform(b, n, seed, lo=-1.05, hi=1.05):
    return np.random.RandomState(seed).uniform(lo, hi, (b, n, 3)).astype(np.float32)


def _clustered(b, n, seed):
    rs = np.random.RandomState(seed)
    centres = rs.uniform(-0.8, 0.8, (b, 4, 3))
    pick = rs.randint(0, 4, (b, n))
    x = centres[np.arange(b)[:, None], pick] + rs.normal(0, 0.02, (b, n, 3))
    return x.astype(np.float32)


def _duplicates(b, n, seed):
    rs = np.random.RandomState(seed)
    base = rs.uniform(-1, 1, (b, 7, 3)).astype(np.float32)
    return base[np.arange(b)[:, None], rs.randint(0, 7, (b, n))]


@pytest.mark.parametrize("nsample", [1, 128, 512])
@pytest.mark.parametrize("kind", ["uniform", "clustered", "duplicates"])
def test_voxels_match_the_oracle(kind, nsample):
    xyz = {"uniform": _uniform, "clustered": _clustered, "duplicates": _duplicates}[kind](3, 4096, 1)
    _, count, _ = _check(xyz, 12, 1.0, nsample, seed=7)
    c = count.cpu().numpy()
    if kind != "uniform":
        assert (c > 128).any()  # the CTA path
        assert nsample == 512 or (c > nsample).any()  # the draw
    if kind == "clustered":  # the warp path's 1, 2 and 4 keys per lane
        assert ((c > 0) & (c <= 32)).any() and ((c > 32) & (c <= 64)).any() and ((c > 64) & (c <= 128)).any()


@pytest.mark.parametrize("isize,nsample", [(1, 512), (32, 128), (32, 512), (128, 1), (128, 128)])
def test_pillars_match_the_oracle(isize, nsample):
    xyz = np.concatenate([_uniform(2, 3000, 2), _clustered(1, 3000, 3)])
    xyz[0, ::17, 2] = np.nan  # z is carried raw
    _check(xyz, isize, 1.0, nsample, seed=-3, dims=2)


@pytest.mark.parametrize("vsize,nsample", [(1, 1), (1, 128), (1, 512), (64, 1), (64, 8), (12, 512)])
def test_grid_sizes(vsize, nsample):
    _check(np.concatenate([_uniform(2, 2500, 4), _clustered(1, 2500, 5)]), vsize, 0.9, nsample, seed=2 ** 63 + 5)


@pytest.mark.parametrize("vsize,dims", [(1, 3), (12, 3), (1, 2)])
def test_one_cell_beyond_the_select_limit(vsize, dims):
    """A cell of more than kSelectMaxRows (16384) rows: V = 1, or a cluster inside one voxel."""
    rs = np.random.RandomState(9)
    xyz = rs.uniform(-0.99, 0.99, (2, 40000, 3)).astype(np.float32)
    xyz[1, :30000] = rs.uniform(0.01, 0.15, (30000, 3))
    _, count, _ = _check(xyz, vsize, 1.0, 128, seed=11, dims=dims)
    assert count.max().item() > 16384


def test_nan_padding_and_lengths():
    n = 3000
    xyz = _clustered(4, n, 6)
    lens = [0, 1, n, 1700]
    for i, l in enumerate(lens):
        xyz[i, l:] = np.nan
    _check(xyz, 12, 1.0, 64, seed=3, lengths=lens)
    _check(xyz, 12, 1.0, 64, seed=3, lengths=lens, dev_lengths=torch.tensor(lens, dtype=torch.int32, device=DEV))
    # device lengths are clamped to [0, N]
    clamped = torch.tensor([-5, 1, n + 9, 1700], dtype=torch.int64, device=DEV)
    _check(xyz, 32, 1.0, 16, seed=3, dims=2, lengths=lens, dev_lengths=clamped)
    with pytest.raises(ValueError, match="lengths"):
        pc_util.voxel_group(torch.from_numpy(xyz).to(DEV), 12, lengths=[0, 1, n + 1, 5])


def test_golden_fixtures_through_the_wrappers():
    """The reference's own point_cloud_to_volume_batch, point_cloud_to_volume_v2_batch and point_cloud_to_image_batch
    outputs, bit for bit, and the fixtures' inputs against the oracle at other nsample (draws included)."""
    g = np.load(os.path.join(GOLDEN, "pcutil_volume.npz"))
    for tag in ("v12_r1", "v7_r0.7", "v1_r1"):
        v, r, s = g[f"{tag}_params"]
        v, r, s = int(v), float(r), int(s)
        x = torch.from_numpy(g[f"{tag}_xyz"]).to(DEV)
        got = pc_util.point_cloud_to_volume_v2_batch(x, v, r, s)
        np.testing.assert_array_equal(got.cpu().numpy(), g[f"{tag}_v2"], err_msg=tag)
        inside = torch.from_numpy(g[f"{tag}_inside"]).to(DEV)
        vol = pc_util.point_cloud_to_volume_batch(inside, v, r)
        np.testing.assert_array_equal(vol.cpu().numpy(), g[f"{tag}_vol"], err_msg=tag)
        vol5 = pc_util.point_cloud_to_volume_batch(inside, v, r, flatten=False)
        assert vol5.shape == (2, v, v, v, 1) and torch.equal(vol5.reshape(2, -1), vol)
        # volume_to_point_cloud is torch.nonzero(vol == 1)
        pts = torch.nonzero(vol5[0, ..., 0] == 1).cpu().numpy()
        want = np.argwhere(g[f"{tag}_vol"][0].reshape(v, v, v) == 1)
        np.testing.assert_array_equal(pts, want)
        _check(g[f"{tag}_xyz"], v, r, 2, seed=1)
    g = np.load(os.path.join(GOLDEN, "pcutil_image.npz"))
    for tag in ("i8_r1", "i13_r0.7", "i1_r1"):
        v, r, s = g[f"{tag}_params"]
        v, r, s = int(v), float(r), int(s)
        got = pc_util.point_cloud_to_image_batch(torch.from_numpy(g[f"{tag}_xyz"]).to(DEV), v, r, s).cpu().numpy()
        want = g[f"{tag}_img"]
        assert np.array_equal(np.isnan(got), np.isnan(want))
        np.testing.assert_array_equal(np.nan_to_num(got), np.nan_to_num(want), err_msg=tag)
        _check(g[f"{tag}_xyz"], v, r, 3, seed=1, dims=2)


def test_two_runs_give_the_same_bits():
    x = torch.from_numpy(_clustered(8, 4096, 12)).to(DEV)
    a = pc_util.voxel_group(x, 12, 1.0, 128, 5)
    b = pc_util.voxel_group(x, 12, 1.0, 128, 5)
    for u, v in zip(a, b):
        assert torch.equal(u, v)
    c = pc_util.voxel_group(x, 12, 1.0, 128, 6)
    assert not torch.equal(a[0], c[0]) and torch.equal(a[1], c[1])


def test_device_seed_in_cuda_graph():
    xyz = _clustered(3, 4096, 13)
    x = torch.from_numpy(xyz).to(DEV)
    seed = torch.tensor([1], dtype=torch.int64, device=DEV)
    pc_util.voxel_group(x, 12, 1.0, 64, seed)  # loads the library and sets the kernels' attributes outside the capture
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    before = _lib.launch_count()
    with torch.cuda.stream(s):
        with torch.cuda.graph(g, stream=s):
            idx, count, grouped = pc_util.voxel_group(x, 12, 1.0, 64, seed)
    torch.cuda.current_stream().wait_stream(s)
    assert _lib.launch_count() > before
    for v in (99, -4, 2 ** 40):
        seed.fill_(v)
        g.replay()
        torch.cuda.synchronize()
        w_idx, w_count, w_grouped = VO.oracle_voxel_group(xyz, 12, 1.0, 64, v)
        np.testing.assert_array_equal(idx.cpu().numpy(), w_idx, err_msg=str(v))
        np.testing.assert_array_equal(count.cpu().numpy(), w_count)
        np.testing.assert_array_equal(grouped.cpu().numpy(), w_grouped)


@pytest.mark.parametrize("dims", [3, 2])
def test_group_point_gives_the_rows_grouped_normalises(dims):
    xyz = np.concatenate([_uniform(1, 4096, 14), _clustered(1, 4096, 15)])
    x = torch.from_numpy(xyz).to(DEV)
    v, r = 12, 1.0
    idx, count, grouped = pc_util.voxel_group(x, v, r, 32, 3, dims=dims)
    raw = group_point(x, idx).cpu().numpy().astype(np.float64)        # (B, C, S, 3)
    i = idx.cpu().numpy()
    np.testing.assert_array_equal(raw, xyz[np.arange(2)[:, None, None], i].astype(np.float64))
    cells = np.arange(v ** dims)
    coord = np.stack([cells // v, cells % v], 1) if dims == 2 else np.stack([cells // (v * v), (cells // v) % v, cells % v], 1)
    voxel = 2 * r / v
    norm = (raw[..., :dims] - ((coord + 0.5) * voxel - r)[None, :, None, :]) / voxel
    if dims == 2:
        norm = norm.astype(np.float32).astype(np.float64)
    full = count.cpu().numpy() > 0
    np.testing.assert_array_equal(grouped.cpu().numpy()[..., :dims][full], norm[full])
    if dims == 2:
        np.testing.assert_array_equal(grouped.cpu().numpy()[..., 2][full], raw[..., 2][full])
