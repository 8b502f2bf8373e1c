"""CPU tests of voxel and pillar grouping (pointnet2_b200.pc_util, csrc/voxel.cu): the numpy oracle against the
reference's own pc_util outputs (tests/golden/pcutil_*.npz, recorded by oracle/pcutil_ref.py), the oracle's draw of
over-full cells, the kernels' resource usage and the argument errors (no launch)."""
import ctypes
import os
import re
import shutil
import subprocess
import sys

import numpy as np
import pytest
import torch
from scipy import stats

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import voxel_oracle as VO  # noqa: E402

from pointnet2_b200 import _lib, pc_util  # noqa: E402

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _cases(name, out_key):
    g = np.load(os.path.join(GOLDEN, f"pcutil_{name}.npz"))
    for tag in sorted({k.rsplit("_", 1)[0] for k in g.files if k.endswith("_params")}):
        v, r, s = g[f"{tag}_params"]
        yield tag, int(v), float(r), int(s), g


def test_oracle_equals_the_reference_volumes():
    seen = 0
    for tag, v, r, s, g in _cases("volume", "v2"):
        xyz = g[f"{tag}_xyz"]
        idx, count, grouped = VO.oracle_voxel_group(xyz, v, r, s)
        assert count.max() <= s, tag  # recorded cells draw nothing at random
        want = g[f"{tag}_v2"]
        assert want.dtype == np.float64
        np.testing.assert_array_equal(grouped.reshape(want.shape), want, err_msg=tag)
        # occupancy, on the in-grid copy the reference can index
        _, c, _ = VO.oracle_voxel_group(g[f"{tag}_inside"], v, r, 1)
        np.testing.assert_array_equal((c > 0).astype(np.float64), g[f"{tag}_vol"], err_msg=tag)
        assert np.isnan(xyz).any() or v == 1, tag
        seen += 1
    assert seen == 3


def test_oracle_equals_the_reference_images():
    seen = 0
    for tag, v, r, s, g in _cases("image", "img"):
        idx, count, grouped = VO.oracle_voxel_group(g[f"{tag}_xyz"], v, r, s, dims=2)
        assert count.max() <= s, tag
        want = g[f"{tag}_img"]
        np.testing.assert_array_equal(grouped.reshape(want.shape), want, err_msg=tag)  # NaN z rows compare equal
        seen += 1
    assert seen == 3


def test_fixtures_cover_the_edges():
    """Both sides of cell edges, quotients in (-1, 0), points outside the grid, duplicates, V = 1 and I = 1."""
    g = np.load(os.path.join(GOLDEN, "pcutil_volume.npz"))
    xyz = g["v12_r1_xyz"]
    q = (xyz + np.float32(1.0)) / np.float32(2 / 12)
    with np.errstate(invalid="ignore"):
        assert ((q > -1) & (q < 0)).any()
        assert (q >= 12).any() and (q <= -1).any()
        frac = q - np.floor(q)
        assert ((frac == 0) & (q >= 1) & (q < 12)).any()       # on an edge
        assert ((frac > 0.99999) & (q < 12)).any()            # just below one
    assert len(np.unique(xyz[1], axis=0)) < len(xyz[1])       # duplicates
    assert g["v1_r1_params"][0] == 1
    assert np.load(os.path.join(GOLDEN, "pcutil_image.npz"))["i1_r1_params"][0] == 1


def _cluster(n, seed, sigma=0.03, centre=0.0):
    rs = np.random.RandomState(seed)
    return np.clip(rs.normal(centre, sigma, (n, 3)), -0.99, 0.99).astype(np.float32)


@pytest.mark.parametrize("dims", [3, 2])
def test_over_full_cells_are_distinct_members(dims):
    pts = _cluster(3000, 1)
    v, s = 8, 37
    idx, count, grouped = VO.oracle_cloud(pts, v, 1.0, s, seed=5, dims=dims)
    cell = VO.cells_of(pts, v, 1.0, dims)
    over = np.nonzero(count > s)[0]
    assert len(over) >= 4 and count.max() > 300
    for c in over:
        rows = idx[c]
        assert len(np.unique(rows)) == s
        assert (cell[rows] == c).all()
    for c in np.nonzero((count > 0) & (count <= s))[0]:
        members = np.nonzero(cell == c)[0]
        k = count[c]
        np.testing.assert_array_equal(idx[c, :k], members)
        assert (idx[c, k:] == members[-1]).all()
    # the seed changes the draw only
    idx2, count2, _ = VO.oracle_cloud(pts, v, 1.0, s, seed=6, dims=dims)
    np.testing.assert_array_equal(count, count2)
    assert not np.array_equal(idx[over], idx2[over])
    small = count <= s
    np.testing.assert_array_equal(idx[small], idx2[small])


def test_draw_does_not_depend_on_the_launch_shape():
    """A cloud's result depends on its rows, its position b in the batch and the seed: not on the row stride, the
    padding, the lengths of other clouds or the batch size."""
    a, b = _cluster(900, 2), _cluster(700, 3, 0.2)
    want = VO.oracle_voxel_group(np.stack([a, a]), 6, 1.0, 20, seed=11)
    n = 1200
    pad = np.full((3, n, 3), np.nan, np.float32)
    pad[0, :700], pad[1, :900], pad[2, :900] = b, a, a
    got = VO.oracle_voxel_group(pad, 6, 1.0, 20, seed=11, lengths=[700, 900, 5000])
    for k in range(3):
        np.testing.assert_array_equal(got[k][1], want[k][1])
    assert (want[1][1] > 20).any()


def test_draw_is_uniform_over_seeds():
    """Every row of an over-full cell is kept with probability S / c: a chi-square test over 3000 seeds."""
    pts = _cluster(400, 4, 0.004, 0.1)
    v, s, trials = 4, 10, 3000
    cell = VO.cells_of(pts, v, 1.0, 3)
    c = np.bincount(cell[cell >= 0]).argmax()
    members = np.nonzero(cell == c)[0]
    assert len(members) == 400
    hits = np.zeros(len(pts))
    first = np.zeros(len(pts))
    for seed in range(trials):
        idx, _, _ = VO.oracle_cloud(pts, v, 1.0, s, seed=seed)
        hits[idx[c]] += 1
        first[idx[c, 0]] += 1
    assert stats.chisquare(hits[members]).pvalue > 1e-3
    assert stats.chisquare(first[members]).pvalue > 1e-3
    assert hits.sum() == trials * s


def test_voxel_kernels_do_not_spill():
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(cuobjdump):
        pytest.skip("cuobjdump not available")
    out = subprocess.run([cuobjdump, "-res-usage", _lib.lib_path()], capture_output=True, text=True).stdout
    found = re.findall(r"Function (\S*voxel_\w+_kernel\S*):\s*\n\s*REG:\d+ STACK:(\d+)", out)
    assert len(found) == 5, found  # count, scan, fill, warp, cta
    assert all(stack == "0" for _, stack in found), found


def test_argument_errors_launch_nothing():
    before = _lib.launch_count()
    x = torch.zeros(2, 10, 3)
    vg = pc_util.voxel_group
    with pytest.raises(RuntimeError, match="no CPU path"):
        vg(x, 12)
    with pytest.raises(TypeError):
        vg(x.double().cuda() if torch.cuda.is_available() else np.zeros((2, 10, 3), np.float32), 12)
    with pytest.raises(ValueError, match="shape"):
        vg(torch.zeros(2, 10, 2), 12)
    with pytest.raises(ValueError, match="dims"):
        vg(x, 12, dims=4)
    with pytest.raises(ValueError, match="nsample"):
        vg(x, 12, nsample=0)
    with pytest.raises(ValueError, match="nsample"):
        vg(x, 12, nsample=pc_util.MAX_NSAMPLE + 1)
    with pytest.raises(TypeError, match="vsize"):
        vg(x, 12.0)
    with pytest.raises(ValueError, match="vsize"):
        vg(x, 0)
    with pytest.raises(ValueError, match="vsize"):
        vg(x, 1291)   # 2 x 1291^3 cells pass 2^31
    for r in (0.0, -1.0, float("nan"), float("inf"), 1e39, 1e-50):
        with pytest.raises(ValueError, match="radius"):
            vg(x, 12, radius=r)
    with pytest.raises(ValueError, match="cell edge"):
        vg(torch.zeros(1, 10, 3), 30000, radius=1e-41, dims=2)
    with pytest.raises(TypeError, match="radius"):
        vg(x, 12, radius="1")
    with pytest.raises(ValueError, match="nsample"):
        pc_util.point_cloud_to_volume_v2_batch(x, 12, num_sample=0)
    with pytest.raises(ValueError, match="dims|shape"):
        pc_util.point_cloud_to_image_batch(torch.zeros(10, 3), 32)
    assert _lib.launch_count() == before


def test_abi_refusals():
    lib = _lib.load()
    before = _lib.launch_count()
    null = ctypes.c_void_p(0)
    one = ctypes.c_void_p(256)  # never dereferenced: every call below is refused first
    wsb = lib.pn2_voxel_group_workspace_bytes
    assert wsb(0, 10, 12, 3) == 0 and wsb(2, 0, 12, 3) == 0 and wsb(2, 10, 0, 3) == 0
    assert wsb(2, 10, 12, 4) == 0 and wsb(2, 10, 1291, 3) == 0 and wsb(2, 10, 46341, 2) == 0
    assert wsb(2, 10, 1290, 3) == 0  # 2 x 1290^3 cells pass 2^31
    ws = wsb(2, 4096, 12, 3)
    assert ws >= 4 * (2 * 1728 + 2 * 4096)
    assert wsb(2, 128, 12, 3) < wsb(2, 129, 12, 3)  # the list of cells over 128 rows: at most n / 129 per cloud
    call = lib.pn2_voxel_group
    args = lambda **kw: dict(dict(b=2, n=4096, xyz=one, lengths=null, dim=12, dims=3, radius=1.0, nsample=128,  # noqa: E731
                                  seed=0, seed_dev=null, count=one, idx=one, grouped=one, ws=one, wsb=ws, stream=null), **kw)
    for bad in (dict(nsample=0), dict(nsample=16385), dict(radius=0.0), dict(radius=float("nan")), dict(radius=1e39),
                dict(radius=-1.0), dict(dims=1), dict(xyz=null), dict(grouped=null), dict(ws=null), dict(wsb=ws - 1),
                dict(ws=ctypes.c_void_p(257)), dict(b=0), dict(dim=0)):
        assert call(*args(**bad).values()) == 1, bad
    assert _lib.launch_count() == before
