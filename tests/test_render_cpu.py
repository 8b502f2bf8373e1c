"""Point-cloud rendering without a device: the C restatement of render_ball against the reference's compiled function
and the render_*.npz fixtures, the tie and depth rules on hand cases, the numpy restatements of the viewer's host steps,
the wrappers' argument errors, and the C entries' refusals and their agreement with the header and the build list."""
import ctypes
import os
import re

import numpy as np
import pytest
import torch

import render_oracle as RO
from conftest import golden_names, load_golden
from oracle import render_ref as RR
from pointnet2_b200 import _build, _lib, render

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
needs_ref = pytest.mark.skipif(not RR.have_refrender(), reason="oracle/_ref/libref_render.so not built here")


def _cloud(rng, n, h, w, zlo=-50, zhi=50, margin=12):
    return np.stack([rng.randint(-margin, h + margin, n), rng.randint(-margin, w + margin, n),
                     rng.randint(zlo, zhi, n)], 1).astype(np.int32)


@needs_ref
@pytest.mark.parametrize("seed", range(6))
def test_oracle_equals_reference_on_random_clouds(seed):
    rng = np.random.RandomState(seed)
    for _ in range(25):
        h, w = rng.randint(1, 60), rng.randint(1, 60)
        n, r = rng.randint(1, 120), int(rng.choice([-3, 0, 1, 2, 3, 8, 10, 25]))
        xyz = _cloud(rng, n, h, w)
        if rng.rand() < 0.5:
            xyz[rng.randint(0, n, n // 2)] = xyz[rng.randint(0, n)]
        col = None if rng.rand() < 0.2 else (rng.rand(n, 3) * rng.choice([1.0, 255.0, 400.0])).astype(np.float32)
        bg = tuple(int(v) for v in rng.randint(0, 256, 3))
        np.testing.assert_array_equal(RR.oracle_render_ball(xyz, col, h, w, r, bg), RR.refrender_ball(xyz, col, h, w, r, bg))


def test_lower_index_wins_equal_depth():
    xyz = np.array([[3, 3, 5], [3, 3, 5], [3, 3, 4]], np.int32)
    col = np.array([[10, 20, 30], [200, 210, 220], [250, 250, 250]], np.float32)
    img = RR.oracle_render_ball(xyz, col, 7, 7, 1)
    # r = 1: the one pattern entry (0, 0), height 1, shade 1; points 0 and 1 both reach z2 = 6, point 0 wins
    zmin, zmax = 4 - 1, 5 + 1
    inten = min(1.0, (6 - zmin) / (zmax - zmin) * 0.7 + 0.3)
    want = [int(np.float32(1.0) * np.float32(c) * inten) for c in (30, 10, 20)]
    assert img[3, 3].tolist() == want
    assert img.reshape(-1, 3).any(1).sum() == 1
    if RR.have_refrender():
        np.testing.assert_array_equal(img, RR.refrender_ball(xyz, col, 7, 7, 1))


def test_depth_test_is_strict_against_the_initial_depth():
    # r = 1: z2 = z + 1.  z2 = -2100000000 is not drawn, -2099999999 is.
    for z, drawn in ((-2100000001, False), (-2100000000, True)):
        xyz = np.array([[1, 1, z]], np.int32)
        img = RR.oracle_render_ball(xyz, None, 3, 3, 1, (7, 7, 7))
        assert (img[1, 1].tolist() != [7, 7, 7]) == drawn
        if RR.have_refrender():
            np.testing.assert_array_equal(img, RR.refrender_ball(xyz, None, 3, 3, 1, (7, 7, 7)))


def test_fixtures_cover_the_cases():
    names = golden_names("render_")
    assert {"render_r0", "render_r1", "render_r2", "render_r8", "render_r25", "render_1x1", "render_ties",
            "render_fractional", "render_background"} <= set(names)


@pytest.mark.parametrize("name", golden_names("render_"))
def test_oracle_reproduces_fixture(name):
    g = load_golden(name)
    out = RR.oracle_render_ball(g["xyz"], g.get("colors"), int(g["h"]), int(g["w"]), int(g["r"]), g["background"])
    np.testing.assert_array_equal(out, g["out"])


def test_view_matrices_follow_showpoints():
    rots = render._views([0.0, 0.3], -0.7, 1.5)
    assert rots.shape == (2, 3, 3)
    for k, xa in enumerate((0.0, 0.3)):
        rx = np.array([[1, 0, 0], [0, np.cos(xa), -np.sin(xa)], [0, np.sin(xa), np.cos(xa)]])
        ry = np.array([[np.cos(-0.7), 0, -np.sin(-0.7)], [0, 1, 0], [np.sin(-0.7), 0, np.cos(-0.7)]])
        np.testing.assert_array_equal(rots[k], np.eye(3).dot(rx).dot(ry) * 1.5)
    assert render._views(0.0, 0.0, 1.0).shape == (1, 3, 3)
    with pytest.raises(ValueError, match="one length"):
        render._views([0.0, 0.1], [0.0, 0.1, 0.2], 1.0)
    with pytest.raises(ValueError, match="1-D"):
        render._views(np.zeros((2, 2)), 0.0, 1.0)


def test_numpy_projection_on_hand_values():
    # mean (1, 0, 0), radius 1, scale 2.2 / 800: (2, 0, 0) -> x = 1 / (2.2/800) + 400 = 763.63.. -> 763
    xyz = np.array([[0.0, 0.0, 0.0], [2.0, 0.0, 0.0]])
    nxyz, ixyz = RO.project_np(xyz)
    assert ixyz.tolist() == [[36, 400, 0], [763, 400, 0]]
    # a quarter turn about y sends +x to -z (p . Ry)
    _, ixyz = RO.project_np(xyz, yangle=np.pi / 2)
    assert ixyz[1].tolist() == [400, 400, -363]
    allowed, bad = RO.near_integer_mismatches(np.array([1.0 - 1e-12, 2.5]), np.array([0, 2]), np.array([1, 2]))
    assert (allowed, bad) == (1, 0)


def test_numpy_magnify_blue_on_hand_values():
    show = np.zeros((4, 5, 3), np.uint8)
    show[0, 0, 0] = 9
    show[0, 0, 1] = 7
    one = RO.magnify_np(show, 1)
    assert sorted(zip(*np.nonzero(one[:, :, 0]))) == [(0, 0), (0, 1), (1, 0), (1, 1)]
    two = RO.magnify_np(show, 2)
    # wrap-around: the pixel's row above is row 3, its column to the left column 4
    assert two[:, :, 0].astype(bool).sum() == 9 and two[3, 4, 0] == 9
    assert (one[:, :, 1] == show[:, :, 1]).all() and (RO.magnify_np(show, 0) == show).all()
    for level in (0, 1, 2):
        got = render.magnify_blue_channel(torch.from_numpy(show.copy())[None], level)[0].numpy()
        np.testing.assert_array_equal(got, RO.magnify_np(show, level))


def test_wrappers_refuse_bad_arguments():
    cpu = torch.zeros(1, 4, 3, dtype=torch.int32)
    with pytest.raises(RuntimeError, match="CUDA"):
        render.render_balls(cpu, None, 8, 8, 2)
    with pytest.raises(TypeError):
        render.render_balls(cpu.float(), None, 8, 8, 2)
    with pytest.raises(RuntimeError, match="CUDA"):
        render.project_points(torch.zeros(1, 4, 3))
    with pytest.raises(ValueError, match="background"):
        render._background((0, 0, 256), "render_balls")
    with pytest.raises(ValueError, match="background"):
        render._background((0, 0), "render_balls")
    with pytest.raises(ValueError, match="0 <= lengths"):
        render._lengths([0, 5], 2, 4, torch.device("cpu"), "render_balls")
    with pytest.raises(ValueError, match="shape"):
        render._lengths([1, 2, 3], 2, 4, torch.device("cpu"), "render_balls")
    assert render._lengths([0, 4], 2, 4, torch.device("cpu"), "render_balls").tolist() == [0, 4]


def _proto_args(name):
    text = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "pn2_api.h")).read(), flags=re.S)
    proto = re.search(rf"(?:int|size_t)\s+{name}\s*\((.*?)\)\s*;", text, flags=re.S).group(1)
    return [a.strip() for a in proto.split(",")]


@pytest.mark.parametrize("name", ["pn2_render_balls_workspace_bytes", "pn2_render_balls", "pn2_render_balls_counted",
                                  "pn2_project_points"])
def test_header_and_ctypes_agree(name):
    assert name in _lib.EXPORTED_SYMBOLS and hasattr(_lib.load(), name)
    args = _proto_args(name)
    _, argtypes = _lib._SIGNATURES[name]
    assert len(args) == len(argtypes)
    scalars = {"int": _lib.c_int, "long long": _lib.c_longlong, "size_t": _lib.c_size_t, "float": _lib.c_float}
    for a, t in zip(args, argtypes):
        want = _lib._P if "*" in a else scalars[a.rsplit(" ", 1)[0]]
        assert t is want, (name, a, t)


def test_c_entries_refuse_bad_arguments_without_a_launch():
    lib = _lib.load()
    assert lib.pn2_render_balls_workspace_bytes(2, 800, 600) == 2 * 800 * 600 * 8 + 256
    assert lib.pn2_render_balls_workspace_bytes(0, 8, 8) == 0
    assert lib.pn2_render_balls_workspace_bytes(1, 0, 8) == 0
    assert lib.pn2_render_balls_workspace_bytes(65536, 8, 8) == 0
    assert lib.pn2_render_balls_workspace_bytes(1, 1 << 16, 1 << 15) == 0
    fake = ctypes.c_void_p(256)  # never dereferenced: every call below must fail its checks first
    null = ctypes.c_void_p(0)
    bg = (ctypes.c_ubyte * 3)(0, 0, 0)
    before = _lib.launch_count()

    def rb(b=2, n=8, h=16, w=16, r=3, xyz=fake, out=fake, ws=fake, wsb=None, back=bg):
        need = lib.pn2_render_balls_workspace_bytes(max(b, 1), max(h, 1), max(w, 1)) if wsb is None else wsb
        return lib.pn2_render_balls(b, n, h, w, xyz, null, null, r, back, ws, need, out, null)

    assert rb(xyz=null) == 1 and rb(out=null) == 1 and rb(ws=null) == 1 and rb(back=None) == 1
    assert rb(n=-1) == 1 and rb(h=0) == 1 and rb(w=-4) == 1 and rb(b=-1) == 1 and rb(b=65536) == 1
    assert rb(r=4097) == 1 and rb(wsb=64) == 1 and rb(ws=ctypes.c_void_p(264)) == 1
    assert rb(b=0) == 0
    assert lib.pn2_render_balls_counted(1, 8, 16, 16, fake, null, null, 3, bg, fake, 1 << 20, fake, null, null) == 1

    def pp(b=2, n=8, v=1, xyz=fake, rot=fake, size=800, wsb=64, out=fake):
        return lib.pn2_project_points(b, n, v, xyz, null, rot, size, fake, wsb, out, null)

    assert pp(xyz=null) == 1 and pp(rot=null) == 1 and pp(out=null) == 1 and pp(v=0) == 1 and pp(size=0) == 1
    assert pp(wsb=63) == 1 and pp(b=-1) == 1 and pp(n=-2) == 1
    assert pp(b=0) == 0 and pp(n=0) == 0
    assert _lib.launch_count() == before
    assert "render.cu" in _build.SOURCES and os.path.exists(os.path.join(_build.CSRC, "render.cu"))


def test_sass_audit_lists_the_render_kernels():
    text = open(os.path.join(ROOT, "tools", "sass_audit.py")).read()
    for k in ("render_zrange_kernel", "render_splat_kernel<false>", "render_resolve_kernel", "project_stats_kernel",
              "project_points_kernel"):
        assert f'"{k}"' in text, k
