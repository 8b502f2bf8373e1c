"""Point-cloud rendering on the GPU: render_balls bit for bit against the reference's render_ball (fixtures, the C
restatement and, where oracle/_ref has it, the compiled reference) on ragged batches, batch independence, the
projection against a float64 numpy restatement, show_points against its parts, a CUDA graph with rewritten lengths under
sync-debug mode "error", and one 10^6-point scene."""
import numpy as np
import pytest
import torch

import render_oracle as RO
from conftest import golden_names, load_golden
from oracle import render_ref as RR
from pointnet2_b200 import render, workloads as W

pytestmark = pytest.mark.gpu

INT_MIN, INT_MAX = np.iinfo(np.int32).min, np.iinfo(np.int32).max


@pytest.fixture(autouse=True)
def no_sync():
    """Every render call here is asynchronous: a device-to-host sync inside one raises."""
    torch.cuda.set_sync_debug_mode("error")
    yield
    torch.cuda.set_sync_debug_mode("default")


def host(t):
    torch.cuda.set_sync_debug_mode("default")
    a = t.cpu().numpy()
    torch.cuda.set_sync_debug_mode("error")
    return a


def to_dev(a, dev):
    torch.cuda.set_sync_debug_mode("default")
    t = torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    torch.cuda.set_sync_debug_mode("error")
    return t


def reference(xyz, col, h, w, r, bg):
    """The C restatement, and the reference's compiled function where it is present: they must agree."""
    want = RR.oracle_render_ball(xyz, col, h, w, r, bg)
    if RR.have_refrender():
        np.testing.assert_array_equal(want, RR.refrender_ball(xyz, col, h, w, r, bg))
    return want


@pytest.mark.parametrize("name", golden_names("render_"))
def test_fixture(name, dev):
    g = load_golden(name)
    col = g.get("colors")
    img = render.render_balls(to_dev(g["xyz"][None], dev), None if col is None else to_dev(col[None], dev), int(g["h"]),
                              int(g["w"]), int(g["r"]), tuple(int(v) for v in g["background"]))
    np.testing.assert_array_equal(host(img)[0], g["out"])


def _batch(rng, b, n, h, w, dup=False):
    xyz = np.stack([rng.randint(-30, h + 30, (b, n)), rng.randint(-30, w + 30, (b, n)),
                    rng.randint(-400, 400, (b, n))], 2).astype(np.int32)
    if dup:  # a few hundred distinct points, many copies each, few depths
        src = xyz[:, :max(1, n // 50)]
        xyz = src[:, rng.randint(0, src.shape[1], n)]
        xyz[..., 2] = rng.randint(-2, 3, (b, n))
    col = (rng.rand(b, n, 3) * 255).astype(np.float32)
    col[:, ::7] = np.round(col[:, ::7]) + 0.5
    return xyz, col


CASES = [  # (seed, b, n, h, w, r, dup)
    (0, 1, 1, 1, 1, 1, False), (1, 8, 500, 1, 300, 2, False), (2, 4, 3000, 120, 90, 8, False),
    (3, 8, 20000, 800, 1200, 10, False), (4, 3, 20000, 640, 480, 25, True), (5, 6, 2048, 256, 256, 1, True),
    (6, 2, 7000, 333, 77, 8, True),
]


@pytest.mark.parametrize("seed,b,n,h,w,r,dup", CASES)
def test_ragged_batches_match_the_reference(seed, b, n, h, w, r, dup, dev):
    rng = np.random.RandomState(seed)
    xyz, col = _batch(rng, b, n, h, w, dup)
    lens = rng.randint(0, n + 1, b)
    lens[0] = n
    if b > 1:
        lens[1] = 0
    pad = xyz.copy()
    colp = col.copy()
    for i, l in enumerate(lens):  # padding rows that would cover the canvas if they were read
        pad[i, l:] = np.where(rng.rand(n - l, 3) < 0.5, INT_MIN, INT_MAX)
        pad[i, l:, :2] = rng.randint(0, min(h, w), (n - l, 2))
        colp[i, l:] = np.nan
    bg = (3, 0, 200) if seed % 2 else (0, 0, 0)
    lt = to_dev(lens.astype(np.int32), dev)
    img = host(render.render_balls(to_dev(pad, dev), to_dev(colp, dev), h, w, r, bg, lengths=lt))
    for i in range(b):
        np.testing.assert_array_equal(img[i], reference(xyz[i, :lens[i]], col[i, :lens[i]], h, w, r, bg), f"cloud {i}")
    # white (colors None) and lengths None
    img = host(render.render_balls(to_dev(xyz, dev), None, h, w, r, bg))
    for i in range(min(b, 2)):
        np.testing.assert_array_equal(img[i], reference(xyz[i], None, h, w, r, bg))


def test_each_image_is_its_cloud_alone_and_batch_order_free(dev):
    rng = np.random.RandomState(11)
    xyz, col = _batch(rng, 6, 4000, 200, 160, True)
    lens = to_dev(np.array([4000, 17, 0, 2500, 4000, 1], np.int32), dev)
    x, c = to_dev(xyz, dev), to_dev(col, dev)
    full = render.render_balls(x, c, 200, 160, 6, lengths=lens)
    perm = to_dev(np.array([3, 0, 5, 1, 4, 2]), dev)
    permuted = render.render_balls(x[perm], c[perm], 200, 160, 6, lengths=lens[perm])
    alone = [render.render_balls(x[i:i + 1], c[i:i + 1], 200, 160, 6, lengths=lens[i:i + 1]) for i in range(6)]
    full, permuted = host(full), host(permuted)
    np.testing.assert_array_equal(permuted, full[[3, 0, 5, 1, 4, 2]])
    for i in range(6):
        np.testing.assert_array_equal(host(alone[i])[0], full[i], str(i))


@pytest.mark.parametrize("seed", range(4))
def test_projection_matches_numpy(seed, dev):
    rng = np.random.RandomState(40 + seed)
    b, n = 3, 5000
    xyz = rng.randn(b, n, 3) * rng.choice([0.01, 1.0, 300.0]) + rng.randn(3) * 5
    xa, ya, zm = [0.0, 0.7, -1.3], [0.0, -0.2, 2.9], [1.0, 1.7, 0.6]
    lens = np.array([n, 1234, 2], np.int32)
    got = host(render.project_points(to_dev(xyz, dev), 800, xa, ya, zm, lengths=to_dev(lens, dev)))
    allowed = 0
    for i in range(b):
        for v in range(3):
            nx, want = RO.project_np(xyz[i, :lens[i]], 800, xa[v], ya[v], zm[v])
            ok, bad = RO.near_integer_mismatches(nx, got[i, v, :lens[i]], want)
            assert bad == 0, (i, v)
            allowed += ok
        if lens[i] < n:
            assert (got[i, :, lens[i]:] == 0).all()
    # float32 input is taken as float64
    got32 = host(render.project_points(to_dev(xyz.astype(np.float32), dev), 600, 0.4, 0.1))
    nx, want = RO.project_np(xyz[0].astype(np.float32).astype(np.float64), 600, 0.4, 0.1)
    ok, bad = RO.near_integer_mismatches(nx, got32[0, 0], want)
    assert bad == 0
    print(f"coordinates within 1e-9 of an integer that truncated differently: {allowed + ok}")


def test_projection_of_coincident_points_and_batch_independence(dev):
    xyz = np.zeros((2, 10, 3))
    xyz[1] = np.random.RandomState(3).randn(10, 3)
    got = host(render.project_points(to_dev(xyz, dev), 801))
    assert (got[0, 0] == [400, 400, 0]).all()
    alone = host(render.project_points(to_dev(xyz[1:], dev), 801))
    np.testing.assert_array_equal(alone[0], got[1])


@pytest.mark.parametrize("mb", [0, 1, 2])
@pytest.mark.parametrize("normalize", [True, False])
def test_show_points_is_render_of_projection(mb, normalize, dev):
    rng = np.random.RandomState(7 + mb)
    b, n = 3, 2048
    xyz = to_dev(rng.randn(b, n, 3), dev)
    colors = to_dev(rng.rand(b, n, 3) * 3.0, dev)  # float64 colour rows, as part_seg/test.py passes them
    lens = to_dev(np.array([n, 700, 0], np.int32), dev)
    xa, ya = [0.0, 0.5, -1.0], 0.3
    img = render.show_points(xyz, colors, size=300, xangle=xa, yangle=ya, zoom=1.2, ballradius=4, background=(5, 6, 7),
                             normalizecolor=normalize, magnify_blue=mb, lengths=lens)
    assert img.shape == (b, 3, 300, 300, 3)
    ixyz = render.project_points(xyz, 300, xa, ya, 1.2, lengths=lens)
    c = host(colors)
    out, ix, hl = host(img), host(ixyz), host(lens)
    for i in range(b):
        ci = RO.normalize_np(c[i, :hl[i]]) if normalize and hl[i] else c[i, :hl[i]].astype(np.float32)
        for v in range(3):
            want = reference(ix[i, v, :hl[i]], ci, 300, 300, 4, (5, 6, 7))
            np.testing.assert_array_equal(out[i, v], RO.magnify_np(want, mb), (i, v))
    white = host(render.show_points(xyz[:1], None, size=200, ballradius=3))
    np.testing.assert_array_equal(white[0, 0], reference(host(render.project_points(xyz[:1], 200))[0, 0], None, 200, 200,
                                                          3, (0, 0, 0)))


def test_graph_replay_with_rewritten_lengths(dev):
    rng = np.random.RandomState(21)
    xyz, col = _batch(rng, 4, 3000, 128, 128)
    x, c = to_dev(xyz, dev), to_dev(col, dev)
    lens = to_dev(np.array([3000, 10, 0, 1500], np.int32), dev)
    render.render_balls(x, c, 128, 128, 5, lengths=lens)  # warm-up outside the capture
    torch.cuda.set_sync_debug_mode("default")
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = render.render_balls(x, c, 128, 128, 5, lengths=lens)
    for new in ([3000, 10, 0, 1500], [0, 3000, 2999, 1], [5, 5, 5, 5]):
        lens.copy_(torch.tensor(new, dtype=torch.int32))
        g.replay()
        torch.cuda.synchronize()
        img = out.cpu().numpy()
        for i, l in enumerate(new):
            np.testing.assert_array_equal(img[i], reference(xyz[i, :l], col[i, :l], 128, 128, 5, (0, 0, 0)), (new, i))


def test_scene_of_a_million_points(dev):
    pts, _ = W.scene_room(1_000_000, 5)
    ixyz = render.project_points(to_dev(pts[None], dev), 800, 0.6, -0.4)
    img = host(render.render_balls(ixyz[:, 0], None, 800, 800, 8))
    ix = host(ixyz)[0, 0]
    np.testing.assert_array_equal(img[0], RR.oracle_render_ball(ix, None, 800, 800, 8))
