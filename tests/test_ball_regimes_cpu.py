"""Without a GPU: tests/ball_regimes.py on its own.  Hand cases for the regimes it names, and the property the grids
rest on: every hit of the C oracle lies in its query's clamped 3x3x3 cell neighbourhood, over several thousand
adversarial clouds (shells at r ± 8 ulps, points on cell edges, far offsets with small radii, degenerate boxes,
16-cell grids, queries outside the box)."""
import numpy as np
import pytest

import ball_regimes as R

f32 = np.float32


def _ulps(x, k):
    x = f32(x)
    for _ in range(abs(k)):
        x = np.nextafter(x, f32(np.inf if k > 0 else -np.inf), dtype=f32)
    return x


# ------------------------------------------------------------------------------------------------- hand cases
def test_geometry_nan_makes_the_box_infinite():
    x = np.random.RandomState(0).random_sample((600, 3)).astype(f32)
    assert R.geometry(x, 0.05)["finite_box"]
    y = x.copy()
    y[5, 1] = np.nan
    assert not R.geometry(y, 0.05)["finite_box"]


def test_nan_axis_cloud_has_no_grid():
    """every point NaN in x: the box must be infinite, not finite on y and z with a NaN extent in x"""
    x = np.random.RandomState(1).random_sample((3000, 3)).astype(f32)
    x[:, 0] = np.nan
    g = R.geometry(x, 0.05)
    assert not g["finite_box"] and g["dims"] == [1, 1, 1]
    assert not R.BgCloud(x, 0.05, 3000).use_grid and R.global_flag(x, 0.05, 64) == (False, "box")


def test_degenerate_boxes_use_the_radius_as_cell_edge():
    for pts in (np.zeros((1, 3), f32), np.stack([np.linspace(0, 1, 50), np.zeros(50), np.zeros(50)], 1).astype(f32)):
        g = R.geometry(pts, 0.3)
        assert g["finite_box"] and g["ext"][2] == 0
    g = R.geometry(np.zeros((4, 3), f32), 0.3)
    assert g["h"] == R._fmul(f32(1.01), f32(0.3)) and g["dims"] == [1, 1, 1]


def test_sixteen_cell_clamp():
    x = (np.random.RandomState(2).randint(0, 16, (2000, 3)) / 16).astype(f32)
    x[0], x[1] = 0, f32(15 / 16)
    g = R.geometry(x, 0.001)
    assert g["dims"] == [16, 16, 16] and g["h"] == f32(1 / 16)
    c = R.cells(np.array([[-5, 0.5, 9]], f32), g, query=True)[0]
    assert list(c) == [-1, 8, 16]


def test_layout_and_fit_edges():
    assert R.bg_dual_layout(4863) and not R.bg_dual_layout(4864)
    assert R.bg_fits(9727) and not R.bg_fits(9728)


def test_batch_rule_and_group_pick():
    assert R.batch_uses_grid([1, 0, 0, 0]) and not R.batch_uses_grid([1, 0, 0, 0, 0])
    assert R.batch_uses_grid([1] * 256 + [0] * 2000)  # judged on the first 1024
    assert R.pick_group(1, 1) == 32 and R.pick_group(1, 270336) == 1 and R.pick_group(4, 1000, forced=8) == 8
    assert R.pick_group(1, 33792) == 8


def test_global_flag_reasons():
    rs = np.random.RandomState(3)
    u = rs.random_sample((4000, 3)).astype(f32)
    assert R.global_flag(u, 0.02, 32) == (True, "grid")
    assert R.global_flag(u[:2047], 0.02, 32)[1] == "small_n"
    assert R.global_flag(u, 0.3, 32)[1] == "prune"
    assert R.global_flag(u, 0.06, 4)[1] == "expect"
    heavy = u.copy()
    heavy[:300] = 0.5
    assert R.global_flag(heavy, 0.02, 64)[1] == "heavy"
    lumpy = u.copy()  # half the cloud in 1/64 of the box: sparse on average, dense where the points are
    lumpy[:1900] = (0.5 + u[:1900] * 0.25).astype(f32)
    assert R.global_flag(lumpy, 0.05, 16)[1] == "expect_local"


def _bg(x, q, r, s, stride=None):
    cl = R.BgCloud(x, r, stride or len(x))
    h = R.hit_rows(r, x, q[None])[0]
    return cl, R.bg_query(cl, q, h, s)


def test_ball_group_query_regimes():
    rs = np.random.RandomState(4)
    u = rs.random_sample((4000, 3)).astype(f32)
    q = np.array([0.5, 0.5, 0.5], f32)
    cl, t = _bg(u, q, 0.03, 32)
    assert cl.use_grid and cl.dual and {"walk_balanced", "sort1", "short_row"} <= t
    full = u.copy()
    full[:1100] = q  # a quarter of the cloud in the neighbourhood
    assert "scan_instead" in _bg(full, q, 0.03, 32)[1]
    assert "query_nonfinite" in _bg(u, np.array([np.nan, 0.5, 0.5], f32), 0.03, 32)[1]
    crowd = u.copy()
    crowd[:600] = q
    assert {"walk_crowded", "overflow_cost", "scan_shared_buffered"} <= _bg(crowd, q, 0.03, 64)[1]
    assert {"overflow_nsample", "scan_global_unbuffered"} <= _bg(crowd, q, 0.03, 300, stride=9000)[1]
    big = rs.random_sample((9000, 3)).astype(f32)
    blob = (q + rs.uniform(-1, 1, (1200, 3)) * 0.04).astype(f32)
    big[:1200] = blob[np.argsort(-blob[:, 2], kind="stable")]
    assert {"compact", "full_row"} <= _bg(big, q, 0.04, 128)[1]
    assert "scan_shared_unbuffered" in _bg(u[:100], q, 0.3, 257)[1]
    assert "empty_row" in _bg(u, np.array([5, 5, 5], f32), 0.03, 8)[1]


def test_brute_force_early_exit():
    x = np.zeros((5000, 3), f32)
    h = R.hit_rows(0.1, x, np.zeros((8, 3), f32))
    assert {"G32", "multi_tile", "early_exit"} <= R.bf_tags(5000, 8, 16, 32, h)
    assert "early_exit" not in R.bf_tags(5000, 8, 4097, 32, h)


# ------------------------------------------------------------------------------------------ soundness of the grid
def _adversarial(rs, kind):
    n = int(rs.randint(1, 160))
    if kind == "shell":
        c = rs.random_sample(3).astype(f32)
        r = f32(rs.uniform(0.01, 0.3))
        x = rs.random_sample((n, 3)).astype(f32)
        for k in range(n):
            a = rs.randint(3)
            x[k] = c
            x[k, a] = f32(c[a] + rs.choice([-1, 1]) * _ulps(r, int(rs.randint(-8, 9))))
        return x, r, np.concatenate([c[None], x[:4]])
    if kind == "edges":  # points on mn + k h: 15 cells of 1/16, h = emax / 15
        x = (rs.randint(0, 16, (n, 3)) / 16).astype(f32)
        x[0], x[-1] = 0, f32(15 / 16)
        r = f32(rs.choice([1 / 16 / 1.01, 0.05, 0.06]))
        return x, r, x[rs.randint(0, n, 8)]
    if kind == "offset":
        x = (f32(1e4) + rs.random_sample((n, 3)) * rs.choice([1e-2, 1.0])).astype(f32)
        r = f32(rs.uniform(1e-4, 1e-2))
        return x, r, x[rs.randint(0, n, 8)]
    if kind == "degenerate":
        x = np.zeros((n, 3), f32) + rs.random_sample(3).astype(f32)
        for a in rs.choice(3, int(rs.randint(0, 3)), replace=False):
            x[:, a] = rs.random_sample(n)
        r = f32(rs.uniform(0.01, 0.5))
        return x, r, x[rs.randint(0, n, 8)]
    if kind == "outside":
        x = rs.random_sample((n, 3)).astype(f32)
        r = f32(rs.uniform(0.01, 0.4))
        q = (rs.random_sample((8, 3)) * 3 - 1).astype(f32)
        return x, r, q
    x = (rs.random_sample((n, 3)) * rs.uniform(0.5, 50, 3)).astype(f32)  # "clamp": 16 cells on some axis
    r = f32(rs.uniform(1e-3, 0.05))
    return x, r, x[rs.randint(0, n, 8)]


KINDS = ["shell", "edges", "offset", "degenerate", "outside", "clamp"]


@pytest.mark.parametrize("kind", KINDS)
def test_every_hit_is_in_the_query_neighbourhood(kind):
    rs = np.random.RandomState(100 + KINDS.index(kind))
    checked = 0
    for _ in range(600):
        x, r, q = _adversarial(rs, kind)
        g = R.geometry(x, r)
        assert g["finite_box"]
        pc = R.cells(x, g)
        qc = R.cells(q, g, query=True)
        hits = R.hit_rows(r, x, q)
        for j in range(len(q)):
            k = np.nonzero(hits[j])[0]
            lo = np.maximum(qc[j] - 1, 0)
            hi = np.minimum(qc[j] + 1, np.array(g["dims"]) - 1)
            assert np.all((pc[k] >= lo) & (pc[k] <= hi)), (kind, r, q[j], x[k][:4])
            checked += len(k)
    assert checked > 0
