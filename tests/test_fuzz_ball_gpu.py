"""A short, fixed-seed slice of tests/fuzz_ball_gpu.py: query_ball_point in every mode, ball_group and the ball-query
set-abstraction layer against the C oracle, bit for bit (tests/test_fuzz_ball_cpu.py checks which regimes these seeds
reach).  Also the regression test for clouds that are NaN on a whole axis."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("seed", [71, 75, 76])
def test_random_ball_cases_match_oracle(dev, seed):
    import fuzz_ball_gpu as F
    assert seed in F.SLICE_SEEDS
    counts, fails = F.run(seed, F.SLICE_ITERATIONS)
    assert counts == {name: F.SLICE_ITERATIONS // len(F.CASES) for name in F.CASES}
    assert not fails, fails


@pytest.mark.parametrize("path", ["ball_group", "global_grid"])
def test_nan_axis_cloud_is_a_hit_in_every_ball(dev, path):
    """Every point NaN in x, spread in y and z: each point is a hit in every ball (the reference's fmaxf(NaN, 1e-20f) <
    radius), so every row holds the first nsample indices.  The box was finite on y and z while x's extent was
    inf - inf = NaN, which emax's fmaxf skipped: the shared-memory and global grids binned the cloud and missed every
    point outside the query's y-z neighbourhood."""
    import torch

    import fuzz_ball_gpu as F
    import ball_regimes as R
    from oracle import oracle as O
    from pointnet2_b200 import _lib
    from pointnet2_b200.sa_layer import ball_group
    from pointnet2_b200.tf_grouping import query_ball_point

    rs = np.random.RandomState(7)
    b, n, m, s, r = 2, 3000, 64, 64, 0.05
    x = rs.random_sample((b, n, 3)).astype(np.float32)
    x[:, :, 0] = np.float32(np.nan)
    q = x[:, rs.randint(0, n, m)].copy()
    q[:, :, 0] = rs.random_sample((b, m)).astype(np.float32)
    assert not R.geometry(x[0], r)["finite_box"]
    lib = _lib.load()
    if path == "ball_group":
        idx, cnt, _ = ball_group(r, s, F.T(x), F.T(q), want_grouped=False)
    else:
        try:
            lib.pn2_set_bq_mode(2)
            idx, cnt = query_ball_point(r, s, F.T(x), F.T(q))
        finally:
            lib.pn2_set_bq_mode(0)
    torch.cuda.synchronize()
    oi, oc = O.oracle_query_ball_point(r, s, x, q)
    assert (oc == s).all() and (oi == np.arange(s)).all()
    assert np.array_equal(F.N(idx), oi) and np.array_equal(F.N(cnt), oc)
