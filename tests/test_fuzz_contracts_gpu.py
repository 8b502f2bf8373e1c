"""A short, fixed-seed slice of tests/fuzz_contracts_gpu.py (per-cloud lengths, 16-bit features, deterministic
gradients, the split grid ball query against the oracle), and the regression tests of what it found."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("seed", [31, 32, 33])
def test_random_contract_cases_match_oracle(dev, seed):
    import fuzz_contracts_gpu as F
    assert seed in F.SLICE_SEEDS  # tests/test_fuzz_contracts_cpu.py checks what these seeds cover
    counts, fails = F.run(seed, F.SLICE_ITERATIONS)
    assert counts == {name: F.SLICE_ITERATIONS // len(F.CASES) for name in F.CASES}
    assert not fails, fails


def test_grid_build_refuses_a_radius_no_distance_passes(dev):
    """pn2_ball_grid_build used to launch at radius <= 1e-20, where its query half (and the whole-path entry's grid)
    refuse; both halves now return cudaErrorInvalidValue there, as documented."""
    from pointnet2_b200 import _lib, workloads as W
    from pointnet2_b200._tensor import ptr, stream_ptr
    lib = _lib.load()
    b, n = 2, 4096
    x = torch.from_numpy(W.cloud_uniform(b, n, 1)).to(dev)
    wsb = int(lib.pn2_query_ball_point_workspace_bytes(b, n))
    ws = torch.empty(wsb, dtype=torch.uint8, device=dev)
    for r in (1e-20, 1e-30, float(np.float32(1e-20))):
        assert lib.pn2_ball_grid_build(b, n, r, 16, ptr(x), ptr(ws), wsb, stream_ptr(dev)) == 1
    assert lib.pn2_ball_grid_build(b, n, 0.1, 16, ptr(x), ptr(ws), wsb, stream_ptr(dev)) == 0
    torch.cuda.synchronize(dev)
