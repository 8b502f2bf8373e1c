"""A short, fixed-seed slice of tests/fuzz_knn_gpu.py: knn_point and the kNN set-abstraction layer against the
selection-sort oracle, bit for bit (tests/test_fuzz_knn_cpu.py checks which regimes these seeds reach)."""
import pytest

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("seed", [61, 62, 63])
def test_random_knn_cases_match_oracle(dev, seed):
    import fuzz_knn_gpu as F
    assert seed in F.SLICE_SEEDS
    counts, fails = F.run(seed, F.SLICE_ITERATIONS)
    assert counts == {name: F.SLICE_ITERATIONS // len(F.CASES) for name in F.CASES}
    assert not fails, fails
