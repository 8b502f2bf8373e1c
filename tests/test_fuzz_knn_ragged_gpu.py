"""A short, fixed-seed slice of tests/fuzz_knn_ragged_gpu.py: knn_point and the kNN set-abstraction layer with per-cloud
lengths against the contract's restatement on the C oracle, bit for bit (tests/test_fuzz_knn_ragged_cpu.py checks which
regimes these seeds reach)."""
import pytest

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("seed", [81, 82, 83])
def test_random_ragged_knn_cases_match_oracle(dev, seed):
    import fuzz_knn_ragged_gpu as G
    assert seed in G.SLICE_SEEDS
    counts, fails = G.run(seed, G.SLICE_ITERATIONS)
    assert counts == {name: G.SLICE_ITERATIONS // len(G.CASES) for name in G.CASES}
    assert not fails, fails
