"""A fixed-seed slice of tests/fuzz_fps_gpu.py: every FPS kernel instantiation, dense and ragged, the planner's own
choice, the global-scratch fallback over more than 32 clouds and the dispatcher's refusals, against the C oracle bit
for bit (tests/test_fuzz_fps_cpu.py checks which kernels, tie stages and data regimes these seeds reach).  Also the
record of cluster capacities the CPU replay plans with."""
import pytest

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("seed", [81, 82])
def test_random_fps_cases_match_oracle(dev, seed):
    import fuzz_fps_gpu as F
    assert seed in F.SLICE_SEEDS
    counts, fails = F.run(seed, F.SLICE_ITERATIONS)
    per_block = {name: F.SCHEDULE.count(name) for name in F.CASES}
    assert counts == {name: F.SLICE_ITERATIONS // len(F.SCHEDULE) * k for name, k in per_block.items()}
    assert not fails, fails


def test_h100_cluster_capacity_record(dev):
    """fps_regimes.H100_CAPACITY holds pn2_fps_cluster_capacity for every cluster plan plan_fps asks about on an H100"""
    import torch

    import fps_regimes as R
    import test_fuzz_fps_cpu as C
    from pointnet2_b200 import _lib
    if torch.cuda.get_device_properties(dev).multi_processor_count != R.SMS:
        pytest.skip("the record is of an H100 with 132 SMs")
    lib = _lib.load()
    asked = set()

    def cap(t, pp, c, packed):
        asked.add((t, pp, c))
        return int(lib.pn2_fps_cluster_capacity(t, pp, c))

    for b in (1, 2, 3, 4, 5, 7, 8, 9, 16, 17, 33, 66, 67, 132, 133, 500):
        for n in C.sweep_sizes():
            R.plan_fps(b, n, capacity=cap)
    live = {k: int(lib.pn2_fps_cluster_capacity(*k)) for k in sorted(asked)}
    assert live == {k: R.H100_CAPACITY.get(k) for k in live}, live
