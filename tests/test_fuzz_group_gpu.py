"""A fixed-seed slice of tests/fuzz_group_gpu.py: every kernel instantiation of group.cu, scatter_det.cu and
interpolate.cu's interpolation against the C oracle and the exact ordered sums of tests/group_regimes.py
(tests/test_fuzz_group_cpu.py checks which kernels and regimes these seeds reach).  Also one child process with
group_point's flat kernel and one CTA per SM, so that the copies take many grid-stride trips at small sizes."""
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu

TESTS = os.path.dirname(os.path.abspath(__file__))


@pytest.mark.parametrize("seed", [91, 92])
def test_random_group_cases_match_oracle(dev, seed):
    import fuzz_group_gpu as F
    assert seed in F.SLICE_SEEDS
    counts, fails = F.run(seed, F.SLICE_ITERATIONS)
    assert counts == {name: F.SLICE_ITERATIONS // len(F.SCHEDULE) * F.SCHEDULE.count(name) for name in set(F.SCHEDULE)}
    assert not fails, fails


def test_flat_kernel_and_one_cta_per_sm(dev, tmp_path):
    """PN2_GROUP_MODE / PN2_GROUP_CTAS are read once per process, so they are set for a child of its own"""
    env = dict(os.environ, PN2_GROUP_MODE="1", PN2_GROUP_CTAS="1")
    out = tmp_path / "flat.json"
    r = subprocess.run([sys.executable, os.path.join(TESTS, "fuzz_group_gpu.py"), "--seed", "93", "--seconds", "600",
                        "--iterations", "56", "--json", str(out)], env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-4000:] + r.stderr[-4000:]
