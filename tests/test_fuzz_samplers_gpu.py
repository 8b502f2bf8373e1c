"""A fixed-seed slice of tests/fuzz_samplers_gpu.py: voxel grouping, shape batches, training crops and virtual scans
against their numpy oracles, with poisoned and guarded outputs, device seeds and refused calls
(tests/test_fuzz_samplers_cpu.py checks which select passes and regimes these seeds reach), and the workspace sizes
against tests/select_regimes.py."""
import pytest

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("seed", [81, 82])
def test_random_sampler_cases_match_oracles(dev, seed):
    import fuzz_samplers_gpu as F
    assert seed in F.SLICE_SEEDS
    counts, fails = F.run(seed, F.SLICE_ITERATIONS)
    assert counts == {name: F.SLICE_ITERATIONS // len(F.SCHEDULE) * F.SCHEDULE.count(name) for name in set(F.SCHEDULE)}
    assert not fails, fails


def test_workspace_bytes_match_the_restatement(dev):
    import select_regimes as R
    from pointnet2_b200 import _lib
    lib = _lib.load()
    for b, n, dim, dims in ((1, 1, 1, 3), (1, 128, 3, 3), (2, 129, 3, 3), (3, 40000, 12, 2), (2, 1 << 30, 3, 3),
                            (2, 10, 1025, 3), (1, 5, 46341, 2), (4, 100000, 31, 2)):
        assert int(lib.pn2_voxel_group_workspace_bytes(b, n, dim, dims)) == R.voxel_workspace_bytes(b, n, dim, dims)
    for b, npoints in ((1, 1), (7, 8192), (65535, 16384), (65536, 1), (2, 16385), (1000, 16384)):
        assert int(lib.pn2_scene_crops_workspace_bytes(b, npoints)) == R.crops_workspace_bytes(b, npoints)
    for b, ms, npoints in ((1, 1, 1), (3, 150000, 8192), (4096, 100, 16384), (4097, 100, 1), (2, 100, 16385)):
        assert int(lib.pn2_virtual_scans_workspace_bytes(b, ms, npoints)) == R.vscan_workspace_bytes(b, ms, npoints)
