"""A fixed-seed slice of tests/fuzz_masked_bn_gpu.py: every <T, V, VEC> instantiation of masked_bn.cu, plain and
max-pooled, forward and backward, against the exact float32 oracle (tests/test_fuzz_masked_bn_cpu.py checks which
instantiations and regimes these seeds reach), the workspace sizes against tests/bn_regimes.py, and the statistics of
a batch without a real row."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("seed", [61, 62])
def test_random_masked_bn_cases_match_oracle(dev, seed):
    import fuzz_masked_bn_gpu as F
    assert seed in F.SLICE_SEEDS
    counts, fails = F.run(seed, F.SLICE_ITERATIONS)
    assert counts == {name: F.SLICE_ITERATIONS // len(F.SCHEDULE) * F.SCHEDULE.count(name) for name in set(F.SCHEDULE)}
    assert not fails, fails


def test_slice_was_planned_with_this_devices_sm_count(dev):
    """the second grid-stride trips the CPU replay counts on assume bn_regimes.SMS multiprocessors"""
    import bn_regimes as R
    if torch.cuda.get_device_properties(dev).multi_processor_count != R.SMS:
        pytest.skip("the slice's grid-stride trips were planned for an H100 SXM's 132 SMs")


def test_workspace_bytes_match_the_restatement(dev):
    import bn_regimes as R
    from pointnet2_b200 import _lib
    lib = _lib.load()
    for rows in (0, 1, 255, 256, 257, 8192, 8193, 100000):
        for c in (1, 3, 4, 8, 33, 132, 260, 1024):
            assert int(lib.pn2_masked_bn_workspace_bytes(rows, c)) == R.workspace_bytes(rows, c), (rows, c)
    for b, n, c in ((1, 1, 1), (70, 33, 132), (33, 1000, 4), (2, 5, 1024), (4096, 3, 7), (65536, 32768, 3)):
        assert int(lib.pn2_masked_bn_relu_max_workspace_bytes(b, n, c)) == R.max_workspace_bytes(b, n, c), (b, n, c)


@pytest.mark.parametrize("fmt", ["f32", "bf16"])
def test_no_real_row_gives_the_statistics_masked_batch_norm_gives(dev, fmt):
    """every keep 0: save_mean, save_invstd and both running buffers NaN (the mean is 0 / 0, as in
    layers.masked_batch_norm), y 0; the backward writes dx 0 and dgamma = dbeta = 0"""
    from pointnet2_b200 import layers
    dt = torch.float32 if fmt == "f32" else torch.bfloat16
    for c in (3, 8):
        x = torch.randn(300, c, device=dev).to(dt).requires_grad_(True)
        keep = torch.zeros(300, dtype=torch.bool, device=dev)
        bn = torch.nn.BatchNorm1d(c).to(dev).train()
        ref = torch.nn.BatchNorm1d(c).train()
        y = layers.masked_batch_norm_relu(bn, x, keep)
        layers.masked_batch_norm(ref, torch.zeros(300, c), keep.cpu().reshape(-1, 1))
        assert torch.isnan(bn.running_mean).all() and torch.isnan(bn.running_var).all()
        assert torch.isnan(ref.running_mean).all() and torch.isnan(ref.running_var).all()
        assert int(bn.num_batches_tracked) == 1 and (y == 0).all()
        y.backward(torch.ones_like(y))
        assert (x.grad == 0).all() and (bn.weight.grad == 0).all() and (bn.bias.grad == 0).all()
        _, mean, invstd = layers.masked_bn_relu_forward_launch(x.detach(), None, None, keep.view(torch.uint8), 1e-5, 0.1,
                                                               None, None, None)
        assert np.isnan(mean.cpu().numpy()).all() and np.isnan(invstd.cpu().numpy()).all()
