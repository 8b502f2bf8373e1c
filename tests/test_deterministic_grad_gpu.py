"""The group_point / gather_point gradients without atomics (pn2_group_point_grad_det, pn2_gather_point_grad_det) and
torch.use_deterministic_algorithms routing through the autograd ops: every point's rows are added in ascending entry
order, so the result is run-to-run identical and equals the reference's group_point_grad_cpu bit for bit, long lists
(> 256 entries on one point) included."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import golden as G
from oracle import oracle as O
from pointnet2_b200 import _lib, workloads as W
from pointnet2_b200.pointnet_util import group_and_concat
from pointnet2_b200.tf_grouping import group_point
from pointnet2_b200.tf_sampling import gather_point

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CODES = {torch.float32: 0, torch.bfloat16: 1, torch.float16: 2}


def T(a, dev):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


def ball_idx(gen, b, n, m, r, s, seed):
    """a set-abstraction layer's ball-query index, computed on the host: FPS centres of one cloud of `gen`"""
    xyz = W.DISTRIBUTIONS[gen](b, n, seed)
    ctr = np.stack([xyz[i][O.oracle_fps(m, xyz[i:i + 1])[0]] for i in range(b)])
    idx, _ = O.oracle_query_ball_point(r, s, xyz, ctr)
    return idx


def det_grad(go, idx, n, misalign=False):
    """pn2_group_point_grad_det(_typed) on a (b, m, s, c) grad_out; misalign: both bases one element past 16 bytes"""
    lib = _lib.load()
    b, m, s, c = go.shape
    if misalign:
        go = torch.cat([go.new_zeros(1), go.reshape(-1)])[1:].view(b, m, s, c)
    gp = torch.full((b * n * c + 1,), 7.0, dtype=go.dtype, device=go.device)  # overwritten: no zero-fill
    gp = (gp[1:] if misalign else gp[:-1]).view(b, n, c)
    wsb = int(lib.pn2_group_point_grad_det_workspace_bytes(b, n, m, s))
    ws = torch.empty(wsb, dtype=torch.uint8, device=go.device)
    rc = lib.pn2_group_point_grad_det_typed(CODES[go.dtype], b, n, c, m, s, go.data_ptr(), idx.data_ptr(), gp.data_ptr(),
                                            ws.data_ptr(), wsb, None)
    assert rc == 0
    torch.cuda.synchronize()
    return gp


# (gen, b, n, m, r, s): cfg2's layer, cfg3 L1 r=0.4 S=128 (lists of thousands of entries), cfg3 L2 r=0.4 S=64, duplicates
LAYERS = [("U", 2, 4096, 1024, 0.1, 32), ("S", 2, 1024, 512, 0.4, 128), ("S", 2, 512, 128, 0.4, 64), ("D", 2, 1024, 256, 0.2, 32)]


@pytest.mark.parametrize("gen,b,n,m,r,s", LAYERS)
@pytest.mark.parametrize("c", [3, 7, 64, 320])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.float16])
def test_group_point_grad_det_equals_the_ordered_sum(dev, gen, b, n, m, r, s, c, dtype):
    idx = ball_idx(gen, b, n, m, r, s, 300)
    go = W.features(b, m * s, c, 301).reshape(b, m, s, c)
    tgo = T(go, dev).to(dtype)
    want = O.oracle_group_point_grad((b, n, c), idx, tgo.float().cpu().numpy())  # ascending (j, k), float32
    want = torch.from_numpy(want).to(dtype)
    ti = T(idx, dev)
    for misalign in (False, True):
        got = det_grad(tgo, ti, n, misalign).cpu()
        assert torch.equal(got.view(torch.int16 if dtype != torch.float32 else torch.int32),
                           want.view(torch.int16 if dtype != torch.float32 else torch.int32)), (gen, c, dtype, misalign)
    if gen == "S" and s == 128:
        assert max(np.bincount(idx[i].ravel(), minlength=n).max() for i in range(b)) > 256  # the long-list kernel ran


def test_every_entry_on_one_point(dev):
    """m*S entries on one list: one long list holds the whole cloud"""
    b, n, m, s, c = 2, 100, 64, 32, 36
    idx = np.full((b, m, s), 17, np.int32)
    idx[1] = 99
    go = W.features(b, m * s, c, 302).reshape(b, m, s, c)
    want = O.oracle_group_point_grad((b, n, c), idx, go)
    got = det_grad(T(go, dev), T(idx, dev), n)
    np.testing.assert_array_equal(got.cpu().numpy(), want)


def test_two_calls_give_identical_bits(dev):
    b, n, m, s, c = 4, 1024, 512, 128, 64
    idx = T(ball_idx("S", b, n, m, 0.4, s, 303), dev)
    go = torch.randn((b, m, s, c), device=dev)
    a, bb = det_grad(go, idx, n), det_grad(go, idx, n)
    assert torch.equal(a.view(torch.int32), bb.view(torch.int32))


def test_gather_point_grad_det_equals_the_ordered_sum(dev):
    lib = _lib.load()
    b, n, m = 4, 4096, 1024
    rs = np.random.RandomState(304)
    idx = rs.randint(0, 300, (b, m)).astype(np.int32)  # ~3.4 entries a point, some points untouched
    idx[0, :600] = 5  # and one list longer than 256
    og = W.features(b, m, 3, 305)
    want = O.oracle_gather_point_grad((b, n, 3), idx, og)
    g = torch.full((b, n, 3), 7.0, device=dev)
    wsb = int(lib.pn2_group_point_grad_det_workspace_bytes(b, n, m, 1))
    ws = torch.empty(wsb, dtype=torch.uint8, device=dev)
    ti, tog = T(idx, dev), T(og, dev)
    assert lib.pn2_gather_point_grad_det(b, n, m, tog.data_ptr(), ti.data_ptr(), g.data_ptr(), ws.data_ptr(), wsb, None) == 0
    np.testing.assert_array_equal(g.cpu().numpy(), want)
    # through autograd, with torch's determinism switched on
    inp = T(W.cloud_uniform(b, n, 306), dev).requires_grad_(True)
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        (gather_point(inp, ti) * tog).sum().backward()
    finally:
        torch.use_deterministic_algorithms(prev)
    np.testing.assert_array_equal(inp.grad.cpu().numpy(), want)


# full-size layers against the reference's own CPU function (stored records: oracle/golden.py)
FULL = {"cfg3_L2_r0.4_S64_C320": ("S", 32, 1024, 512, 128, 0.4, 64, 320), "cfg4_SA256_C64": ("D", 16, 8192, 1024, 256, 0.2, 32, 64)}


def full_size_inputs(key):
    gen, b, n0, n, m, r, s, c = FULL[key]
    xyz = W.DISTRIBUTIONS[gen](b, n0, 100)
    l1 = np.stack([xyz[i][O.oracle_fps(n, xyz[i:i + 1])[0]] for i in range(b)])  # the layer's input: the previous FPS
    ctr = np.stack([l1[i][O.oracle_fps(m, l1[i:i + 1])[0]] for i in range(b)])
    idx, _ = O.oracle_query_ball_point(r, s, l1, ctr)
    go = W.features(b, m * s, c, 307).reshape(b, m, s, c)
    return (b, n, c), idx, go


@pytest.mark.parametrize("key", sorted(FULL))
def test_full_size_group_point_grad_det_matches_reference(dev, key):
    shape, idx, go = full_size_inputs(key)
    got = det_grad(T(go, dev), T(idx, dev), shape[1]).cpu().numpy()
    G.expect(f"group_point_grad_det_{key}", lambda: dict(grad=O.refcpu_group_point_grad(shape, idx, go)), grad=got)


def test_det_grad_beyond_2_to_31_elements(dev):
    free, _ = torch.cuda.mem_get_info(dev)
    if free < 16 * (1 << 30):
        pytest.skip("needs 16 GiB of free device memory")
    b, n, m, s, c = 2, 1536, 16384, 128, 520  # 2 * 2^21 rows of 520 floats: > 2^31 elements
    g = torch.Generator(device=dev).manual_seed(8)
    idx = torch.randint(0, n, (b, m, s), device=dev, generator=g, dtype=torch.int32)
    go = torch.randn((b, m, s, c), device=dev, generator=g)
    assert go.numel() > (1 << 31)
    got = det_grad(go, idx, n)
    want = torch.zeros((b * n, c), device=dev, dtype=torch.float64)
    flat = (torch.arange(b, device=dev).view(b, 1, 1) * n + idx.long()).view(-1)
    for k in range(0, c, 130):  # float64 sums in slices of channels
        want[:, k:k + 130] = torch.zeros((b * n, min(130, c - k)), device=dev, dtype=torch.float64).index_add_(
            0, flat, go.view(-1, c)[:, k:k + 130].double())
    assert torch.allclose(got.view(-1, c).double(), want, rtol=1e-4, atol=1e-3)
    last = idx[-1, -1, -1].item()  # the last entry of the last cloud reaches its row
    assert got[-1, last].abs().sum().item() > 0


# ------------------------------------------------------------------------------------------------ through autograd
def _steps_child(name, amp, det):
    """two SGD steps of a network in a fresh process; prints a SHA-256 of the last step's parameter gradients"""
    code = f"""
import hashlib, sys, torch
sys.path.insert(0, {ROOT!r})
from pointnet2_b200 import nets, workloads as W
torch.use_deterministic_algorithms({det})
torch.manual_seed(0)
dev = torch.device("cuda:0")
net = {{"cls_ssg": nets.PointNet2ClsSSG, "cls_msg": nets.PointNet2ClsMSG, "sem_seg": nets.PointNet2SemSeg}}[{name!r}]().to(dev)
b, n = (2, 2048) if {name!r} == "sem_seg" else (4, 1024)
xyz = torch.from_numpy(W.cloud_surface(b, n, 400)).to(dev)
opt = torch.optim.SGD(net.parameters(), lr=0.01)
for _ in range(2):
    opt.zero_grad()
    with torch.autocast(device_type="cuda", dtype=torch.bfloat16, enabled={amp == 'bf16'}):
        pred, _ = net(xyz)
        loss = pred.float().square().mean()
    loss.backward()
    opt.step()
h = hashlib.sha256()
for p in net.parameters():
    h.update(p.grad.detach().float().cpu().numpy().tobytes())
print(h.hexdigest())
"""
    env = dict(os.environ, CUBLAS_WORKSPACE_CONFIG=":4096:8")
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, env=env, cwd=ROOT, timeout=900)
    assert r.returncode == 0, r.stderr[-3000:]
    return r.stdout.strip().splitlines()[-1]


@pytest.mark.parametrize("name", ["cls_ssg", "cls_msg", "sem_seg"])
@pytest.mark.parametrize("amp", ["fp32", "bf16"])
def test_training_steps_are_bit_reproducible_in_deterministic_mode(name, amp):
    assert _steps_child(name, amp, True) == _steps_child(name, amp, True)


@pytest.mark.parametrize("det", [False, True])
def test_autograd_gradients_in_both_modes(dev, det):
    """deterministic mode off: the atomic kernels as before; on: the ordered sums.  Both hold the oracle's values to the
    float32 tolerance of a reordered sum, and deterministic mode holds them bit for bit."""
    b, n, m, s, c = 2, 1024, 512, 128, 64
    idx = ball_idx("S", b, n, m, 0.4, s, 309)
    go = W.features(b, m * s, c, 310).reshape(b, m, s, c)
    want = O.oracle_group_point_grad((b, n, c), idx, go)
    pts = T(W.features(b, n, c, 311), dev).requires_grad_(True)
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(det)
    try:
        (group_point(pts, T(idx, dev)) * T(go, dev)).sum().backward()
    finally:
        torch.use_deterministic_algorithms(prev)
    got = pts.grad.cpu().numpy()
    if det:
        np.testing.assert_array_equal(got, want)
    else:
        np.testing.assert_allclose(got, want, rtol=1e-5, atol=1e-5 * float(np.abs(want).max()))


def test_group_and_concat_skips_the_coordinate_scatter(dev):
    b, n, m, s, c = 2, 512, 128, 32, 16
    idx = T(ball_idx("S", b, n, m, 0.2, s, 308), dev)
    xyz = T(W.cloud_surface(b, n, 308), dev)
    new_xyz = xyz[:, :m].contiguous()
    pts = torch.randn((b, n, c), device=dev, requires_grad=True)
    before = _lib.launch_count()
    out, _ = group_and_concat(xyz, new_xyz, pts, idx, xyz_first=False)
    out.sum().backward()
    torch.cuda.synchronize()
    assert _lib.launch_count() - before == 2  # the forward and one feature scatter
    cnt = torch.stack([torch.bincount(idx[i].reshape(-1).long(), minlength=n) for i in range(b)]).float()
    assert torch.equal(pts.grad, cnt.unsqueeze(2).expand(b, n, c))  # each point's reference count, exactly
