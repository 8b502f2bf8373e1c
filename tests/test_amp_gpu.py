"""The networks under torch.autocast: bfloat16, and float16 with a GradScaler.  The learned layers produce 16-bit
features, which the grouping and interpolation kernels take as they are; the geometry stays float32."""
import importlib.util
import os

import numpy as np
import pytest
import torch

from pointnet2_b200 import nets, workloads as W
from pointnet2_b200.pointnet_util import pointnet_sa_module

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NETS = [("cls_ssg", 4, 1024, (4, 40)), ("cls_msg", 3, 1024, (3, 40)), ("sem_seg", 2, 2048, (2, 2048, 21))]


def _net(name, dev):
    return {"cls_ssg": nets.PointNet2ClsSSG, "cls_msg": nets.PointNet2ClsMSG, "sem_seg": nets.PointNet2SemSeg}[name]().to(dev)


@pytest.mark.parametrize("name,b,n,out", NETS)
@pytest.mark.parametrize("amp", ["bf16", "fp16"])
def test_network_trains_a_step_under_autocast(dev, name, b, n, out, amp):
    torch.manual_seed(0)
    net = _net(name, dev)
    xyz = torch.from_numpy(W.cloud_surface(b, n, 400)).to(dev)
    dt = torch.bfloat16 if amp == "bf16" else torch.float16
    # float16: the GradScaler's loop — a step whose scaled gradients overflow float16 is skipped and the scale halved
    scaler = torch.amp.GradScaler("cuda") if amp == "fp16" else None
    opt = torch.optim.SGD(net.parameters(), lr=0.0)
    for _ in range(24 if scaler else 1):
        opt.zero_grad(set_to_none=True)
        with torch.autocast(device_type="cuda", dtype=dt):
            pred, _ = net(xyz)
            loss = pred.float().square().mean()
        assert tuple(pred.shape) == out and pred.dtype == dt
        assert bool(torch.isfinite(loss))
        if scaler is None:
            loss.backward()
            break
        scaler.scale(loss).backward()
        scaler.unscale_(opt)
        finite = all(bool(torch.isfinite(p.grad).all()) for p in net.parameters() if p.grad is not None)
        scaler.step(opt)
        scaler.update()
        if finite:
            break
    assert scaler is None or scaler.get_scale() >= 1.0
    bad = [k for k, p in net.named_parameters() if p.grad is None or not bool(torch.isfinite(p.grad).all())]
    assert not bad, bad
    first = next(net.parameters())  # the gradient reaches the first layer through the 16-bit backward kernels
    assert float(first.grad.abs().sum()) > 0


def test_sa_module_idx_is_the_float32_idx_under_autocast(dev):
    torch.manual_seed(0)
    xyz = torch.from_numpy(W.cloud_surface(4, 1024, 401)).to(dev)
    mlp1, mlp2 = nets.SharedMLP(3, [32, 64]).to(dev), nets.SharedMLP(64 + 3, [64, 128]).to(dev)
    runs = []
    for amp in (False, True):
        with torch.autocast(device_type="cuda", dtype=torch.bfloat16, enabled=amp):
            l1_xyz, l1_points, idx1 = pointnet_sa_module(xyz, None, 256, 0.2, 32, mlp1)
            _, l2_points, idx2 = pointnet_sa_module(l1_xyz, l1_points, 64, 0.4, 32, mlp2)
        runs.append((idx1, idx2, l1_points.dtype, l2_points.dtype))
    (a1, a2, f1, f2), (b1, b2, h1, h2) = runs
    assert f1 == f2 == torch.float32 and h1 == h2 == torch.bfloat16
    assert torch.equal(a1, b1) and torch.equal(a2, b2)


def test_training_under_bf16_autocast_reduces_the_loss(dev):
    """the same bar as the float32 training test (test_nets_gpu.py)"""
    spec = importlib.util.spec_from_file_location("train_ddp_demo", os.path.join(ROOT, "tools", "train_ddp_demo.py"))
    demo = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(demo)
    torch.manual_seed(0)
    net = nets.PointNet2ClsSSG(3).to(dev)
    opt = torch.optim.Adam(net.parameters(), lr=1e-3)
    rs = np.random.RandomState(7)
    losses = []
    for _ in range(24):
        xyz, lab = demo.synthetic_shapes(16, 512, 3, rs)
        with torch.autocast(device_type="cuda", dtype=torch.bfloat16):
            pred, _ = net(torch.from_numpy(xyz).to(dev))
            loss = nets.cls_loss(pred, torch.from_numpy(lab).to(dev))
        opt.zero_grad()
        loss.backward()
        opt.step()
        losses.append(float(loss.detach()))
    assert np.mean(losses[-6:]) < 0.7 * np.mean(losses[:6]), losses
