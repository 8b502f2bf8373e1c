"""GPU tests of the part segmentation nets (PointNet2PartSeg, PointNet2PartSegMSG): forward and backward in float32 and
under bf16 autocast, inert padding with per-shape lengths, each shape of a padded batch against the shape alone,
training on synthetic part data, deterministic gradients, and the evaluation helpers on the device."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from pointnet2_b200 import nets, workloads as W
from pointnet2_b200.layers import row_mask
from test_ragged_fp_gpu import T, bits, both_paddings, pad

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
N = 2048
# very short shapes (fewer points than sa1's 512 centroids, down to one) next to a full one
LENGTHS = [1, 20, 63, 300, 511, N]
NETS = ["PointNet2PartSeg", "PointNet2PartSegMSG"]


def make(name, dev, seed=0):
    torch.manual_seed(seed)
    return getattr(nets, name)().to(dev)


def run(net, x, cls, lengths=None):
    if isinstance(net, nets.PointNet2PartSegMSG):
        return net(x, cls, lengths=lengths)
    return net(x, lengths=lengths)


@pytest.mark.parametrize("amp", [False, True])
@pytest.mark.parametrize("name", NETS)
def test_forward_and_backward(dev, name, amp):
    b = 4
    pts, cls, label = W.part_shapes(b, N, 1, nets.PART_OFFSETS)
    net = make(name, dev).train()
    with torch.autocast("cuda", dtype=torch.bfloat16, enabled=amp):
        pred, end_points = run(net, T(pts, dev), T(cls, dev))
        loss = nets.part_seg_loss(pred, T(label, dev))
    loss.backward()
    assert pred.shape == (b, N, 50) and pred.dtype == (torch.bfloat16 if amp else torch.float32)
    assert end_points["feats"].shape == (b, N, 128) and end_points["l1_xyz"].shape == (b, 512, 3)
    assert torch.isfinite(loss)
    for pname, p in net.named_parameters():
        assert p.grad is not None and bool(torch.isfinite(p.grad).all()), pname


def _padding_child():
    """In a fresh process with deterministic algorithms: for both nets, in train and eval mode, in float32 and under bf16
    autocast, a forward, part_seg_loss and backward with poisoned padding, with copied padding and with poisoned padding
    again.  Prints per case whether the real-row logits, the loss and every gradient agree bit for bit between the
    paddings and between the two poisoned runs, and whether the padding rows of the logits are 0."""
    code = f"""
import sys, numpy as np, torch
sys.path.insert(0, {ROOT!r})
sys.path.insert(0, {os.path.join(ROOT, 'tests')!r})
from pointnet2_b200 import nets, workloads as W
from pointnet2_b200.layers import row_mask
from test_ragged_fp_gpu import pad
torch.use_deterministic_algorithms(True)
dev = torch.device("cuda:0")
lengths, n = {LENGTHS!r}, {N}
pts, cls, label = W.part_shapes(len(lengths), n, 2, nets.PART_OFFSETS)
cls, lens, label = torch.from_numpy(cls).to(dev), torch.tensor(lengths, device=dev), torch.from_numpy(label).to(dev)
mask = row_mask(lens, n)
label[~mask] = 999  # out of range: the loss must not read it
out = []
for name in ("PointNet2PartSeg", "PointNet2PartSegMSG"):
    for mode in ("train", "eval"):
        for amp in (False, True):
            res = []
            for kind in ("poison", "copy", "poison"):
                torch.manual_seed(0)
                net = getattr(nets, name)().to(dev).train(mode == "train")
                x = torch.from_numpy(pad(pts, lengths, kind)).to(dev)
                torch.manual_seed(1)  # the same dropout masks in every run
                with torch.autocast("cuda", dtype=torch.bfloat16, enabled=amp):
                    args = (x, cls) if name == "PointNet2PartSegMSG" else (x,)
                    pred, _ = net(*args, lengths=lens)
                    loss = nets.part_seg_loss(pred, label, lengths=lens)
                loss.backward()
                zero = bool((pred[~mask] == 0).all())
                stats = [b for m in net.modules() if isinstance(m, torch.nn.BatchNorm1d) for b in (m.running_mean, m.running_var)]
                res.append([loss.detach(), pred.detach()[mask]] + [p.grad.clone() for p in net.parameters()] + stats)
            same = all(torch.equal(a, b) for a, b in zip(res[0], res[1]))
            again = all(torch.equal(a, b) for a, b in zip(res[0], res[2]))
            finite = all(bool(torch.isfinite(t).all()) for t in res[0])
            out.append(f"{{name}} {{mode}} amp={{amp}}: same {{same}} again {{again}} finite {{finite}} zero {{zero}}")
print("\\n".join(out))
"""
    env = dict(os.environ, CUBLAS_WORKSPACE_CONFIG=":4096:8")
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, env=env, cwd=ROOT, timeout=900)
    assert r.returncode == 0, r.stderr[-3000:]
    return r.stdout.strip().splitlines()[-8:]


def test_padding_is_inert_and_training_steps_are_deterministic():
    lines = _padding_child()
    assert len(lines) == 8, lines
    for line in lines:
        assert line.endswith("same True again True finite True zero True"), lines


@pytest.mark.parametrize("name", NETS)
def test_lengths_mean_per_shape(dev, name):
    pts, cls, _ = W.part_shapes(len(LENGTHS), N, 3, nets.PART_OFFSETS)
    net = make(name, dev).eval()
    mask = row_mask(torch.tensor(LENGTHS, device=dev), N)

    def logits_and_centroids(x):
        pred, end_points = run(net, x, T(cls, dev), LENGTHS)
        return [pred, end_points["l1_xyz"]]

    with torch.no_grad():
        pred, ep = both_paddings(logits_and_centroids, [pts], LENGTHS, dev)
        assert bool((pred[~mask] == 0).all())
        for i, l in enumerate(LENGTHS):
            alone, ep_alone = run(net, T(pts[i:i + 1, :l], dev), T(cls[i:i + 1], dev))
            # sampling is bit-exact per shape (the ragged FPS contract)
            assert torch.equal(bits(ep[i:i + 1]), bits(ep_alone["l1_xyz"])), f"length {l}"
            # the linear layers run cuBLAS at another row count (B*N rows against l), which may round differently in
            # the last bits, and a dozen layers carry that on: a float32 tolerance a few hundred ulps wide
            torch.testing.assert_close(pred[i:i + 1, :l], alone, rtol=1e-4, atol=1e-4, msg=f"length {l}")


@pytest.mark.parametrize("ragged", [False, True])
@pytest.mark.parametrize("name", NETS)
def test_training_lowers_the_loss(dev, name, ragged):
    b, steps = 8, 30
    pts, cls, label = W.part_shapes(b, N, 4, nets.PART_OFFSETS)
    lengths = None
    if ragged:
        lengths = np.random.RandomState(5).randint(N // 2, N + 1, b)
        for i, l in enumerate(lengths):
            pts[i, l:] = np.nan
        lengths = T(lengths.astype(np.int32), dev)
    x, c, y = T(pts, dev), T(cls, dev), T(label, dev)
    net = make(name, dev).train()
    opt = torch.optim.Adam(net.parameters(), lr=1e-3)
    losses = []
    for _ in range(steps):
        pred, _ = run(net, x, c, lengths)
        loss = nets.part_seg_loss(pred, y, lengths=lengths)
        opt.zero_grad(set_to_none=True)
        loss.backward()
        opt.step()
        losses.append(float(loss.detach()))
    assert all(np.isfinite(losses))
    assert np.mean(losses[-5:]) < 0.8 * np.mean(losses[:5]), losses


def test_evaluation_helpers_stay_on_the_device(dev):
    b, n = 16, N
    pts, cls, label = W.part_shapes(b, n, 6, nets.PART_OFFSETS)
    rs = np.random.RandomState(7)
    logits = T(rs.randn(b, n, 50).astype(np.float32), dev)
    c, y = T(cls, dev), T(label, dev)
    lens = T(rs.randint(1, n + 1, b).astype(np.int32), dev)
    want = nets.part_seg_iou(nets.part_seg_predict(logits.cpu(), cls), torch.from_numpy(label), cls, lengths=lens.cpu())
    nets.part_seg_iou(nets.part_seg_predict(logits, c), y, c, lengths=lens)  # first call: the offsets table is copied
    torch.cuda.synchronize(dev)
    torch.cuda.set_sync_debug_mode("error")
    try:
        got = nets.part_seg_iou(nets.part_seg_predict(logits, c), y, c, lengths=lens)
        loss = nets.part_seg_loss(logits, y, lengths=lens)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    torch.testing.assert_close(got.cpu(), want, rtol=1e-12, atol=1e-12)
    assert torch.isfinite(loss)
