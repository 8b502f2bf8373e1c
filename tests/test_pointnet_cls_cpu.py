"""PointNet v1 (nets.PointNetClsBasic) and its whole-cloud max-pool layers without a device: the port's parameters and
initialisation, the torch composition against the float64 restatement (tests/pointnet_cls_oracle.py), the gradient of
tied maxima, the wrappers' argument errors and the new C entries' refusals."""
import ctypes
import inspect
import math
import os
import re

import numpy as np
import pytest
import torch
from torch import nn

import numerics as NUM
import pointnet_cls_oracle as PO
from pointnet2_b200 import _build, _lib, layers, nets, workloads as W
from pointnet2_b200.layers import SharedMLP, masked_bn_relu_max, sa_mlp_max, shared_mlp_max

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def make_net(num_class=40, dtype=torch.float32):
    torch.manual_seed(0)
    net = nets.PointNetClsBasic(num_class).to(dtype)
    net.dp1.p = 0.0
    return net


def test_parameters_match_the_reference_variables():
    """models/pointnet_cls_basic.py: conv1 [1,3,1,64], conv2-conv5 [1,1,in,out], fc1 [1024,512], fc2 [512,256], fc3
    [256,40], a batch norm after every layer but fc3.  torch's Linear holds (out, in)."""
    net = nets.PointNetClsBasic(40)
    ref = {"feat.body.0": (1 * 3 * 1, 64), "feat.body.3": (64, 64), "feat.body.6": (64, 64), "feat.body.9": (64, 128),
           "conv5.body.0": (128, 1024), "fc1.body.0": (1024, 512), "fc2.body.0": (512, 256), "fc3.body.0": (256, 40)}
    sd = net.state_dict()
    for name, (cin, cout) in ref.items():
        assert tuple(sd[f"{name}.weight"].shape) == (cout, cin), name
        assert tuple(sd[f"{name}.bias"].shape) == (cout,), name
    bns = [m for m in net.modules() if isinstance(m, nn.BatchNorm1d)]
    assert [m.num_features for m in bns] == [64, 64, 64, 128, 1024, 512, 256]
    assert all(m.eps == layers.BN_EPS for m in bns)
    assert not any(isinstance(m, nn.BatchNorm1d) for m in net.fc3.modules())
    assert math.isclose(net.dp1.p, 0.3)
    assert list(inspect.signature(nets.PointNetClsBasic.forward).parameters)[1:] == ["point_cloud", "lengths"]
    assert inspect.signature(nets.PointNetClsBasic.forward).parameters["lengths"].default is None


def test_conv1_init_uses_the_1x3_kernel_fans():
    torch.manual_seed(3)
    w = nets.PointNetClsBasic().feat.body[0].weight.detach()
    bound = math.sqrt(6.0 / (3 + 192))
    assert float(w.abs().max()) <= bound
    assert float(w.abs().max()) > 0.9 * bound  # 192 draws: the largest is near the bound
    w2 = nets.PointNetClsBasic().feat.body[3].weight.detach()  # 1x1 layers keep SharedMLP's xavier on (64, 64)
    assert float(w2.abs().max()) > bound and float(w2.abs().max()) <= math.sqrt(6.0 / 128)


def _case(layout):
    b, n = 3, 96
    pts = W.DISTRIBUTIONS["S"](b, n, 11)
    lengths = [96, 40, 1] if layout == "ragged" else None
    label = np.array([3, 0, 7])
    return pts, lengths, label


def _port_step(layout, dtype):
    pts, lengths, label = _case(layout)
    net = make_net(10, dtype).train()
    x = torch.from_numpy(NUM.pad_rows(pts, lengths, "poison") if lengths else pts).to(dtype)
    logits, _ = net(x, lengths=lengths)
    loss = nets.cls_loss(logits, torch.from_numpy(label))
    loss.backward()
    grads = {k: p.grad.detach().double() for k, p in net.named_parameters()}
    stats = {k: v.detach().clone() for k, v in net.state_dict().items() if "running" in k or "num_batches" in k}
    net.eval()
    with torch.no_grad():
        ev = net(x, lengths=lengths)[0].double()
    return logits.detach().double(), loss.detach().double(), grads, stats, ev


def _reference(layout, dtype):
    pts, lengths, label = _case(layout)
    state = make_net(10, dtype).state_dict()
    res = PO.run(state, pts, lengths=lengths, label=label, training=True)
    ev = PO.run(dict(state, **res.stats), pts, lengths=lengths, training=False)
    assert set(res.taken) == set(state) - {k for k in state if "running" in k or "num_batches" in k} | set(res.stats)
    return res, ev


def _rel(got, ref):
    got, ref = got.double().reshape(-1), ref.double().reshape(-1)
    return float((got - ref).norm()) / max(float(ref.norm()), 1e-300)


@pytest.mark.parametrize("layout", ["dense", "ragged"])
@pytest.mark.parametrize("dtype,bound", [(torch.float64, 1e-10), (torch.float32, 1e-3)])
def test_torch_composition_matches_the_float64_restatement(layout, dtype, bound):
    logits, loss, grads, stats, ev = _port_step(layout, dtype)
    res, ref_ev = _reference(layout, dtype)
    assert torch.isfinite(logits).all() and torch.isfinite(ev).all()
    assert _rel(logits, res.logits) <= bound and _rel(loss, res.loss) <= bound and _rel(ev, ref_ev.logits) <= bound
    for k, g in grads.items():
        # a bias before a training-mode batch norm has gradient 0 in exact arithmetic: compare it absolutely
        scale = max(float(res.grads[k].norm()), float(next(iter(res.grads.values())).norm()) * 1e-3, 1e-12)
        assert float((g - res.grads[k]).norm()) / scale <= 50 * bound, k
    for k, v in stats.items():
        if k.endswith("num_batches_tracked"):
            assert int(v) == int(res.stats[k])
        else:
            # a running mean of zero-bias layers on centred clouds is near 0: measured against a floor of 1e-3
            ref = res.stats[k].double()
            assert float((v.double() - ref).norm()) / max(float(ref.norm()), 1e-3) <= bound, k


def test_tied_rows_send_the_whole_gradient_to_the_first():
    y = torch.tensor([[[1.0, 5.0], [3.0, 5.0], [3.0, 2.0], [float("nan"), 0.0]]]).requires_grad_(True)
    m = layers._first_max(y[:, :3])
    assert m.tolist() == [[3.0, 5.0]]
    m.sum().backward()
    assert y.grad[0].tolist() == [[0.0, 1.0], [1.0, 0.0], [0.0, 0.0], [0.0, 0.0]]
    y.grad = None
    m = layers._first_max(y)
    assert math.isnan(float(m[0, 0])) and float(m[0, 1]) == 5.0
    m.sum().backward()
    assert y.grad[0].tolist() == [[0.0, 1.0], [0.0, 0.0], [0.0, 0.0], [1.0, 0.0]]
    # through the whole step: two identical points give identical rows; in eval mode with grad the max alone routes
    mlp = SharedMLP(3, [16]).eval()
    t = torch.randn(1, 6, 3, dtype=torch.float64)
    t[0, 1] *= 100.0  # the maximum of about half the columns
    t[0, 4] = t[0, 1]
    t.requires_grad_(True)
    shared_mlp_max(mlp.double(), t).sum().backward()
    assert t.grad[0, 4].abs().sum() == 0 and t.grad[0, 1].abs().sum() > 0


def test_shared_mlp_max_ignores_the_padding_rows():
    torch.manual_seed(1)
    mlp = SharedMLP(5, [8, 12]).double().train()
    t = torch.randn(2, 7, 5, dtype=torch.float64)
    a = shared_mlp_max(mlp, t, [7, 3])
    t2 = t.clone()
    t2[1, 3:] = float("nan")
    b = shared_mlp_max(mlp, t2, torch.tensor([7, 3]))
    assert torch.equal(a, b)


def test_wrappers_refuse_cpu_tensors_and_misplaced_lengths():
    bn = nn.BatchNorm1d(8).train()
    with pytest.raises(RuntimeError, match="CUDA"):
        masked_bn_relu_max(bn, torch.zeros(2, 4, 8))
    mlp = SharedMLP(4, [8]).eval()
    with torch.no_grad():
        with pytest.raises(RuntimeError, match="no CPU path"):
            sa_mlp_max(None, None, torch.zeros(2, 5, 4), None, mlp, True, False, lengths=[5, 2])
        with pytest.raises(ValueError, match="lengths only with idx=None"):
            sa_mlp_max(torch.zeros(2, 5, 3), None, None, torch.zeros(2, 1, 5, dtype=torch.int32), SharedMLP(3, [8]).eval(),
                       lengths=[5, 2])
        with pytest.raises(ValueError, match="needs xyz"):
            sa_mlp_max(None, None, torch.zeros(2, 5, 4), None, SharedMLP(7, [8]).eval(), True, True)


def _proto_args(name):
    text = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "pn2_api.h")).read(), flags=re.S)
    proto = re.search(rf"(?:int|size_t)\s+{name}\s*\((.*?)\)\s*;", text, flags=re.S).group(1)
    return [a.strip() for a in proto.split(",")]


@pytest.mark.parametrize("name", ["pn2_sa_mlp_max_all_typed", "pn2_sa_mlp_max_all_workspace_bytes",
                                  "pn2_masked_bn_relu_max_workspace_bytes", "pn2_masked_bn_relu_max_forward_typed",
                                  "pn2_masked_bn_relu_max_backward_typed"])
def test_header_and_ctypes_agree(name):
    assert name in _lib.EXPORTED_SYMBOLS and hasattr(_lib.load(), name)
    args = _proto_args(name)
    _, argtypes = _lib._SIGNATURES[name]
    assert len(args) == len(argtypes)
    scalars = {"int": _lib.c_int, "long long": _lib.c_longlong, "size_t": _lib.c_size_t, "float": _lib.c_float}
    for a, t in zip(args, argtypes):
        want = _lib._P if "*" in a else scalars[a.rsplit(" ", 1)[0]]
        assert t is want, (name, a, t)


def test_workspace_sizes_need_no_device():
    lib = _lib.load()
    assert lib.pn2_sa_mlp_max_all_workspace_bytes(32, 1024) == 32 * 1024 * 4
    assert lib.pn2_sa_mlp_max_all_workspace_bytes(3, 5) == 256
    assert lib.pn2_sa_mlp_max_all_workspace_bytes(0, 5) == 0
    ws = lib.pn2_masked_bn_relu_max_workspace_bytes(32, 1024, 1024)
    assert ws >= lib.pn2_masked_bn_workspace_bytes(32 * 1024, 1024) and ws >= 4 * (3 + 32) * 1024
    assert lib.pn2_masked_bn_relu_max_workspace_bytes(0, 4, 4) == 0


def test_c_entries_refuse_bad_arguments_without_a_launch():
    lib = _lib.load()
    fake = ctypes.c_void_p(256)  # never dereferenced: every call below must fail its checks first
    null = ctypes.c_void_p(0)
    before = _lib.launch_count()

    def sa(b=2, n=8, nl=1, out=fake, ws_bytes=None, widths=(4,), xyz=fake, dtype=0):
        k = max(nl, 1)
        w = (ctypes.c_int * k)(*(list(widths) * k)[:k])
        ptrs = (ctypes.c_void_p * k)(*([256] * k))
        eps = (ctypes.c_float * k)(*([1e-3] * k))
        relu = (ctypes.c_int * k)(*([1] * k))
        need = lib.pn2_sa_mlp_max_all_workspace_bytes(max(b, 1), widths[0])
        return lib.pn2_sa_mlp_max_all_typed(dtype, b, n, 0, xyz, null, null, null, 1, 1, nl, w, ptrs, ptrs, null, null, null,
                                            null, eps, relu, out, widths[0], fake, need if ws_bytes is None else ws_bytes,
                                            null)

    assert sa(out=null) == 1 and sa(xyz=null) == 1          # null pointers
    assert sa(nl=0) == 1 and sa(nl=5) == 1                  # no layer, five layers
    assert sa(b=-1) == 1 and sa(n=-3) == 1 and sa(n=0) == 1  # negative sizes
    assert sa(ws_bytes=16) == 1                              # a short workspace
    assert sa(dtype=7) == 1 and sa(widths=(2048,)) == 1
    assert sa(b=0) == 0                                      # nothing to do: no launch either

    def fwd(b=2, n=8, c=4, x=fake, out=fake, argmax=fake, ws_bytes=None):
        need = lib.pn2_masked_bn_relu_max_workspace_bytes(max(b, 1), max(n, 1), max(c, 1))
        return lib.pn2_masked_bn_relu_max_forward_typed(0, b, n, c, x, fake, null, null, 1e-3, 0.1, null, null, null, out,
                                                        argmax, fake, fake, fake, need if ws_bytes is None else ws_bytes,
                                                        null)

    def bwd(b=2, n=8, c=4, dx=fake, ws_bytes=None):
        need = lib.pn2_masked_bn_relu_max_workspace_bytes(max(b, 1), max(n, 1), max(c, 1))
        return lib.pn2_masked_bn_relu_max_backward_typed(0, b, n, c, fake, fake, fake, fake, fake, null, fake, fake, dx, null,
                                                         null, fake, need if ws_bytes is None else ws_bytes, null)

    assert fwd(x=null) == 1 and fwd(out=null) == 1 and fwd(argmax=null) == 1
    assert fwd(b=-1) == 1 and fwd(n=0) == 1 and fwd(c=0) == 1 and fwd(ws_bytes=8) == 1
    assert fwd(b=1 << 16, n=1 << 16) == 1  # 2^32 rows
    assert bwd(dx=null) == 1 and bwd(b=-2) == 1 and bwd(c=-1) == 1 and bwd(ws_bytes=0) == 1
    assert fwd(b=0) == 0 and bwd(b=0) == 0
    assert _lib.launch_count() == before
    assert "masked_bn.cu" in _build.SOURCES and "sa_mlp.cu" in _build.SOURCES
