"""CPU checks of the float64 restatement of the reference models (tests/net_oracle.py): it reads every state-dict key
of each net exactly once, its Linear + batch norm + ReLU is nets' SharedMLP (in float64 on the CPU, where SharedMLP
runs plain torch), its gradients pass gradcheck, and it never loads the CUDA library."""
import os
import subprocess
import sys
from unittest import mock

import numpy as np
import pytest
import torch

import net_oracle as NO
from pointnet2_b200 import _lib, nets, workloads as W
from pointnet2_b200.layers import SharedMLP, row_mask

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def make_net(name):
    torch.manual_seed(0)
    return {"cls_ssg": lambda: nets.PointNet2ClsSSG(10), "cls_msg": lambda: nets.PointNet2ClsMSG(10),
            "sem_seg": lambda: nets.PointNet2SemSeg(13), "part_seg": nets.PointNet2PartSeg,
            "part_seg_msg": nets.PointNet2PartSegMSG}[name]()


def small_inputs(name, b, n, seed):
    rs = np.random.RandomState(seed)
    if name.startswith("part"):
        pts, cls, label = W.part_shapes(b, n, seed, nets.PART_OFFSETS)
        return dict(points=pts, cls_label=cls, label=label)
    pts = W.cloud_surface(b, n, seed)
    if name == "sem_seg":
        return dict(points=pts, label=rs.randint(0, 13, (b, n)), smpw=rs.rand(b, n) * (rs.rand(b, n) > 0.2))
    return dict(points=pts, label=rs.randint(0, 10, b))


@pytest.mark.parametrize("name", NO.NETS)
@pytest.mark.parametrize("lengths", [None, [96, 33]])
def test_every_state_dict_key_is_read_exactly_once(name, lengths):
    net = make_net(name)
    state = net.state_dict()
    res = NO.run(name, state, lengths=lengths, **small_inputs(name, 2, 96, 1))
    assert len(res.taken) == len(set(res.taken))
    assert set(res.taken) == set(state), (set(state) - set(res.taken), set(res.taken) - set(state))
    params = dict(net.named_parameters())
    assert set(res.grads) == set(params)
    for k, g in res.grads.items():
        assert g.shape == params[k].shape and bool(torch.isfinite(g).all()), k
    bn_buffers = {k for k in state if k.endswith(("running_mean", "running_var", "num_batches_tracked"))}
    assert set(res.stats) == bn_buffers
    assert torch.isfinite(res.loss)
    if lengths is not None and not name.startswith("cls"):
        assert torch.equal(res.logits[1, lengths[1]:], torch.zeros_like(res.logits[1, lengths[1]:]))


def _mlp_case(masked):
    torch.manual_seed(3)
    m = SharedMLP(6, [16, 8]).double().train()
    t = (torch.randn(3, 40, 6, dtype=torch.float64) * 0.02).requires_grad_(True)  # pre-BN variance well below 1e-3
    mask = row_mask(torch.tensor([40, 17, 1]), 40) if masked else None
    state = {k: v.clone() for k, v in m.state_dict().items()}
    out = m(t) if mask is None else m(t, mask)
    g = torch.randn_like(out)
    if mask is not None:
        g = torch.where(mask.unsqueeze(-1), g, 0)
    out.backward(g)
    P = NO.Params(state)
    rows = t.detach().reshape(-1, 6) if mask is None else t.detach()[mask]
    x = rows.clone().requires_grad_(True)
    ref = NO.mlp(P, "", x, [16, 8], training=True)
    got = out.detach().reshape(-1, 8) if mask is None else out.detach()[mask]
    ref.backward(g.reshape(-1, 8) if mask is None else g[mask])
    return m, P, got, ref, t, x, mask


@pytest.mark.parametrize("masked", [False, True])
def test_shared_mlp_equals_linear_bn_relu_with_the_reference_epsilon(masked):
    m, P, got, ref, t, x, mask = _mlp_case(masked)
    torch.testing.assert_close(got, ref.detach(), rtol=1e-10, atol=1e-12)
    tg = t.grad.reshape(-1, 6) if mask is None else t.grad[mask]
    torch.testing.assert_close(tg, x.grad, rtol=1e-10, atol=1e-12)
    if mask is not None:
        assert torch.equal(t.grad[~mask], torch.zeros_like(t.grad[~mask]))
    for k, p in m.named_parameters():
        torch.testing.assert_close(p.grad, P.leaves[k].grad, rtol=1e-10, atol=1e-12, msg=k)
    for k, v in m.state_dict().items():
        if k in P.stats:
            torch.testing.assert_close(v.to(P.stats[k].dtype), P.stats[k], rtol=1e-10, atol=1e-12, msg=k)


def _tiny_state(seed, c_in=3, dtype=torch.float64):
    """parameters of a tiny SA (mlp 4, 5) -> FP (mlp 4) -> head (3 classes, no bn) stack, as float64 leaves"""
    g = torch.Generator().manual_seed(seed)
    state = {}

    def lin(prefix, i, cin, cout):
        state[f"{prefix}.body.{i}.weight"] = torch.randn(cout, cin, generator=g, dtype=dtype) / cin ** 0.5
        state[f"{prefix}.body.{i}.bias"] = torch.randn(cout, generator=g, dtype=dtype) * 0.1

    def bn(prefix, i, c):
        state[f"{prefix}.body.{i}.weight"] = 1 + 0.1 * torch.randn(c, generator=g, dtype=dtype)
        state[f"{prefix}.body.{i}.bias"] = 0.1 * torch.randn(c, generator=g, dtype=dtype)
        state[f"{prefix}.body.{i}.running_mean"] = torch.zeros(c, dtype=dtype)
        state[f"{prefix}.body.{i}.running_var"] = torch.ones(c, dtype=dtype)
        state[f"{prefix}.body.{i}.num_batches_tracked"] = torch.tensor(0)

    lin("sa.mlp", 0, c_in, 4), bn("sa.mlp", 1, 4), lin("sa.mlp", 3, 4, 5), bn("sa.mlp", 4, 5)
    lin("fp.mlp", 0, 5 + 2, 4), bn("fp.mlp", 1, 4)
    lin("head", 0, 4, 3)
    return state


@pytest.mark.parametrize("lengths", [None, [40, 13]])
def test_gradcheck_of_a_tiny_sa_fp_head_composition(lengths):
    b, n = 2, 40
    xyz = W.cloud_uniform(b, n, 5)
    state = _tiny_state(6)
    names = [k for k in state if not k.endswith(("running_mean", "running_var", "num_batches_tracked"))]
    feats = torch.from_numpy(W.features(b, n, 2, 7)).double().requires_grad_(True)
    leaves = [state[k].requires_grad_(True) for k in names]

    def f(feats, *params):
        st = dict(state, **dict(zip(names, params)))
        P = NO.Params(st)
        new_xyz, l1 = NO.sa(P, "sa", xyz, None, 8, 0.5, 4, [4, 5], training=True, lengths=lengths)
        l0 = NO.fp(P, "fp", xyz, new_xyz, feats, l1, [4], training=True, lengths=NO._lengths(lengths, b, n))
        if lengths is None:
            l0 = l0.reshape(-1, 4)
        return NO.mlp(P, "head", l0, [3], training=True, bn=False, last_activation=False)

    assert torch.autograd.gradcheck(f, (feats, *leaves), eps=1e-6, atol=1e-6, rtol=1e-5)


def test_the_restatement_never_loads_the_library():
    net = make_net("sem_seg")
    with mock.patch.object(_lib, "load", side_effect=AssertionError("the library was loaded")):
        res = NO.run("sem_seg", net.state_dict(), lengths=[64, 20], **small_inputs("sem_seg", 2, 64, 9))
    assert torch.isfinite(res.loss)
    # and it imports nothing of the package
    code = ("import sys; sys.path[:0] = [{root!r}, {tests!r}]; import net_oracle; "
            "assert not any(m.startswith('pointnet2_b200') for m in sys.modules), sorted(sys.modules); print('ok')")
    r = subprocess.run([sys.executable, "-c", code.format(root=ROOT, tests=os.path.join(ROOT, "tests"))],
                       capture_output=True, text=True, cwd=ROOT, timeout=300)
    assert r.returncode == 0 and r.stdout.strip() == "ok", r.stderr[-2000:]
