"""The pn2:: torch operators on the GPU: torch.library.opcheck of every operator, one graph and no graph break for each
network's training step and eval forwards, compiled results equal to eager ones (bit for bit where the library's
kernels compute everything, within the float64 checks' tolerances where torch's own layers are compiled), CUDA-graph
replay on new clouds and new lengths, and the deterministic and batch-invariant modes honoured between calls."""
import copy

import pytest
import torch
import torch._dynamo

from pointnet2_b200 import layers, nets, workloads as W
from pointnet2_b200.pointnet_util import fp_interpolate_concat, group_and_concat, sample_and_group

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
UTILS = ("test_schema", "test_autograd_registration", "test_faketensor", "test_aot_dispatch_dynamic")
F32_BOUNDS = {"fwd": 3e-4, "grad": 5e-2, "stats": 1e-4}  # the float32 bounds of test_nets_float64_gpu


def _cloud(b, n, seed, ch=3):
    x = torch.from_numpy(W.cloud_uniform(b, n, seed)).to(DEV)
    if ch == 6:
        x = torch.cat([x, torch.nn.functional.normalize(torch.randn(b, n, 3, device=DEV, generator=torch.Generator(DEV).manual_seed(seed)), dim=-1)], -1)
    return x.contiguous()


def _feat(b, n, c, dtype=torch.float32, seed=0, grad=False):
    g = torch.Generator(DEV).manual_seed(seed)
    return torch.randn(b, n, c, device=DEV, generator=g).to(dtype).requires_grad_(grad)


# ------------------------------------------------------------------------------------------------------------ opcheck
def _op_samples(b, dtype, lens):
    n, m, s, c = 256, 32, 8, 5
    xyz, q = _cloud(b, n, 1), _cloud(b, m, 2)
    pts = _feat(b, n, c, dtype, 3, grad=True)
    pts2 = _feat(b, m, c, dtype, 4, grad=True)
    lq = None if lens is None else lens.clamp(max=m)
    idx = torch.randint(0, n, (b, m, s), dtype=torch.int32, device=DEV)
    nn_idx = torch.randint(0, m, (b, n, 3), dtype=torch.int32, device=DEV)
    w = torch.rand(b, n, 3, device=DEV)
    mlp = layers.SharedMLP(c + 3, [16, 24]).to(DEV).eval()
    params, eps, relu = layers._stack_params(layers._mlp_stack(mlp))
    params = [None if t is None else t.detach() for t in params]  # the fused MLPs have no backward
    bn = torch.nn.BatchNorm1d(c, eps=1e-3).to(DEV)
    keep = torch.rand(b * n, device=DEV) < 0.8
    o = torch.ops.pn2
    return [
        (o.farthest_point_sample, (m, xyz, lens)),
        (o.farthest_point_sample_and_gather, (m, xyz, lens)),
        (o.prob_sample, (torch.rand(b, n, device=DEV), torch.rand(b, m, device=DEV))),
        (o.gather_point, (xyz.clone().requires_grad_(True), idx[:, :, 0].contiguous())),
        (o.gather_point_grad, (torch.randn(b, m, 3, device=DEV), idx[:, :, 0].contiguous(), n)),
        (o.query_ball_point, (0.3, s, xyz, q, lens)),
        (o.select_top_k, (4, torch.rand(b, m, 40, device=DEV))),
        (o.group_point, (pts, idx)),
        (o.group_point_grad, (torch.randn(b, m, s, c, device=DEV).to(dtype), idx, n)),
        (o.knn_point, (s, xyz, q, lens, lq)),
        (o.three_nn, (xyz, q, lens)),
        (o.three_interpolate, (pts2, nn_idx, w, lens)),
        (o.three_interpolate_grad, (torch.randn(b, n, c, device=DEV).to(dtype), nn_idx, w, lens, m)),
        (o.three_nn_interpolate, (xyz, q, pts2.detach(), lens, True)),
        (o.fp_interpolate_concat, (xyz, q, pts.detach(), pts2.detach(), lens)),
        (o.sample_group, (m, 0.3, s, xyz, True, True, lens)),
        (o.sample_group_msg, (m, [0.2, 0.4], [s, 2 * s], xyz, True, True, lens)),
        (o.sample_knn, (m, s, xyz, True, True, True, lens)),
        (o.ball_group, (0.3, s, xyz, q, True, True)),
        (o.group_and_concat, (xyz, q, pts, idx, True)),
        (o.group_and_concat_backward, (torch.randn(b, m, s, 3 + c, device=DEV).to(dtype), torch.randn(b, m, s, 3, device=DEV),
                                       idx, n, False, True, True, True)),
        (o.masked_batch_norm_relu, (_feat(b * n, 1, c, dtype, 5, grad=True).view(b * n, c), bn.weight, bn.bias,
                                    keep.view(torch.uint8), bn.running_mean, bn.running_var, bn.num_batches_tracked, 1e-3, 0.1)),
        (o.masked_bn_relu_max, (_feat(b, n, c, dtype, 6, grad=True), bn.weight, bn.bias, keep.view(torch.uint8),
                                bn.running_mean, bn.running_var, bn.num_batches_tracked, 1e-3, 0.1)),
        (o.sa_mlp_max, (xyz, q, pts.detach(), idx, None, params, eps, relu, True, True, dtype)),
        (o.sa_mlp_max, (xyz, None, pts.detach(), None, lens, params, eps, relu, True, True, dtype)),
        (o.fp_mlp, (xyz, q, _feat(b, n, 3, dtype), pts2.detach(), lens, params, eps, relu, dtype)),
        (o.mlp_rows, (_feat(b, n, c + 3, dtype), keep[: b * n].view(b, n), params, eps, relu, dtype)),
    ]


@pytest.mark.parametrize("case", ["dense_f32", "ragged_bf16", "ragged_f16_det", "empty_batch"])
def test_opcheck(case):
    b = 0 if case == "empty_batch" else 3
    dtype = {"dense_f32": torch.float32, "ragged_bf16": torch.bfloat16, "ragged_f16_det": torch.float16,
             "empty_batch": torch.float32}[case]
    lens = torch.tensor([256, 100, 7], dtype=torch.int32, device=DEV)[:b] if "ragged" in case else None
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms("det" in case, warn_only=True)
    try:
        with torch.no_grad():
            samples = _op_samples(b, dtype, lens)
        for op, args in samples:
            if b == 0 and op in (torch.ops.pn2.masked_batch_norm_relu, torch.ops.pn2.masked_bn_relu_max):
                continue  # the wrappers never send an empty batch to the batch-norm kernels
            torch.library.opcheck(op, args, test_utils=UTILS)
    finally:
        torch.use_deterministic_algorithms(prev)


def test_registered_backward_ops_follow_the_deterministic_flag():
    b, n, m, s, c = 2, 300, 40, 16, 7
    idx = torch.randint(0, n, (b, m, s), dtype=torch.int32, device=DEV)
    g = torch.randn(b, m, s, c, device=DEV)
    prev = torch.are_deterministic_algorithms_enabled()
    try:
        torch.use_deterministic_algorithms(True, warn_only=True)
        det = [torch.ops.pn2.group_point_grad(g, idx, n) for _ in range(2)]
        torch.use_deterministic_algorithms(False)
        atom = torch.ops.pn2.group_point_grad(g, idx, n)
    finally:
        torch.use_deterministic_algorithms(prev)
    assert torch.equal(det[0], det[1])
    torch.testing.assert_close(atom, det[0], rtol=1e-5, atol=1e-5)


# ------------------------------------------------------------------------------------------------- the six networks
NETS = {
    "sem_seg": (nets.PointNet2SemSeg, 3, 8, 2048),
    "cls_ssg": (nets.PointNet2ClsSSG, 3, 8, 1024),
    "cls_msg": (nets.PointNet2ClsMSG, 3, 4, 1024),
    "part_seg": (nets.PointNet2PartSeg, 6, 4, 2048),
    "part_seg_msg": (nets.PointNet2PartSegMSG, 6, 4, 2048),
    "cls_basic": (nets.PointNetClsBasic, 3, 8, 1024),
}


def _net_inputs(name, ragged, seed=7):
    cls, ch, b, n = NETS[name]
    x = _cloud(b, n, seed, ch)
    lens = torch.randint(n // 3, n + 1, (b,), device=DEV, generator=torch.Generator(DEV).manual_seed(seed)).to(torch.int32) \
        if ragged else None
    extra = (torch.arange(b, device=DEV) % nets.NUM_CATEGORIES,) if name == "part_seg_msg" else ()
    return x, extra, lens


def _make(name, seed=0):
    torch.manual_seed(seed)
    net = NETS[name][0]().to(DEV)
    for m in net.modules():
        if isinstance(m, torch.nn.Dropout):
            m.p = 0.0  # compiled and eager steps draw the same (no) masks
    return net


def _loss(name, pred, lens):
    b = pred.shape[0]
    if name.startswith("cls"):
        return nets.cls_loss(pred, torch.arange(b, device=DEV) % pred.shape[-1])
    label = (torch.arange(pred.shape[1], device=DEV) % pred.shape[-1]).expand(b, -1)
    if name == "sem_seg":
        return nets.sem_seg_loss(pred, label, torch.ones(label.shape, device=DEV), lengths=lens)
    return nets.part_seg_loss(pred, label, lengths=lens)


def _train_step(name):
    def step(net, x, extra, lens):
        pred = net(x, *extra, lengths=lens)[0]
        return pred, _loss(name, pred, lens)
    return step


def _eval_fwd(net, x, extra, lens):
    with torch.no_grad():
        return net(x, *extra, lengths=lens)[0]


def _eval_inv(net, x, extra, lens):
    with torch.no_grad(), layers.batch_invariant():
        return net(x, *extra, lengths=lens)[0]


def _one_graph(fn, *args):
    torch._dynamo.reset()
    ex = torch._dynamo.explain(fn)(*args)
    assert ex.graph_count == 1 and ex.graph_break_count == 0, ex.break_reasons


@pytest.mark.parametrize("ragged", [False, True], ids=["dense", "ragged"])
@pytest.mark.parametrize("name", list(NETS))
def test_one_graph(name, ragged):
    net = _make(name)
    x, extra, lens = _net_inputs(name, ragged)
    _one_graph(_train_step(name), net.train(), x, extra, lens)
    net.eval()
    _one_graph(_eval_fwd, net, x, extra, lens)
    _one_graph(_eval_inv, net, x, extra, lens)


def test_reference_call_sites_one_graph_after_an_eager_call():
    import test_reference_callers_gpu as R
    layers.reset_scopes()
    x = _cloud(2, 8192, 7)
    R.sem_seg_trunk(x, is_training=True, bn_decay=0.5)  # creates the scoped layers
    _one_graph(lambda x: R.sem_seg_trunk(x, is_training=True, bn_decay=0.5)[0].sum(), x)
    with torch.no_grad():
        _one_graph(lambda x: R.sem_seg_trunk(x, is_training=False)[0], x)
    layers.reset_scopes()


# ------------------------------------------------------------------------------------------------------ bit identity
def _library_step(xyz, feats, lens):
    new_xyz, new_points, idx, _ = sample_and_group(256, 0.2, 16, xyz, feats, lengths=lens)
    up = fp_interpolate_concat(xyz, new_xyz, feats.detach(), new_points.max(dim=2).values.detach(), lengths=lens)
    g, gx = group_and_concat(xyz, new_xyz, feats, idx, xyz_first=False)
    loss = (new_points * new_points).sum() + (g * g).sum() + (gx * gx).sum()
    return new_xyz, new_points, idx, up, loss


@pytest.mark.parametrize("det", [False, True], ids=["atomic", "deterministic"])
@pytest.mark.parametrize("ragged", [False, True], ids=["dense", "ragged"])
def test_library_step_bit_identical_under_aot_eager(ragged, det):
    b, n = 4, 2048
    xyz = _cloud(b, n, 11)
    lens = torch.tensor([2048, 1500, 700, 64], dtype=torch.int32, device=DEV) if ragged else None
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(det, warn_only=True)
    try:
        torch._dynamo.reset()
        compiled = torch.compile(_library_step, backend="aot_eager", fullgraph=True)
        res = []
        for fn in (_library_step, compiled):
            feats = _feat(b, n, 32, seed=12, grad=True)
            out = fn(xyz, feats, lens)
            out[-1].backward()
            res.append((*out, feats.grad))
    finally:
        torch.use_deterministic_algorithms(prev)
    for e, c in zip(*res):
        if det or e.dtype != torch.float32 or e.dim() != 3 or e.shape[-1] != 32:
            assert torch.equal(e, c)
        else:  # the atomic scatter's order is the GPU's, in eager and compiled runs alike
            torch.testing.assert_close(c, e, rtol=1e-5, atol=1e-5)


@pytest.mark.parametrize("ragged", [False, True], ids=["dense", "ragged"])
@pytest.mark.parametrize("name", list(NETS))
def test_batch_invariant_eval_bit_identical(name, ragged):
    net = _make(name).eval()
    x, extra, lens = _net_inputs(name, ragged)
    want = _eval_inv(net, x, extra, lens)
    torch._dynamo.reset()
    got = torch.compile(_eval_inv, fullgraph=True)(net, x, extra, lens)
    assert torch.equal(got, want)


def _rel(got, ref):
    den = float(ref.double().norm())
    return float((got.double() - ref.double()).norm()) / (den if den > 0 else 1.0)


def _check_stack_grads(got, ref):
    """each learned stack's gradient (its weights, biases and batch-norm parameters as one vector, as
    test_nets_float64_gpu compares them: a bias before a batch norm has a gradient of rounding noise alone)"""
    for prefix in sorted({k.rpartition(".body.")[0] for k in ref}):
        keys = [k for k in ref if k.rpartition(".body.")[0] == prefix]
        g = torch.cat([got[k].reshape(-1) for k in keys])
        r = torch.cat([ref[k].reshape(-1) for k in keys])
        assert _rel(g, r) <= F32_BOUNDS["grad"], prefix


def _geometry_probe(net):
    """the (new_xyz, idx) of the first set-abstraction level, recorded on every call"""
    seen = []
    sa1 = getattr(net, "sa1", None)
    if sa1 is None:
        return seen
    sa1.register_forward_hook(lambda m, a, out: seen.append([t.detach().clone() for t in out if t.dtype != torch.float32 or t.shape[-1] == 3][:2]))
    return seen


@pytest.mark.parametrize("backend", ["aot_eager", "inductor"])
@pytest.mark.parametrize("ragged", [False, True], ids=["dense", "ragged"])
@pytest.mark.parametrize("name", list(NETS))
def test_training_step_matches_eager(name, ragged, backend):
    if backend == "inductor" and name not in ("sem_seg", "cls_basic"):
        pytest.skip("inductor is checked on one PointNet++ net and on PointNet: the other nets share their layers")
    x, extra, lens = _net_inputs(name, ragged)
    results = []
    for compiled in (False, True):
        net = _make(name).train()
        probe = _geometry_probe(net)
        step = _train_step(name)
        if compiled:
            torch._dynamo.reset()
            step = torch.compile(step, backend=backend, fullgraph=True)
        pred, loss = step(net, x, extra, lens)
        loss.backward()
        stats = {k: v.detach().clone() for k, v in net.named_buffers()}
        grads = {k: p.grad.detach().clone() for k, p in net.named_parameters()}
        results.append((pred.detach(), loss.detach(), grads, stats, probe))
    (pe, le, ge, se, geo_e), (pc, lc, gc, sc, geo_c) = results
    for a, b in zip(geo_e, geo_c):
        for u, v in zip(a, b):
            assert torch.equal(u, v)
    assert _rel(pc, pe) <= F32_BOUNDS["fwd"] and _rel(lc, le) <= F32_BOUNDS["fwd"]
    _check_stack_grads(gc, ge)
    for k in se:
        if k.endswith("num_batches_tracked"):
            assert int(sc[k]) == int(se[k]) == 1, k
        else:
            assert _rel(sc[k], se[k]) <= F32_BOUNDS["stats"], k


# ---------------------------------------------------------------------------------------------------- CUDA graphs
def test_cudagraph_replay_on_new_clouds_and_lengths():
    name = "sem_seg"
    b, n = 4, 2048
    x = torch.empty(b, n, 3, device=DEV)
    lens = torch.empty(b, dtype=torch.int32, device=DEV)
    net_c = _make(name).train()
    net_e = copy.deepcopy(net_c)
    probe_c, probe_e = _geometry_probe(net_c), _geometry_probe(net_e)

    def step(net, x, lens):
        pred = net(x, lengths=lens)[0]
        return pred, _loss(name, pred, lens)

    torch._dynamo.reset()
    compiled = torch.compile(step, backend="cudagraphs", fullgraph=True)
    for it in range(5):
        x.copy_(_cloud(b, n, 100 + it))
        lens.copy_(torch.randint(n // 4, n + 1, (b,), device=DEV, generator=torch.Generator(DEV).manual_seed(it)))
        torch.compiler.cudagraph_mark_step_begin()
        if it >= 3:
            torch.cuda.set_sync_debug_mode("error")
        try:
            pred_c, loss_c = compiled(net_c, x, lens)
            loss_c.backward()
        finally:
            torch.cuda.set_sync_debug_mode(0)
        geo_c = [t.clone() for t in probe_c[-1]]  # the replay's outputs live in the graph's pool until the next one
        probe_c.clear()
        pred_e, loss_e = step(net_e, x.clone(), lens.clone())
        loss_e.backward()
        for u, v in zip(geo_c, probe_e[-1]):
            assert torch.equal(u, v), it
        assert _rel(pred_c.detach(), pred_e.detach()) <= F32_BOUNDS["fwd"], it
        _check_stack_grads({k: p.grad for k, p in net_c.named_parameters()},
                           {k: p.grad for k, p in net_e.named_parameters()})
        for p, q in zip(net_c.parameters(), net_e.parameters()):
            p.grad = q.grad = None


# ------------------------------------------------------------------------------------------------------ state toggles
def test_deterministic_toggle_between_calls_of_one_compiled_step():
    xyz = _cloud(4, 2048, 21)
    torch._dynamo.reset()
    compiled = torch.compile(_library_step, backend="aot_eager", fullgraph=True)
    prev = torch.are_deterministic_algorithms_enabled()
    try:
        for det in (True, False, True):
            torch.use_deterministic_algorithms(det, warn_only=True)
            grads = []
            for fn in (_library_step, compiled):
                feats = _feat(4, 2048, 32, seed=22, grad=True)
                fn(xyz, feats, None)[-1].backward()
                grads.append(feats.grad)
            if det:
                assert torch.equal(grads[0], grads[1])
            else:
                torch.testing.assert_close(grads[1], grads[0], rtol=1e-5, atol=1e-5)
    finally:
        torch.use_deterministic_algorithms(prev)


def test_batch_invariant_toggle_between_calls_of_one_compiled_forward():
    net = _make("sem_seg").eval()
    x, extra, lens = _net_inputs("sem_seg", True)
    torch._dynamo.reset()
    compiled = torch.compile(_eval_fwd, backend="aot_eager", fullgraph=True)
    for inv in (False, True, False, True):
        with layers.batch_invariant(inv):
            want = _eval_fwd(net, x, extra, lens)
            got = compiled(net, x, extra, lens)
        assert torch.equal(got, want), inv
    with layers.batch_invariant():
        a = _eval_fwd(net, x, extra, lens)
    assert not torch.equal(a, _eval_fwd(net, x, extra, lens))  # the two modes do take different routes
