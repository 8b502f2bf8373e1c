"""The five networks against a float64 restatement of the reference models (tests/net_oracle.py).

Each net runs one training step (dropout p = 0) and then an eval-mode forward under torch.no_grad(), which takes the
fused fp_interpolate_concat route and running-statistics batch norm.  The logits, the loss, every parameter gradient,
every batch-norm running statistic after the step and the eval logits are compared with the restatement by the relative
Frobenius error ‖got − ref‖ / ‖ref‖.  A norm-wise error absorbs an isolated max-pool or ReLU decision that flips between
float32 and float64 and still sees structural errors; the mutation test at the end shows that each of four plausible
wiring mistakes fails the comparison.  The parameter gradients are compared per learned stack (each SharedMLP's
weights, biases and batch-norm parameters as one vector): several of them are exactly 0 in exact arithmetic (a bias
feeding a training-mode batch norm, the shift of a batch norm whose output reaches the loss only through another batch
norm), so compared alone they would measure float32 rounding against 0.

Arms: float32; float32 under torch.use_deterministic_algorithms(True) (in a child process); bf16 autocast.  Dense and
ragged batches (poisoned padding, clouds shorter than sa1's npoint); the padding rows of the logits must be exactly 0.
The restatement runs in float64 through plain torch on the GPU (its geometry decisions come from the C oracle).

Bounds: each is at least 10x the largest error observed over the whole matrix on an H100, and at most 1/10 of the
smallest mutation error.  The bf16 arm is the exception: see the note at BOUNDS.
"""
import os
import subprocess
import sys
import tempfile

import numpy as np
import pytest
import torch

import net_oracle as NO
import numerics as NUM
from pointnet2_b200 import layers, nets, pointnet_util, workloads as W
from pointnet2_b200.layers import SharedMLP
from pointnet2_b200.pointnet_util import pointnet_sa_module

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# Relative Frobenius error bounds of the whole nets, per arm and check.  Largest error observed over the matrix on one
# H100 80GB HBM3: f32 fwd 2.5e-5, grad 4.7e-3, stats 6.3e-6.
# bf16: autocast rounds every Linear output to 8 bits, and a batch norm over rows whose mean is large against their
# spread turns that into a large relative error (observed fwd 0.24, stats 0.061; a CPU emulation of the forward rounding
# alone gives logits error 0.21 and per-stack gradient errors near 1).  Compared with float64, a bf16 gradient says
# nothing beyond its magnitude, so the bf16 arm checks each stack's gradient for finite values and a norm within a
# factor 2 of the restatement's (GRAD_NORM_RATIO), and its fwd / stats bounds catch gross failures only.  The 16-bit
# kernels themselves are held to tight bounds by the single-module checks (SA_BOUNDS) and by their own op tests.
# Observed bf16 stack-gradient norm ratios: within [0.83, 1.38].
BOUNDS = {
    "f32": {"fwd": 3e-4, "grad": 5e-2, "stats": 1e-4},
    "bf16": {"fwd": 0.5, "stats": 0.15},
}
GRAD_NORM_RATIO = (0.5, 2.0)

CASES = {
    "cls_ssg": dict(b=4, n=1024, lengths=[1024, 700, 300, 1000], cloud="S"),
    "cls_msg": dict(b=3, n=1024, lengths=[1024, 513, 200], cloud="S"),
    "sem_seg": dict(b=3, n=2048, lengths=[2048, 1500, 700], cloud="D"),  # duplicates: three_nn meets zero distances
    "part_seg": dict(b=4, n=2048, lengths=[2048, 1800, 400, 1300]),
    "part_seg_msg": dict(b=3, n=2048, lengths=[2048, 1000, 300], cls=[0, 15, 7]),
}
LAYOUTS = ("dense", "ragged")


@pytest.fixture(autouse=True)
def no_tf32():
    """float32 GEMMs and convolutions in full float32: TF32 would make the float32 bound meaningless"""
    old = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = old


def make_net(name):
    torch.manual_seed(0)
    net = {"cls_ssg": lambda: nets.PointNet2ClsSSG(40), "cls_msg": lambda: nets.PointNet2ClsMSG(40),
           "sem_seg": lambda: nets.PointNet2SemSeg(21), "part_seg": nets.PointNet2PartSeg,
           "part_seg_msg": nets.PointNet2PartSegMSG}[name]()
    for m in net.modules():
        if isinstance(m, torch.nn.Dropout):
            m.p = 0.0
    return net


def case_inputs(name, layout):
    """points (b, n, c) float32 numpy (real rows; the padding is poisoned for the net), lengths, labels"""
    c = CASES[name]
    b, n = c["b"], c["n"]
    rs = np.random.RandomState(100 + list(CASES).index(name))
    out = dict(lengths=c["lengths"] if layout == "ragged" else None, cls_label=None, smpw=None)
    if name.startswith("part"):
        pts, cls, label = W.part_shapes(b, n, 200 + b, nets.PART_OFFSETS)
        out.update(points=pts, label=label, cls_label=np.asarray(c.get("cls", cls), np.int64))
    else:
        out["points"] = W.DISTRIBUTIONS[c["cloud"]](b, n, 300 + b)
        if name == "sem_seg":
            out["label"] = rs.randint(0, 21, (b, n))
            out["smpw"] = (rs.rand(b, n) * 2 * (rs.rand(b, n) > 0.25)).astype(np.float32)  # some weights 0
        else:
            out["label"] = rs.randint(0, 40, b)
    return out


def _bn_buffers(net):
    return {k: v for k, v in net.state_dict().items() if k.endswith(("running_mean", "running_var", "num_batches_tracked"))}


def port_step(name, layout, amp=False):
    """the net's training step and eval forward, as float64 CPU tensors"""
    dev = torch.device("cuda:0")
    inp = case_inputs(name, layout)
    net = make_net(name).to(dev).train()
    pts, lengths = inp["points"], inp["lengths"]
    x = torch.from_numpy(NUM.pad_rows(pts, lengths, "poison") if lengths else pts).to(dev)
    lens = None if lengths is None else torch.tensor(lengths, device=dev)

    def fwd():
        with torch.autocast("cuda", dtype=torch.bfloat16, enabled=amp):
            if name == "part_seg_msg":
                return net(x, torch.from_numpy(inp["cls_label"]).to(dev), lengths=lens)[0]
            return net(x, lengths=lens)[0]

    pred = fwd().float()
    label = torch.from_numpy(np.asarray(inp["label"])).to(dev)
    if name.startswith("cls"):
        loss = nets.cls_loss(pred, label)
    elif name == "sem_seg":
        loss = nets.sem_seg_loss(pred, label, torch.from_numpy(inp["smpw"]).to(dev), lengths=lens)
    else:
        loss = nets.part_seg_loss(pred, label, lengths=lens)
    loss.backward()
    out = dict(logits=pred.detach().double().cpu(), loss=loss.detach().double().cpu(),
               grads={k: p.grad.detach().double().cpu() for k, p in net.named_parameters()},
               stats={k: v.detach().cpu().clone() for k, v in _bn_buffers(net).items()})
    net.eval()
    with torch.no_grad():
        out["eval_logits"] = fwd().double().cpu()
    return out


_REF = {}


def reference(name, layout):
    """the restatement's training step and eval forward (cached: it does not depend on the arm)"""
    key = (name, layout)
    if key not in _REF:
        inp = case_inputs(name, layout)
        state = make_net(name).state_dict()
        kw = dict(lengths=inp["lengths"], cls_label=inp["cls_label"], device="cuda:0")
        res = NO.run(name, state, inp["points"], label=inp["label"], smpw=inp["smpw"], training=True, **kw)
        ev = NO.run(name, dict(state, **res.stats), inp["points"], training=False, **kw)
        _REF[key] = dict(logits=res.logits.cpu(), loss=res.loss.cpu(), grads={k: g.cpu() for k, g in res.grads.items()},
                         stats={k: v.cpu() for k, v in res.stats.items()}, eval_logits=ev.logits.cpu())
    return _REF[key]


def rel(got, ref):
    got, ref = got.double().reshape(-1), ref.double().reshape(-1)
    den = float(ref.norm())
    return float((got - ref).norm()) / (den if den > 0 else 1.0)


def stack_grads(got, ref):
    """(got, ref) gradient vectors of each learned stack: its weights, biases and batch-norm parameters as one vector"""
    for prefix in sorted({k.rpartition(".body.")[0] for k in got}):
        keys = [k for k in got if k.rpartition(".body.")[0] == prefix]
        yield torch.cat([got[k].reshape(-1) for k in keys]), torch.cat([ref[k].reshape(-1) for k in keys])


def norm_ratios(pairs):
    """(smallest, largest) ‖got‖ / ‖ref‖ over (got, ref) pairs; every got must be finite"""
    ratios = []
    for g, r in pairs:
        assert bool(torch.isfinite(g).all()), "non-finite gradient"
        ratios.append(float(g.double().norm()) / float(r.double().norm()))
    return min(ratios), max(ratios)


def errors(got, ref):
    """check -> worst relative error: fwd (train and eval logits, loss), grad (every learned stack), stats"""
    e = {"fwd": max(rel(got["logits"], ref["logits"]), rel(got["eval_logits"], ref["eval_logits"]),
                    rel(got["loss"], ref["loss"])), "grad": 0.0, "stats": 0.0}
    for g, r in stack_grads(got["grads"], ref["grads"]):
        e["grad"] = max(e["grad"], rel(g, r))
    for k, v in got["stats"].items():
        if k.endswith("num_batches_tracked"):
            assert int(v) == int(ref["stats"][k]), k
        else:
            e["stats"] = max(e["stats"], rel(v, ref["stats"][k]))
    return e


def assert_padding_is_zero(name, layout, got):
    lengths = CASES[name]["lengths"]
    if layout != "ragged" or name.startswith("cls"):
        return
    for key in ("logits", "eval_logits"):
        for i, l in enumerate(lengths):
            pad = got[key][i, l:]
            assert torch.equal(pad, torch.zeros_like(pad)), (key, i)


def check(name, layout, arm, got):
    assert_padding_is_zero(name, layout, got)
    ref = reference(name, layout)
    e = errors(got, ref)
    bound = BOUNDS["bf16" if arm == "bf16" else "f32"]
    if arm == "bf16":
        lo, hi = norm_ratios(stack_grads(got["grads"], ref["grads"]))
        print(f"\n{name} {layout} {arm}: fwd {e['fwd']:.3e} (bound {bound['fwd']:.2g}), stats {e['stats']:.3e} "
              f"(bound {bound['stats']:.2g}), grad norm ratio [{lo:.3f}, {hi:.3f}] (bound {GRAD_NORM_RATIO}; grad error "
              f"{e['grad']:.3e}, not bounded)")
        assert GRAD_NORM_RATIO[0] <= lo and hi <= GRAD_NORM_RATIO[1], (name, layout, lo, hi)
        del e["grad"]
    else:
        print(f"\n{name} {layout} {arm}: " + ", ".join(f"{k} {v:.3e} (bound {bound[k]:.2g})" for k, v in e.items()))
    for k, v in e.items():
        assert v <= bound[k], (name, layout, arm, k, v, bound[k])


@pytest.mark.parametrize("layout", LAYOUTS)
@pytest.mark.parametrize("name", list(CASES))
@pytest.mark.parametrize("arm", ["f32", "bf16"])
def test_net_against_the_float64_restatement(name, layout, arm):
    check(name, layout, arm, port_step(name, layout, amp=arm == "bf16"))


_DET = {}


def _deterministic_results():
    """every case's float32 step in a fresh process under torch.use_deterministic_algorithms(True)"""
    if not _DET:
        with tempfile.TemporaryDirectory() as tmp:
            path = os.path.join(tmp, "det.pt")
            code = f"""
import sys, torch
sys.path[:0] = [{ROOT!r}, {os.path.join(ROOT, 'tests')!r}]
import test_nets_float64_gpu as T
torch.backends.cuda.matmul.allow_tf32 = False
torch.backends.cudnn.allow_tf32 = False
torch.use_deterministic_algorithms(True)
torch.save({{(n, l): T.port_step(n, l) for n in T.CASES for l in T.LAYOUTS}}, {path!r})
"""
            env = dict(os.environ, CUBLAS_WORKSPACE_CONFIG=":4096:8")
            r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, env=env, cwd=ROOT, timeout=900)
            assert r.returncode == 0, r.stderr[-3000:]
            _DET.update(torch.load(path))
    return _DET


@pytest.mark.parametrize("layout", LAYOUTS)
@pytest.mark.parametrize("name", list(CASES))
def test_net_against_the_float64_restatement_deterministic(name, layout):
    check(name, layout, "det", _deterministic_results()[(name, layout)])


# ---------------------------------------------------------------------------------------------- SA-module options
SA_OPTIONS = [
    dict(pooling="max"), dict(pooling="avg", mlp2=[64, 32]), dict(pooling="weighted_avg", mlp2=[64, 32]),
    dict(pooling="max_and_avg", mlp2=[64, 32]), dict(pooling="max", mlp2=[48]), dict(use_xyz=False), dict(knn=True),
    dict(group_all=True), dict(group_all=True, pooling="max_and_avg", mlp2=[32]),
]


# Relative Frobenius error bounds of one pointnet_sa_module call, per dtype: the module's own rounding, far below the
# whole nets' (where float32 max-pool decision flips dominate the gradients).  Largest error observed over SA_OPTIONS
# on one H100 80GB HBM3: f32 fwd 8.6e-7, grad 3.5e-6; bf16 fwd 2.1e-2.  The group_point_grad mutation below gives
# gradient errors of 7.0e-2 (avg) and 9.6e-2 (max), over 1000x the f32 gradient bound.  The bf16 gradients get the
# norm-ratio check of the nets (the batch norms amplify the 8-bit Linear outputs, as above: observed relative error
# up to 0.20, norm ratios within [0.96, 1.04]).
SA_BOUNDS = {"f32": {"fwd": 1e-5, "grad": 4e-5}, "bf16": {"fwd": 0.25}}


def sa_errors(opt, dtype):
    """(forward error, gradient error, gradient norm ratios) of one pointnet_sa_module call: the gradient error is the
    worst over points and the parameters (a Linear's weight and bias as one vector), the norm ratios are (smallest,
    largest) over the same vectors"""
    dev = torch.device("cuda:0")
    c = 6
    b = 8 if opt.get("group_all") else 2  # group_all: mlp2's batch norm sees b rows
    n = 256 if opt.get("group_all") else 1024
    npoint, radius, nsample = 128, 0.2, 32
    xyz = W.cloud_surface(b, n, 501)
    feats = W.features(b, n, c, 502)
    use_xyz = opt.get("use_xyz", True)
    pooling = opt.get("pooling", "max")
    torch.manual_seed(0)
    holder = torch.nn.Module()
    holder.mlp = SharedMLP(c + 3 if use_xyz else c, [32, 64])
    pooled = 128 if pooling == "max_and_avg" else 64
    holder.mlp2 = SharedMLP(pooled, opt["mlp2"]) if opt.get("mlp2") else None
    state = holder.state_dict()
    holder.to(dev).train()
    g = torch.from_numpy(np.random.RandomState(503).standard_normal(
        (b, 1 if opt.get("group_all") else npoint, holder.mlp2.out_channels if holder.mlp2 else pooled)))

    p = torch.from_numpy(feats).to(dev).to(dtype).requires_grad_(True)
    with torch.autocast("cuda", dtype=torch.bfloat16, enabled=dtype == torch.bfloat16):
        _, out, _ = pointnet_sa_module(torch.from_numpy(xyz).to(dev), p, npoint, radius, nsample, holder.mlp, holder.mlp2,
                                       group_all=opt.get("group_all", False), pooling=pooling, knn=opt.get("knn", False),
                                       use_xyz=use_xyz)
    (out.float() * g.float().to(dev)).sum().backward()

    P = NO.Params(state, "cuda:0")
    f64 = torch.from_numpy(NUM.quantize(feats, "bf16" if dtype == torch.bfloat16 else "f32")).to(dev, torch.float64)
    f64.requires_grad_(True)
    _, ref = NO.sa(P, "", xyz, f64, npoint, radius, nsample, [32, 64], True, mlp2=opt.get("mlp2"),
                   group_all=opt.get("group_all", False), pooling=pooling, knn=opt.get("knn", False), use_xyz=use_xyz)
    (ref * g.to(dev)).sum().backward()
    assert set(P.taken) == set(state)

    e_fwd = rel(out.detach().cpu(), ref.detach().cpu())
    pairs = [(p.grad.cpu(), f64.grad.cpu())]
    named = dict(holder.named_parameters())
    for k, leaf in P.leaves.items():
        got, want = named[k].grad, leaf.grad
        if k.endswith(".bias"):
            w = k[:-len("bias")] + "weight"
            got, want = torch.cat([named[w].grad.reshape(-1), got]), torch.cat([P.leaves[w].grad.reshape(-1), want])
        pairs.append((got.cpu(), want.cpu()))
    return e_fwd, max(rel(g, r) for g, r in pairs), norm_ratios(pairs)


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("opt", SA_OPTIONS, ids=lambda o: "-".join(f"{k}={v}" for k, v in o.items()))
def test_sa_module_options_against_the_float64_restatement(opt, dtype):
    e_fwd, e_grad, (lo, hi) = sa_errors(opt, dtype)
    bf16 = dtype == torch.bfloat16
    bound = SA_BOUNDS["bf16" if bf16 else "f32"]
    print(f"\nSA {opt} {dtype}: fwd {e_fwd:.3e} (bound {bound['fwd']:.2g}), grad {e_grad:.3e}, "
          f"grad norm ratio [{lo:.3f}, {hi:.3f}]")
    assert e_fwd <= bound["fwd"], e_fwd
    if bf16:
        assert GRAD_NORM_RATIO[0] <= lo and hi <= GRAD_NORM_RATIO[1], (lo, hi)
    else:
        assert e_grad <= bound["grad"], e_grad


# ---------------------------------------------------------------------------------------------------- mutations
def _flip_xyz_first(monkeypatch):
    orig = pointnet_util.group_and_concat
    monkeypatch.setattr(pointnet_util, "group_and_concat",
                        lambda xyz, new_xyz, points, idx, xyz_first=True: orig(xyz, new_xyz, points, idx, not xyz_first))


def _permute_fp_weights(monkeypatch):
    orig = pointnet_util.three_interpolate
    monkeypatch.setattr(pointnet_util, "three_interpolate",
                        lambda points, idx, weight, lengths=None: orig(points, idx, weight[..., [1, 0, 2]].contiguous(),
                                                                       lengths=lengths))


def _drop_last_slot_grad(monkeypatch):
    orig = pointnet_util.group_point_grad

    def grad(g, idx, shape):
        g = g.clone()
        g[:, :, -1] = 0
        return orig(g, idx, shape)

    monkeypatch.setattr(pointnet_util, "group_point_grad", grad)


MUTATIONS = {
    "bn_eps_1e-5": ("sem_seg", lambda mp: mp.setattr(layers, "BN_EPS", 1e-5)),
    "msg_xyz_first_flipped": ("cls_msg", _flip_xyz_first),
    "fp_weight_columns_permuted": ("sem_seg", _permute_fp_weights),
}


@pytest.mark.parametrize("mutation", list(MUTATIONS))
def test_each_mutation_fails_the_comparison(monkeypatch, mutation):
    name, apply = MUTATIONS[mutation]
    apply(monkeypatch)
    e = errors(port_step(name, "dense"), reference(name, "dense"))
    ratio = {k: v / BOUNDS["f32"][k] for k, v in e.items()}
    print(f"\nmutation {mutation} on {name}: " + ", ".join(f"{k} {v:.3e}" for k, v in e.items()))
    assert max(ratio.values()) > 10, ratio


@pytest.mark.parametrize("pooling", ["avg", "max"])
def test_group_point_grad_mutation_fails_the_sa_comparison(monkeypatch, pooling):
    """In a whole net the last slot's share of the gradient (about 6e-3 of a stack's gradient in the part-seg net) is at
    the level of float32 max-pool decision flips, so this mutation is checked on one SA module, whose own float32
    gradient error is about 1e-6: its error must be at least 10x the module's gradient bound, with the average pooling
    (every slot carries gradient) and with the max pooling the nets use (only the slots that win a channel do)."""
    _drop_last_slot_grad(monkeypatch)
    e_fwd, e_grad, _ = sa_errors(dict(pooling=pooling), torch.float32)
    print(f"\nmutation group_point_grad_last_slot_zeroed on an SA module ({pooling}): fwd {e_fwd:.3e}, grad {e_grad:.3e}")
    assert e_grad >= 10 * SA_BOUNDS["f32"]["grad"], e_grad
