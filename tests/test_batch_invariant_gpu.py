"""Batch-invariant inference on the GPU: layers.fp_mlp / layers.mlp_rows (csrc/fp_mlp.cu) against the torch layers in
float64 for every feature-propagation level and head of the five networks; the FP front end bit for bit against
fp_interpolate_concat; whole networks inside layers.batch_invariant() bit for bit against each cloud alone, a permuted
batch, other predict_scene batch sizes and other classify_votes chunks; the mode's accuracy against the float64
restatement; a CUDA graph with rewritten lengths; NaN and inf; and training steps untouched by the mode."""
import copy
import os
import sys
import warnings

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import net_oracle as NO  # noqa: E402
import numerics as NUM  # noqa: E402
import test_nets_float64_gpu as NF  # noqa: E402
import test_sa_mlp_gpu as SA  # noqa: E402

from pointnet2_b200 import batch_invariant, layers, nets, scene, shapes as SH  # noqa: E402
from pointnet2_b200 import workloads as W  # noqa: E402
from pointnet2_b200.layers import SharedMLP, fp_mlp, mlp_rows  # noqa: E402
from pointnet2_b200.tf_interpolate import fp_interpolate_concat  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
DTYPES = [torch.float32, torch.bfloat16, torch.float16]
DTYPE_IDS = ["f32", "bf16", "f16"]


@pytest.fixture(autouse=True)
def _no_tf32():
    """float32 products stay float32 in the torch layers the kernel is compared with"""
    old = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = old


# (name, n1, n2, c1, c2, widths, bn, last_activation): n2 = 0 marks a head (mlp_rows on (2, n1, c2) rows)
LEVELS = [
    ("sem_seg.fp1", 64, 16, 256, 512, [256, 256], True, True),
    ("sem_seg.fp2", 256, 64, 128, 256, [256, 256], True, True),
    ("sem_seg.fp3", 1024, 256, 64, 256, [256, 128], True, True),
    ("sem_seg.fp4", 2048, 1024, 0, 128, [128, 128, 128], True, True),
    ("sem_seg.fc1", 2048, 0, 0, 128, [128], True, True),
    ("sem_seg.fc2", 2048, 0, 0, 128, [21], False, False),
    ("part_seg.fp1", 128, 1, 256, 1024, [256, 256], True, True),
    ("part_seg.fp2", 512, 128, 128, 256, [256, 128], True, True),
    ("part_seg.fp3", 2048, 512, 6, 128, [128, 128, 128], True, True),
    ("part_seg_msg.fp1", 128, 1, 512, 1024, [256, 256], True, True),
    ("part_seg_msg.fp2", 512, 128, 320, 256, [256, 128], True, True),
    ("part_seg_msg.fp3", 2048, 512, 22, 128, [128, 128], True, True),
    ("cls.fc1", 16, 0, 0, 1024, [512], True, True),
    ("cls.fc2", 16, 0, 0, 512, [256], True, True),
    ("cls.fc3", 16, 0, 0, 256, [40], False, False),
]

# Largest |kernel - float64| over a level's outputs relative to the largest |output|, as test_sa_mlp_gpu.F64_BOUNDS.
# Observed on an H100 80GB HBM3: see DESIGN.md 6.14.
F64_BOUNDS = SA.F64_BOUNDS


def _level_inputs(n1, n2, c1, c2, seed, dtype, b=2):
    xyz1 = torch.from_numpy(W.cloud_uniform(b, n1, seed)).to(DEV)
    xyz2 = torch.from_numpy(W.cloud_uniform(b, max(n2, 1), seed + 1)).to(DEV)
    points2 = torch.from_numpy(W.features(b, max(n2, 1) if n2 else n1, c2, seed + 2)).to(DEV).to(dtype)
    points1 = None if c1 == 0 else torch.from_numpy(W.features(b, n1, c1, seed + 3)).to(DEV).to(dtype)
    return xyz1, xyz2, points1, points2


def _run_level(level, dtype, seed):
    name, n1, n2, c1, c2, widths, bn, last_act = level
    xyz1, xyz2, points1, points2 = _level_inputs(n1, n2, c1, c2, seed, dtype)
    mlp = SA._mlp(c2 + c1, widths, seed + 7, bn=bn, last_activation=last_act)
    with torch.no_grad():
        if n2:
            rows = fp_interpolate_concat(xyz1, xyz2, points1, points2)
            got = fp_mlp(xyz1, xyz2, points1, points2, mlp)
        else:
            rows = points2
            got = mlp_rows(points2, mlp)
    return mlp, rows, got


@pytest.mark.parametrize("level", LEVELS, ids=[l[0] for l in LEVELS])
@pytest.mark.parametrize("dtype", DTYPES, ids=DTYPE_IDS)
def test_kernel_against_float64(level, dtype):
    mlp, rows, got = _run_level(level, dtype, 31 + len(level[0]))
    assert got.dtype == dtype and got.shape == (*rows.shape[:-1], level[5][-1])
    with torch.no_grad():
        want = copy.deepcopy(mlp).double()(rows.double())
    err = SA._scaled_err(got, want)
    print(f"{level[0]} {dtype}: scaled error {err:.3g}")
    assert err <= F64_BOUNDS[dtype], (level[0], err)
    if dtype != torch.float32:
        # no further from float64 than the torch layers under autocast, on the mean error, with 10 % for the scatter
        with torch.no_grad(), torch.autocast("cuda", dtype=dtype):
            auto = mlp(rows)
        mine, theirs = (got.double() - want).abs().mean().item(), (auto.double() - want).abs().mean().item()
        assert mine <= 1.1 * theirs, (level[0], mine, theirs)


def _identity(c):
    m = SharedMLP(c, [c], bn=False, last_activation=False).to(DEV).eval()
    with torch.no_grad():
        m.body[0].weight.copy_(torch.eye(c))
        m.body[0].bias.zero_()
    return m


@pytest.mark.parametrize("ragged", [False, True], ids=["dense", "ragged"])
@pytest.mark.parametrize("dtype", DTYPES, ids=DTYPE_IDS)
def test_front_end_reproduces_fp_interpolate_concat(dtype, ragged):
    xyz1, xyz2, points1, points2 = _level_inputs(700, 150, 40, 72, 5, dtype, b=3)
    lengths = torch.tensor([700, 333, 1], dtype=torch.int32, device=DEV) if ragged else None
    if ragged:  # the padding is never read
        for i, l in enumerate(lengths.tolist()):
            xyz1[i, l:] = float("nan")
            points1[i, l:] = float("nan")
    with torch.no_grad():
        want = fp_interpolate_concat(xyz1, xyz2, points1, points2, lengths=lengths)
        got = fp_mlp(xyz1, xyz2, points1, points2, _identity(112), lengths=lengths)
        # and without points1
        want1 = fp_interpolate_concat(xyz1, xyz2, None, points2, lengths=lengths)
        got1 = fp_mlp(xyz1, xyz2, None, points2, _identity(72), lengths=lengths)
    assert torch.equal(got.view(torch.uint8), want.view(torch.uint8))
    assert torch.equal(got1.view(torch.uint8), want1.view(torch.uint8))


# ---- whole networks --------------------------------------------------------------------------------------------------
NETS = list(NF.CASES)


def _seeded_net(name):
    """the net after two training-mode forwards, so that the running statistics are not the identity"""
    net = NF.make_net(name).to(DEV).train()
    inp = NF.case_inputs(name, "dense")
    x = torch.from_numpy(inp["points"]).to(DEV)
    with torch.no_grad():
        for _ in range(2):
            _call(net, name, x, None, inp)
    return net.eval(), inp


def _call(net, name, x, lengths, inp, rows=None):
    if name == "part_seg_msg":
        cls = torch.from_numpy(inp["cls_label"]).to(DEV)
        return net(x, cls if rows is None else cls[rows], lengths=lengths)[0]
    return net(x, lengths=lengths)[0]


def _eval(net, name, x, lengths, inp, amp, rows=None):
    with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16, enabled=amp), batch_invariant():
        return _call(net, name, x, lengths, inp, rows)


def _bits(t):
    return t.contiguous().view(torch.int16 if t.element_size() == 2 else torch.int32)


@pytest.mark.parametrize("layout", NF.LAYOUTS)
@pytest.mark.parametrize("amp", [False, True], ids=["f32", "bf16"])
@pytest.mark.parametrize("name", NETS)
def test_net_is_batch_invariant(name, amp, layout):
    net, inp = _seeded_net(name)
    b, n = NF.CASES[name]["b"], NF.CASES[name]["n"]
    lengths = NF.CASES[name]["lengths"] if layout == "ragged" else [n] * b
    pts = inp["points"]
    x = torch.from_numpy(NUM.pad_rows(pts, lengths, "poison") if layout == "ragged" else pts).to(DEV)
    lens = torch.tensor(lengths, device=DEV) if layout == "ragged" else None
    seg = not name.startswith("cls")
    got = _eval(net, name, x, lens, inp, amp)
    # each cloud alone, truncated to its length
    for i, l in enumerate(lengths):
        alone = _eval(net, name, x[i:i + 1, :l].contiguous(), None, inp, amp, rows=slice(i, i + 1))
        want = got[i, :l] if seg else got[i]
        assert torch.equal(_bits(alone[0]), _bits(want)), (name, i)
        if seg and l < n:
            assert torch.equal(got[i, l:], torch.zeros_like(got[i, l:])), (name, i)
    # a permuted batch
    perm = torch.tensor(list(range(b))[::-1][1:] + [b - 1], device=DEV)
    pl = None if lens is None else lens[perm]
    got_p = _eval(net, name, x[perm].contiguous(), pl, inp, amp, rows=perm.cpu())
    assert torch.equal(_bits(got_p), _bits(got[perm]))


@pytest.mark.parametrize("layout", NF.LAYOUTS)
@pytest.mark.parametrize("amp", [False, True], ids=["f32", "bf16"])
@pytest.mark.parametrize("name", NETS)
def test_mode_against_the_float64_restatement(name, amp, layout):
    net, _ = _seeded_net(name)
    inp = NF.case_inputs(name, layout)
    pts, lengths = inp["points"], inp["lengths"]
    x = torch.from_numpy(NUM.pad_rows(pts, lengths, "poison") if lengths else pts).to(DEV)
    lens = None if lengths is None else torch.tensor(lengths, device=DEV)
    got = _eval(net, name, x, lens, inp, amp).double().cpu()
    ref = NO.run(name, net.state_dict(), pts, training=False, lengths=lengths, cls_label=inp["cls_label"],
                 device="cuda:0").logits.cpu()
    if lengths and not name.startswith("cls"):
        for i, l in enumerate(lengths):
            assert torch.equal(got[i, l:], torch.zeros_like(got[i, l:]))
    err = NF.rel(got, ref)
    bound = NF.BOUNDS["bf16" if amp else "f32"]["fwd"]
    print(f"\n{name} {layout} {'bf16' if amp else 'f32'}: eval logits {err:.3e} (bound {bound:.2g})")
    assert err <= bound, (name, layout, amp, err)


def test_predict_scene_does_not_depend_on_batch_size():
    net, _ = _seeded_net("sem_seg")
    xyz = torch.from_numpy(W.scene_room(40000, 9)[0]).to(DEV)
    outs = []
    for bs in (16, 5, 1):
        with batch_invariant():
            accum, count, label = scene.predict_scene(net, xyz, batch_size=bs, max_points=2048)
        outs.append((accum, count, label))
    for accum, count, label in outs[1:]:
        assert torch.equal(_bits(accum), _bits(outs[0][0])) and torch.equal(label, outs[0][2])
        assert torch.equal(count, outs[0][1])


def test_classify_votes_does_not_depend_on_chunk():
    torch.manual_seed(0)
    rs = np.random.RandomState(3)
    sizes = [1024, 3000, 2048, 1500, 800]
    ss = SH.ShapeSet([rs.standard_normal((s, 3)).astype(np.float32) for s in sizes], rs.randint(0, 10, len(sizes)),
                     num_class=10, normalize=False, device=DEV)
    idx = torch.tensor([0, 1, 2, 3, 4, 1], device=DEV)
    net, _ = _seeded_net("cls_ssg")
    with batch_invariant():
        a = SH.classify_votes(net, ss, idx, 4, 7, chunk=1)
        b = SH.classify_votes(net, ss, idx, 4, 7, chunk=4)
    assert torch.equal(_bits(a), _bits(b))


def test_cuda_graph_follows_rewritten_lengths():
    net, inp = _seeded_net("sem_seg")
    b, n = 3, 2048
    x = torch.from_numpy(NUM.pad_rows(inp["points"], [2048, 1500, 700], "poison")).to(DEV)
    lens = torch.tensor([2048, 1500, 700], dtype=torch.int32, device=DEV)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s), torch.no_grad(), batch_invariant():
        for _ in range(2):
            net(x, lens)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.no_grad(), batch_invariant(), torch.cuda.graph(g):
        out = net(x, lens)[0]
    for new in ([2048, 1500, 700], [900, 2048, 64], [1, 1024, 2000]):
        lens.copy_(torch.tensor(new, dtype=torch.int32))
        g.replay()
        with torch.no_grad(), batch_invariant():
            want = net(x, lens)[0]
        assert torch.equal(_bits(out), _bits(want)), new


def test_nan_and_inf_propagate_as_in_torch():
    mlp = SA._mlp(64, [64, 32], 3)
    t = torch.from_numpy(W.features(1, 256, 64, 4)).to(DEV)[0]
    t[3, 5] = float("nan")
    t[7, 0] = float("inf")
    t[9, 63] = float("-inf")
    t[11, :] = float("inf")
    with torch.no_grad():
        got = mlp_rows(t, mlp)
        want = mlp(t)
    assert torch.equal(torch.isnan(got), torch.isnan(want))
    assert torch.equal(torch.isinf(got), torch.isinf(want))
    assert torch.equal(got[torch.isinf(got)], want[torch.isinf(want)])
    fin = torch.isfinite(want)
    torch.testing.assert_close(got[fin], want[fin], rtol=1e-5, atol=1e-5)
    # the FP front end: a NaN feature of a known point reaches the rows that interpolate it
    xyz1, xyz2, points1, points2 = _level_inputs(300, 40, 8, 56, 9, torch.float32)
    points2[0, 7, 2] = float("nan")
    points2[1, 3, :] = float("inf")
    fmlp = SA._mlp(64, [64, 32], 4)
    with torch.no_grad():
        got = fp_mlp(xyz1, xyz2, points1, points2, fmlp)
        want = fmlp(fp_interpolate_concat(xyz1, xyz2, points1, points2))
    assert bool(torch.isnan(got).any())
    assert torch.equal(torch.isnan(got), torch.isnan(want))
    assert torch.equal(torch.isinf(got), torch.isinf(want))


def _train_step(name, layout, mode):
    inp = NF.case_inputs(name, layout)
    net = NF.make_net(name).to(DEV).train()
    pts, lengths = inp["points"], inp["lengths"]
    x = torch.from_numpy(NUM.pad_rows(pts, lengths, "poison") if lengths else pts).to(DEV)
    lens = None if lengths is None else torch.tensor(lengths, device=DEV)
    with batch_invariant(mode):
        pred = _call(net, name, x, lens, inp)
        label = torch.from_numpy(np.asarray(inp["label"])).to(DEV)
        if name.startswith("cls"):
            loss = nets.cls_loss(pred, label)
        else:
            loss = nets.sem_seg_loss(pred, label, torch.from_numpy(inp["smpw"]).to(DEV), lengths=lens)
        loss.backward()
    return loss.detach(), {k: p.grad.clone() for k, p in net.named_parameters()}, \
        {k: v.clone() for k, v in net.state_dict().items()}


@pytest.mark.parametrize("name,layout", [("sem_seg", "ragged"), ("cls_ssg", "dense")])
def test_training_is_unchanged(name, layout, monkeypatch):
    # the library's deterministic gradient kernels, so that two steps can be compared bit for bit
    det, warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(True, warn_only=True)
    try:
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            off = _train_step(name, layout, False)

            def refuse(*a, **k):
                raise AssertionError("a training step entered a batch-invariant kernel")

            for fn in ("fp_mlp", "mlp_rows"):
                monkeypatch.setattr(layers, fn, refuse)
            on = _train_step(name, layout, True)
    finally:
        torch.use_deterministic_algorithms(det, warn_only=warn)
    assert torch.equal(off[0], on[0])
    for part in (1, 2):
        assert off[part].keys() == on[part].keys()
        for k in off[part]:
            assert torch.equal(off[part][k], on[part][k]), k


def test_mode_raises_for_layers_the_kernels_cannot_take():
    x = torch.randn(5, 6, device=DEV)
    with torch.no_grad(), batch_invariant():
        for mlp in (SharedMLP(6, [8] * 5), SharedMLP(6, [2048]), SharedMLP(6, [8]).to(torch.bfloat16)):
            with pytest.raises(RuntimeError, match="batch_invariant"):
                mlp.to(DEV).eval()(x.to(mlp.body[0].weight.dtype))
        with pytest.raises(RuntimeError, match="batch_invariant"):
            SharedMLP(6, [8]).to(DEV).eval()(x.double())
        # a training-mode stack keeps the torch layers
        SharedMLP(6, [8]).to(DEV).train()(x)
