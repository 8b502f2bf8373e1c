"""The pn2:: torch operators without a GPU: registration loads nothing, every fake implementation gives the shapes the
wrappers promise, the six networks export (non-strict torch.export on fake CUDA tensors) to graphs of pn2 operators
with no library load, and argument errors raise the same exception types under export as in eager calls."""
import os
import subprocess
import sys

import pytest
import torch
from torch._subclasses.fake_tensor import FakeTensorMode

import pointnet2_b200 as P
from pointnet2_b200 import _lib, _ops, layers, nets, sa_layer, tf_grouping, tf_interpolate, tf_sampling
from pointnet2_b200.pointnet_util import group_and_concat

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CUDA = torch.device("cuda")
I32, F32 = torch.int32, torch.float32


@pytest.fixture
def no_lib(monkeypatch):
    def refuse():
        raise AssertionError("the library was loaded")
    monkeypatch.setattr(_lib, "load", refuse)


def test_import_registers_every_op_without_loading_the_library():
    code = ("import torch, pointnet2_b200 as P\n"
            "assert P._lib._lib is None\n"
            "missing = [o for o in P._ops.OPS if not hasattr(torch.ops.pn2, o)]\n"
            "assert not missing, missing\n"
            "assert P._lib._lib is None\n")
    r = subprocess.run([sys.executable, "-c", code], cwd=ROOT, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    assert len(_ops.OPS) == len(set(_ops.OPS)) == 28


def _e(shape, dtype=F32):
    return torch.empty(shape, dtype=dtype, device=CUDA)


def _check(t, shape, dtype):
    assert tuple(t.shape) == tuple(shape) and t.dtype == dtype and t.device.type == "cuda", (t.shape, t.dtype, shape, dtype)


GRID = [(0, 40, 8, 4, 5), (3, 40, 8, 4, 5), (2, 300, 64, 16, 1), (1, 7, 7, 3, 33)]


@pytest.mark.parametrize("b,n,m,s,c", GRID)
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.float16])
@pytest.mark.parametrize("ragged", [False, True])
def test_fake_shapes(no_lib, b, n, m, s, c, dtype, ragged):
    ops = torch.ops.pn2
    with FakeTensorMode():
        xyz, q = _e((b, n, 3)), _e((b, m, 3))
        lens = _e((b,), I32) if ragged else None
        feats = _e((b, n, c), dtype)
        idx = _e((b, m, s), I32)
        _check(ops.farthest_point_sample(m, xyz, lens), (b, m), I32)
        i, nx = ops.farthest_point_sample_and_gather(m, xyz, lens)
        _check(i, (b, m), I32), _check(nx, (b, m, 3), F32)
        _check(ops.prob_sample(_e((b, n)), _e((b, m))), (b, m), I32)
        _check(ops.gather_point(xyz, _e((b, m), I32)), (b, m, 3), F32)
        _check(ops.gather_point_grad(_e((b, m, 3)), _e((b, m), I32), n), (b, n, 3), F32)
        i, cnt = ops.query_ball_point(0.2, s, xyz, q, lens)
        _check(i, (b, m, s), I32), _check(cnt, (b, m), I32)
        i, d = ops.select_top_k(s, _e((b, m, n)))
        _check(i, (b, m, n), I32), _check(d, (b, m, n), F32)
        _check(ops.group_point(feats, idx), (b, m, s, c), dtype)
        _check(ops.group_point_grad(_e((b, m, s, c), dtype), idx, n), (b, n, c), dtype)
        v, i = ops.knn_point(s, xyz, q, lens, lens)
        _check(v, (b, m, s), F32), _check(i, (b, m, s), I32)
        d, i = ops.three_nn(xyz, q, lens)
        _check(d, (b, n, 3), F32), _check(i, (b, n, 3), I32)
        pts2 = _e((b, m, c), dtype)
        _check(ops.three_interpolate(pts2, _e((b, n, 3), I32), _e((b, n, 3)), lens), (b, n, c), dtype)
        _check(ops.three_interpolate_grad(_e((b, n, c), dtype), _e((b, n, 3), I32), _e((b, n, 3)), lens, m), (b, m, c), dtype)
        for aux in (False, True):
            out, d, i, w = ops.three_nn_interpolate(xyz, q, pts2, lens, aux)
            _check(out, (b, n, c), dtype)
            shape = (b, n, 3) if aux else (0,)
            _check(d, shape, F32), _check(i, shape, I32), _check(w, shape, F32)
        _check(ops.fp_interpolate_concat(xyz, q, feats, pts2, lens), (b, n, 2 * c), dtype)
        _check(ops.fp_interpolate_concat(xyz, q, None, pts2, lens), (b, n, c), dtype)
        for want in (False, True):
            fi, nx, i, cnt, g = ops.sample_group(m, 0.2, s, xyz, True, want, lens)
            _check(fi, (b, m), I32), _check(nx, (b, m, 3), F32), _check(i, (b, m, s), I32), _check(cnt, (b, m), I32)
            _check(g, (b, m, s, 3) if want else (0,), F32)
            fi, nx, il, cl, gl = ops.sample_group_msg(m, [0.1, 0.2], [s, 2 * s], xyz, True, want, lens)
            _check(fi, (b, m), I32), _check(nx, (b, m, 3), F32)
            assert [tuple(t.shape) for t in il] == [(b, m, s), (b, m, 2 * s)] and all(t.dtype == I32 for t in il + cl)
            assert [tuple(t.shape) for t in cl] == [(b, m)] * 2
            assert [tuple(t.shape) for t in gl] == ([(b, m, s, 3), (b, m, 2 * s, 3)] if want else [])
            for want_d in (False, True):
                fi, nx, i, d, g = ops.sample_knn(m, s, xyz, True, want, want_d, lens)
                _check(i, (b, m, s), I32), _check(d, (b, m, s) if want_d else (0,), F32)
                _check(g, (b, m, s, 3) if want else (0,), F32)
            i, cnt, g = ops.ball_group(0.2, s, xyz, q, True, want)
            _check(i, (b, m, s), I32), _check(cnt, (b, m), I32), _check(g, (b, m, s, 3) if want else (0,), F32)
        for first in (False, True):
            out, g = ops.group_and_concat(xyz, q, feats, idx, first)
            _check(out, (b, m, s, 3 + c), dtype), _check(g, (b, m, s, 3), F32)
            out, g = ops.group_and_concat(xyz, q, None, idx, first)
            _check(out, (b, m, s, 3), F32)
        gx, gn, gp = ops.group_and_concat_backward(_e((b, m, s, 3 + c), dtype), _e((b, m, s, 3)), idx, n, True, True, True, True)
        _check(gx, (b, n, 3), F32), _check(gn, (b, m, 3), F32), _check(gp, (b, n, c), dtype)
        gx, gn, gp = ops.group_and_concat_backward(_e((b, m, s, 3)), None, idx, n, True, False, False, False)
        _check(gx, (0,), F32), _check(gn, (0,), F32), _check(gp, (0,), F32)
        rows = b * n
        x, keep = _e((rows, c), dtype), _e((rows,), torch.uint8)
        w, st, nbt = _e((c,)), _e((c,)), _e((), torch.int64)
        y, sm, si, rm2, rv2, nb2 = ops.masked_batch_norm_relu(x, w, w, keep, st, st, nbt, 1e-3, 0.1)
        _check(y, (rows, c), dtype), _check(sm, (c,), F32), _check(si, (c,), F32)
        _check(rm2, (c,), F32), _check(rv2, (c,), F32), _check(nb2, (), torch.int64)
        y, sm, si, rm2, rv2, nb2 = ops.masked_batch_norm_relu(x, None, None, keep, None, None, None, 1e-3, -1.0)
        _check(rm2, (0,), F32), _check(nb2, (0,), torch.int64)
        dx, dg, db = ops.masked_batch_norm_relu_backward(x, x, x, keep, w, sm, si)
        _check(dx, (rows, c), dtype), _check(dg, (c,), F32), _check(db, (c,), F32)
        x3 = _e((b, n, c), dtype)
        out, am, sm, si, rm2, rv2, nb2 = ops.masked_bn_relu_max(x3, w, w, keep, st, st, nbt, 1e-3, 0.1)
        _check(out, (b, c), dtype), _check(am, (b, c), I32), _check(rm2, (c,), F32)
        dx, dg, db = ops.masked_bn_relu_max_backward(_e((b, c), dtype), x3, out, am, keep, None, sm, si)
        _check(dx, (b, n, c), dtype), _check(dg, (0,), F32)
        mlp = layers.SharedMLP(c + 3, [16, 24])
        params, eps, relu = layers._stack_params(layers._mlp_stack(mlp))
        params = [None if p is None else _e(tuple(p.shape)) for p in params]
        _check(ops.sa_mlp_max(xyz, q, feats, idx, None, params, eps, relu, True, True, dtype), (b, m, 24), dtype)
        _check(ops.sa_mlp_max(xyz, None, feats, None, lens, params, eps, relu, True, True, dtype), (b, 1, 24), dtype)
        _check(ops.fp_mlp(xyz, q, _e((b, n, 3), dtype), pts2, lens, params, eps, relu, dtype), (b, n, 24), dtype)
        _check(ops.mlp_rows(_e((b, n, s, c + 3), dtype), None, params, eps, relu, dtype), (b, n, s, 24), dtype)


def _export(fn, args):
    class Wrap(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.mods = torch.nn.ModuleList([a for a in [getattr(fn, "__self__", None)] if isinstance(a, torch.nn.Module)])

        def forward(self, *a):
            return fn(*a)

    return torch.export.export(Wrap(), args, strict=False)


def _pn2_ops(ep):
    return {str(nd.target).split(".")[1] for gm in ep.graph_module.modules() if hasattr(gm, "graph")
            for nd in gm.graph.nodes if str(nd.target).startswith("pn2.")}


NETS = [  # class, channels, n, logits shape (b, n) -> tuple, training ops, eval ops
    (nets.PointNet2SemSeg, 3, 2048, lambda b, n: (b, n, 21), {"sample_group", "group_and_concat", "three_nn", "three_interpolate"},
     {"sample_group", "sa_mlp_max", "fp_interpolate_concat"}),
    (nets.PointNet2ClsSSG, 3, 1024, lambda b, n: (b, 40), {"sample_group", "group_and_concat"}, {"sample_group", "sa_mlp_max"}),
    (nets.PointNet2ClsMSG, 3, 1024, lambda b, n: (b, 40), {"sample_group_msg", "group_and_concat"},
     {"sample_group_msg", "sa_mlp_max"}),
    (nets.PointNet2PartSeg, 6, 1024, lambda b, n: (b, n, 50), {"sample_group", "group_and_concat", "three_nn", "three_interpolate"},
     {"sample_group", "sa_mlp_max", "fp_interpolate_concat"}),
    (nets.PointNet2PartSegMSG, 6, 1024, lambda b, n: (b, n, 50),
     {"sample_group_msg", "group_and_concat", "three_nn", "three_interpolate"},
     {"sample_group_msg", "sa_mlp_max", "fp_interpolate_concat"}),
    (nets.PointNetClsBasic, 3, 1024, lambda b, n: (b, 40), {"masked_batch_norm_relu", "masked_bn_relu_max"}, {"sa_mlp_max"}),
]


@pytest.mark.parametrize("cls,ch,n,logits,train_ops,eval_ops", NETS, ids=[c[0].__name__ for c in NETS])
@pytest.mark.parametrize("train", [True, False], ids=["train", "eval"])
@pytest.mark.parametrize("ragged", [False, True], ids=["dense", "ragged"])
def test_export_networks(no_lib, cls, ch, n, logits, train_ops, eval_ops, train, ragged):
    b = 4
    with FakeTensorMode(allow_non_fake_inputs=True):
        with torch.device("cuda"):
            net = cls().train(train)
        x = _e((b, n, ch))
        extra = (_e((b,), torch.int64),) if cls is nets.PointNet2PartSegMSG else ()
        lens = (_e((b,), I32),) if ragged else ()
        args = (x, *extra, *lens)

        class Step(torch.nn.Module):
            def __init__(self):
                super().__init__()
                self.net = net

            def forward(self, *a):
                if train:
                    return self.net(*a)[0]
                with torch.no_grad():
                    return self.net(*a)[0]

        ep = torch.export.export(Step(), args, strict=False)
    want = set(train_ops if train else eval_ops)
    if train and ragged and cls in (nets.PointNet2SemSeg, nets.PointNet2PartSeg, nets.PointNet2PartSegMSG):
        want.add("masked_batch_norm_relu")  # the padded rows' batch norms of the dense level
    assert _pn2_ops(ep) == want
    out = [nd for nd in ep.graph.nodes if nd.op == "output"][0].args[0][0].meta["val"]
    assert tuple(out.shape) == logits(b, n)


def _fake_call(fn, args, export: bool):
    """the exception type of fn(*args) on fake CUDA tensors, in an eager call or under torch.export"""
    try:
        with FakeTensorMode(allow_non_fake_inputs=True):
            real = [a() if callable(a) else a for a in args]
            if export:
                _export(fn, tuple(t for t in real if isinstance(t, torch.Tensor)))
            else:
                fn(*[t for t in real if isinstance(t, torch.Tensor)])
    except Exception as e:  # noqa: BLE001
        return type(e)
    return None


BAD = [
    (lambda x, i: tf_sampling.gather_point(x, i), [lambda: _e((2, 8, 3), torch.float64), lambda: _e((2, 4), I32)], TypeError),
    (lambda x, i: tf_sampling.gather_point(x, i), [lambda: _e((2, 8, 4)), lambda: _e((2, 4), I32)], ValueError),
    (lambda p, i: tf_grouping.group_point(p, i), [lambda: _e((2, 8, 5)), lambda: _e((2, 4, 3))], TypeError),
    (lambda p, i: tf_grouping.group_point(p, i), [lambda: _e((2, 8, 5)), lambda: _e((3, 4, 3), I32)], ValueError),
    (lambda x: tf_sampling.farthest_point_sample(4, x), [lambda: _e((2, 8, 2))], ValueError),
    (lambda x, q: tf_interpolate.three_nn(x, q), [lambda: _e((2, 8, 3), torch.float16), lambda: _e((2, 4, 3))], TypeError),
    (lambda x, l: sa_layer.sample_group(4, 0.2, 8, x, lengths=l), [lambda: _e((2, 8, 3)), lambda: _e((3,), I32)], ValueError),
    (lambda x, l: sa_layer.sample_group(4, 0.2, 8, x, lengths=l), [lambda: _e((2, 8, 3)), lambda: _e((2,))], TypeError),
    (lambda x, q, p, i: group_and_concat(x, q, p, i), [lambda: _e((2, 8, 3)), lambda: _e((2, 4, 3)), lambda: _e((2, 7, 5)),
                                                       lambda: _e((2, 4, 3), I32)], ValueError),
]


@pytest.mark.parametrize("k", range(len(BAD)))
def test_errors_match_eager(no_lib, k):
    fn, args, want = BAD[k]
    assert _fake_call(fn, args, export=False) is want
    assert _fake_call(fn, args, export=True) is want


def test_host_lengths_export_as_constants(no_lib):
    """a host sequence of lengths is checked at trace time (ValueError as in eager) and becomes a constant"""
    with FakeTensorMode(allow_non_fake_inputs=True):
        x = _e((2, 64, 3))
        ep = _export(lambda x: tf_sampling.farthest_point_sample(8, x, lengths=[64, 30]), (x,))
        assert _pn2_ops(ep) == {"farthest_point_sample"}
        with pytest.raises(ValueError):
            _export(lambda x: tf_sampling.farthest_point_sample(8, x, lengths=[65, 30]), (x,))


def test_batch_invariant_eval_exports_to_the_row_kernels(no_lib):
    with FakeTensorMode(allow_non_fake_inputs=True):
        with torch.device("cuda"):
            net = nets.PointNet2SemSeg().eval()
        x = _e((2, 2048, 3))

        class Step(torch.nn.Module):
            def __init__(self):
                super().__init__()
                self.net = net

            def forward(self, x):
                with torch.no_grad(), P.batch_invariant():
                    return self.net(x)[0]

        ep = torch.export.export(Step(), (x,), strict=False)
    assert _pn2_ops(ep) == {"sample_group", "sa_mlp_max", "fp_mlp", "mlp_rows"}
