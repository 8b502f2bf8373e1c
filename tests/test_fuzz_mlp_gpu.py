"""The fused inference MLP kernels (sa_mlp_max_kernel, row_mlp_kernel) on the GPU: a fixed-seed slice of
tests/fuzz_mlp_gpu.py; an edge table with one shape per planner branch, each compared with the float32 C oracle or
the 16-bit bound and each checked against the planner restatement through the launched kernel's name and grid in a
torch.profiler trace; and defects on the oracle side that the comparisons must catch on real kernel output."""
import json
import os
import re
import tempfile

import numpy as np
import pytest
import torch

import fuzz_mlp_gpu as F
import mlp_oracle as MO
import numerics as NUM
from oracle import oracle as O

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("seed", F.SLICE_SEEDS)
def test_random_mlp_cases_match_oracle(dev, seed):
    stats = {}
    counts, fails = F.run(seed, F.SLICE_ITERATIONS, stats)
    assert counts == {name: F.SLICE_ITERATIONS // len(F.CASES) for name in F.CASES}
    print(f"seed {seed}: worst 16-bit err / bound {stats.get('worst_ratio', 0):.3g} over {stats.get('elements', 0)} "
          f"elements, {stats.get('unbounded', 0)} past the format's range")
    assert not fails, fails


# ------------------------------------------------------------------------------------------------- edge table
def _sa(name, fmt, c, widths, k, b, s, use_xyz=True, xyz_first=True, group_all=False, sl=None):
    rs = np.random.RandomState(sum(map(ord, name)))
    cin = c + 3 if (use_xyz or c == 0) else c
    n = k if group_all else max(k, 50)
    xyz = rs.random_sample((b, n, 3)).astype(np.float32)
    p = dict(case="sa", fmt=fmt, autocast=c == 0 and fmt != "f32", b=b, n=n, s=1 if group_all else s, k=k, c=c,
             cin=cin, widths=widths, group_all=group_all, xyz_first=xyz_first, use_xyz=use_xyz, slice=sl,
             xyz=xyz, new_xyz=None if group_all else xyz[:, rs.randint(0, n, s)].copy(),
             idx=None if group_all else rs.randint(0, n, (b, s, k)).astype(np.int32),
             points=F._scaled(rs, (b, n, c), fmt) if c else None) | F._layers(rs, cin, widths, fmt)
    plan = MO.sa_plan(MO.ESIZE[fmt], cin, widths, k, b * p["s"])
    return name, p, plan


def _rows(name, fmt, c, widths, rows, masked=False, sl=None):
    rs = np.random.RandomState(sum(map(ord, name)))
    p = dict(case="rows", fmt=fmt, autocast=False, rows=rows, lead=(rows,), c=c, cin=c, widths=widths, slice=sl,
             x=F._scaled(rs, (rows, c), fmt), mask=(rs.rand(rows) < 0.7) if masked else None) | F._layers(rs, c, widths, fmt)
    return name, p, MO.row_plan(MO.ESIZE[fmt], c, widths, rows)


def _fp(name, fmt, c2, c1, widths, b, n, m, lengths=None, sl=None):
    rs = np.random.RandomState(sum(map(ord, name)))
    p = dict(case="fp", fmt=fmt, autocast=False, b=b, n=n, m=m, c2=c2, c1=c1, cin=c2 + c1, widths=widths,
             lengths=lengths, slice=sl, xyz1=rs.random_sample((b, n, 3)).astype(np.float32),
             xyz2=rs.random_sample((b, m, 3)).astype(np.float32), p2=F._scaled(rs, (b, m, c2), fmt),
             p1=F._scaled(rs, (b, n, c1), fmt) if c1 else None) | F._layers(rs, c2 + c1, widths, fmt)
    return name, p, MO.row_plan(MO.ESIZE[fmt], c2 + c1, widths, b * n)


EDGES = [
    # the plans no other test launched: float32 TM 16, 16-bit TM 32, TM 32 with several groups, the slot trimming
    _sa("sa_f32_tm16_pieces", "f32", 1024, [512, 1024], 64, 1, 2),  # misses TM 32 by 128 bytes
    _sa("sa_bf16_tm32", "bf16", 1024, [1024, 32], 32, 1, 3),
    _sa("sa_f16_tm32_pieces", "f16", 1024, [1024, 65], 33, 1, 2, sl=(3, 2)),
    _sa("sa_f32_tm32_groups", "f32", 256, [1024, 64], 7, 1, 13),
    _sa("sa_bf16_tm32_groups", "bf16", 1024, [1024, 32], 5, 1, 13, xyz_first=False),
    _sa("sa_f32_trimmed", "f32", 0, [1024], 1, 2, 60),
    _sa("sa_bf16_trimmed_autocast", "bf16", 0, [1024], 1, 2, 60),
    _sa("sa_f16_extreme_trimmed", "f16", 1024, [1024] * 4, 1, 1, 40),   # 1027 -> [1024] x 4 at K = 1
    _sa("sa_f32_extreme", "f32", 1024, [1024] * 4, 1, 1, 20),
    _sa("sa_f16_group_all", "f16", 5, [33, 65], 200, 2, 1, group_all=True),
    _sa("sa_f32_k5", "f32", 8, [63, 129], 5, 2, 30, xyz_first=False, sl=(1, 4)),
    _sa("sa_bf16_features_only_c1", "bf16", 1, [7, 1], 17, 3, 9, use_xyz=False),
    _rows("rows_f32_tm16_extreme", "f32", 1536, [1024] * 4, 17),         # 1536 -> [1024] x 4
    _rows("rows_bf16_tm32", "bf16", 1536, [1024, 65], 70, masked=True),
    _rows("rows_f32_tm32_four_layers", "f32", 7, [1, 65, 1024, 33], 130, sl=(2, 5)),
    _rows("rows_f32_tm64", "f32", 65, [129, 7], 200, masked=True),
    _rows("rows_f16_tm64", "f16", 33, [64], 64, masked=True),
    _fp("fp_f16_tm32", "f16", 1024, 512, [256, 256], 2, 40, 9, lengths=[40, 17]),
    _fp("fp_f32_tm16", "f32", 1024, 512, [256, 256], 2, 40, 9, lengths=[3, 40], sl=(0, 3)),
    _fp("fp_bf16_tm64", "bf16", 131, 0, [129, 1], 3, 150, 20),
]
KERNEL_DTYPE = {"f32": "float", "bf16": "__nv_bfloat16", "f16": "__half"}


def test_edge_table_reaches_every_reachable_branch():
    seen = set()
    for _, p, plan in EDGES:
        kind = "sa" if p["case"] == "sa" else "rows"
        rows = None if kind == "sa" else (p["rows"] if p["case"] == "rows" else p["b"] * p["n"])
        seen |= MO.branches(kind, MO.ESIZE[p["fmt"]], p["cin"], p["widths"], plan, k=p.get("k"), rows=rows)
    import test_fuzz_mlp_cpu as C
    assert C.REQUIRED_BRANCHES <= seen, sorted(C.REQUIRED_BRANCHES - seen)


def _launches(fn):
    """fn() under torch.profiler: the (name, args) of every fused-MLP kernel it launched"""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "trace.json")
        prof.export_chrome_trace(path)
        with open(path) as f:
            events = json.load(f)["traceEvents"]
    return [(e["name"], e.get("args", {})) for e in events
            if e.get("cat") == "kernel" and re.search(r"(sa_mlp_max|row_mlp)_kernel", e.get("name", ""))]


@pytest.mark.parametrize("edge", EDGES, ids=[e[0] for e in EDGES])
def test_edge_against_oracle_and_plan(dev, edge):
    name, p, plan = edge
    stats = {}
    launches = _launches(lambda: stats.update(ok=F.RUN[p["case"]](p, stats)))
    assert stats["ok"], name
    assert len(launches) == 1, launches
    kname, args = launches[0]
    m = re.search(r"(sa_mlp_max|row_mlp)_kernel<([\w:]+), (\d+)>", kname)
    assert m, kname
    want_kernel = "sa_mlp_max" if p["case"] == "sa" else "row_mlp"
    assert (m.group(1), m.group(2), int(m.group(3))) == (want_kernel, KERNEL_DTYPE[p["fmt"]], plan["tm"]), kname
    grid = args.get("grid")
    if grid is not None:
        assert list(grid) == [plan["grid"], 1, 1], (grid, plan)
    smem = args.get("shared memory")
    if smem is not None:
        assert int(smem) == plan["smem"], (smem, plan)
    print(f"{name}: {kname} grid {grid} smem {smem} (planned {plan}); 16-bit err / bound "
          f"{stats.get('worst_ratio', 0):.3g}")


# -------------------------------------------------------------------------------------------------- mutations
@pytest.mark.parametrize("case", ["sa", "rows"])
@pytest.mark.parametrize("fmt", ["f32", "bf16", "f16"])
def test_comparison_catches_every_mutation(dev, fmt, case):
    """A kernel with one of these defects would give what the mutated oracle gives: on real kernel output the
    comparison must accept the true reference and reject every mutated one."""
    rs = np.random.RandomState(31)
    layers = F.mutation_layers(rs)
    if case == "sa":
        _, p, _ = _sa("mutations", fmt, 34, [96, 80], 8, 2, 16)
        p.update(layers=layers)
        got, _, rows = F.sa_output(p)
        rows, pool_k = rows.reshape(-1, rows.shape[-1]), 8
    else:
        _, p, _ = _rows("mutations", fmt, 37, [96, 80], 100)
        p.update(layers=layers)
        got, _, x = F.rows_output(p)
        rows, pool_k = NUM.quantize(x, fmt), None
    got = F.values(got).reshape(-1, 80)
    assert F.compare(got, rows, layers, fmt, pool_k)
    for kind in MO.MUTATIONS:
        bad = F.oracle_layers(MO.mutate(layers, kind))
        if fmt == "f32":
            want = O.oracle_mlp_rows_f32(rows, bad)
            want = MO.max_pool(want, pool_k) if pool_k else want
            if kind == "swap":
                want = MO.swap_partial_pass(want)
            assert not F.same_values(got, want), kind
        else:
            ref, bound = MO.bound16(rows, MO.mutate(layers, kind), [O.oracle_mlp_affine_f32(L) for L in bad], fmt,
                                    pool_k)
            if kind == "swap":
                ref, bound = MO.swap_partial_pass(ref), MO.swap_partial_pass(bound)
            assert not MO.check16(got, ref, bound)[0], kind
