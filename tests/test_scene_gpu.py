"""GPU tests of whole-scene segmentation (csrc/scene.cu, pointnet2_b200/scene.py): the block partition against the
numpy oracle bit for bit, determinism, the ordered merge against a float32 sequential restatement in every logits
dtype, chunked against whole merges, and predict_scene with a seeded PointNet2SemSeg against blocks run alone."""
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import scene_oracle as SO  # noqa: E402

from pointnet2_b200 import _lib, scene, workloads as W  # noqa: E402
from pointnet2_b200.nets import PointNet2SemSeg  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
FIELDS = ("xyz", "lengths", "point_idx", "core", "block", "occ_off", "occ_row")


def _bits(a: np.ndarray) -> np.ndarray:
    return a.view(np.int32) if a.dtype == np.float32 else a


def _edges():
    base = np.array([0.0, 1.5, 3.0, 4.5, 1.7, 1.3, 0.5, 1.0, 2.0, 2.5], np.float32)
    edge = np.concatenate([base, np.nextafter(base, np.float32(-1)), np.nextafter(base, np.float32(9))])
    return np.stack(np.meshgrid(edge, edge, [0.0, 1.0]), -1).reshape(-1, 3).astype(np.float32)


def _dups():
    d = W.cloud_duplicates(1, 200000, 11)[0] * np.float32(3.0)
    return d.astype(np.float32)


SCENES = {
    "room_150k": lambda: W.scene_room(150000, 1)[0],
    "room_2M": lambda: W.scene_room(2000000, 2)[0],
    "dups": _dups,
    "edges": _edges,
    "one_point": lambda: np.array([[0.25, -3.0, 1.0]], np.float32),
    "shared_x": lambda: np.stack([np.full(5000, 2.0, np.float32), np.linspace(-3, 4, 5000, dtype=np.float32),
                                  np.zeros(5000, np.float32)], 1),
}
CASES = [("room_150k", {}), ("room_150k", dict(stride=0.5)), ("room_150k", dict(max_points=64)), ("room_2M", {}),
         ("dups", {}), ("dups", dict(stride=0.5, max_points=64)), ("edges", {}), ("edges", dict(stride=0.5)),
         ("one_point", {}), ("shared_x", {}), ("shared_x", dict(stride=0.5, max_points=64)),
         ("room_150k", dict(block_size=1.0, padding=0.0, max_points=1000))]


def _run(xyz, **kw):
    return scene.scene_blocks(torch.from_numpy(xyz).to(DEV), **kw)


@pytest.mark.parametrize("name,kw", CASES, ids=[f"{n}-{'-'.join(f'{k}{v}' for k, v in kw.items()) or 'default'}" for n, kw in CASES])
def test_scene_blocks_match_oracle(name, kw):
    xyz = SCENES[name]()
    got = _run(xyz, **kw)
    want = SO.oracle_scene_blocks(xyz, **kw)
    for f in FIELDS:
        g = getattr(got, f).cpu().numpy()
        assert g.shape == want[f].shape, (f, g.shape, want[f].shape)
        assert np.array_equal(_bits(g), _bits(want[f].astype(g.dtype))), f
    assert got.lengths.dtype == torch.int32 and got.core.dtype == torch.bool
    counts = np.diff(got.occ_off.cpu().numpy())
    assert counts.min() >= 1  # every point is scored at least once
    if kw.get("stride") == 0.5:
        assert counts.max() <= 16  # size 1.5 at stride 0.5: up to 4 x 4 cores ...
        if name == "edges":
            assert counts.max() == 16  # ... reached by points on the grid lines


def test_scene_blocks_deterministic():
    xyz = torch.from_numpy(W.scene_room(300000, 5)[0]).to(DEV)
    a = scene.scene_blocks(xyz, stride=0.5, max_points=2048)
    b = scene.scene_blocks(xyz, stride=0.5, max_points=2048)
    for f in FIELDS:
        assert torch.equal(getattr(a, f), getattr(b, f)), f


def test_scene_blocks_rejects_non_finite():
    xyz = torch.from_numpy(W.scene_room(1000, 1)[0]).to(DEV)
    before = _lib.launch_count()
    for bad in (float("nan"), float("inf")):
        x = xyz.clone()
        x[17, 2] = bad
        with pytest.raises(ValueError, match="finite"):
            scene.scene_blocks(x)
    assert _lib.launch_count() == before


def _host(blocks):
    return {f: getattr(blocks, f).cpu().numpy() for f in FIELDS}


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.float16])
def test_merge_matches_sequential_sum(dtype):
    xyz = torch.from_numpy(W.scene_room(150000, 3)[0]).to(DEV)
    blocks = scene.scene_blocks(xyz, stride=0.5, max_points=4096)
    b, n = blocks.point_idx.shape
    c = 21
    g = torch.Generator(device=DEV).manual_seed(0)
    logits = (torch.randn(b, n, c, device=DEV, generator=g) * 4).to(dtype)
    start = torch.randn(xyz.shape[0], c, device=DEV, generator=g)
    whole = scene.merge_block_logits(blocks, logits, start.clone())
    want = SO.sequential_merge(_host(blocks), logits.float().cpu().numpy(), start.cpu().numpy())
    assert np.array_equal(whole.cpu().numpy().view(np.int32), want.view(np.int32))
    # chunk by chunk, in uneven chunks: the same bits, and no host synchronisation
    acc = start.clone()
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        for b0, b1 in ((0, 3), (3, 4), (4, 17), (17, b)):
            scene.merge_block_logits(blocks, logits[b0:b1], acc, row_begin=b0 * n)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert torch.equal(acc.view(torch.int32), whole.view(torch.int32))


def test_merge_wide_classes_and_repeat():
    """More classes than a warp has lanes; two merges give the same bits."""
    xyz = torch.from_numpy(W.scene_room(40000, 6)[0]).to(DEV)
    blocks = scene.scene_blocks(xyz, max_points=1024)
    b, n = blocks.point_idx.shape
    logits = torch.randn(b, n, 70, device=DEV)
    a = scene.merge_block_logits(blocks, logits, torch.zeros(xyz.shape[0], 70, device=DEV))
    a2 = scene.merge_block_logits(blocks, logits, torch.zeros(xyz.shape[0], 70, device=DEV))
    want = SO.sequential_merge(_host(blocks), logits.cpu().numpy(), np.zeros((xyz.shape[0], 70), np.float32))
    assert np.array_equal(a.cpu().numpy().view(np.int32), want.view(np.int32))
    assert torch.equal(a, a2)


def _seeded_net():
    torch.manual_seed(0)
    net = PointNet2SemSeg(21).to(DEV)
    # train briefly on random data so the running statistics are not the identity
    net.train()
    with torch.no_grad():
        for s in range(2):
            net(torch.rand(4, 2048, 3, device=DEV) * 1.5)
    return net.eval()


def test_predict_scene_against_blocks_alone():
    net = _seeded_net()
    xyz = torch.from_numpy(W.scene_room(40000, 9)[0]).to(DEV)
    kw = dict(max_points=2048)
    captured = {"sa1": [], "logits": []}
    h1 = net.sa1.register_forward_hook(lambda m, i, o: captured["sa1"].append(o[2].clone()))
    h2 = net.register_forward_hook(lambda m, i, o: captured["logits"].append(o[0].clone()))
    try:
        accum, count, label = scene.predict_scene(net, xyz, batch_size=16, **kw)
        sa1 = torch.cat(captured["sa1"])
        logits = torch.cat(captured["logits"])
        blocks = scene.scene_blocks(xyz, **kw)
        lengths = blocks.lengths.cpu().tolist()
        assert len(lengths) > 16  # more than one chunk
        for bi, ln in enumerate(lengths):
            captured["sa1"].clear()
            captured["logits"].clear()
            with torch.no_grad():
                net(blocks.xyz[bi:bi + 1, :ln].contiguous())
            assert torch.equal(captured["sa1"][0][0], sa1[bi]), bi
            torch.testing.assert_close(captured["logits"][0][0], logits[bi, :ln], rtol=1e-4, atol=1e-4)
    finally:
        h1.remove()
        h2.remove()
    assert count.min().item() >= 1 and count.dtype == torch.int32
    assert label.shape == (xyz.shape[0],) and torch.equal(label, accum.argmax(1))
    # the merged sums are those of the captured logits
    want = SO.sequential_merge(_host(blocks), logits.cpu().numpy(), np.zeros(accum.shape, np.float32))
    assert np.array_equal(accum.cpu().numpy().view(np.int32), want.view(np.int32))
    accum2, count2, label2 = scene.predict_scene(net, xyz, batch_size=16, **kw)
    assert torch.equal(accum, accum2) and torch.equal(count, count2) and torch.equal(label, label2)
    accum1, _, _ = scene.predict_scene(net, xyz, batch_size=1, **kw)
    torch.testing.assert_close(accum1, accum, rtol=1e-4, atol=1e-4)


def test_voxel_labels_on_device_match_pc_util():
    pts, lab = W.scene_room(100000, 4)
    pred = np.roll(lab, 7)
    keys, labels, _ = scene.surface_voxel_labels(torch.from_numpy(pts).to(DEV),
                                                 torch.from_numpy(np.stack([lab, pred], 1)).to(DEV), 0.02)
    wk, wl, _ = SO.reference_voxel_labels(pts, np.stack([lab, pred], 1), 0.02)
    np.testing.assert_array_equal(keys.cpu().numpy(), wk)
    np.testing.assert_array_equal(labels.cpu().numpy(), wl)
