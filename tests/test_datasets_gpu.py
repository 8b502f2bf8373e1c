"""GPU tests of the dataset loaders (DESIGN.md §6.18): the device text parser against np.loadtxt and the restated
grammar on adversarial files, the streaming layer across many chunks, and load_modelnet / load_shapenet_part /
load_scannet against what the reference's readers make of the seeded fixture trees."""
import os
import sys
import warnings

import numpy as np
import pytest
import torch

from oracle import dataset_ref as D
from pointnet2_b200 import _lib, datasets
from pointnet2_b200._tensor import ptr, stream_ptr
from pointnet2_b200.scene import sample_crops
from pointnet2_b200.shapes import sample_shapes

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import text_oracle as T  # noqa: E402

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
DEV = torch.device("cuda", 0)


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _field(rng):
    """A field in the grammar (mostly), or one of the strings that send a file to the host."""
    r = rng.random()
    if r < 0.55:
        return "%.6f" % rng.uniform(-3, 3)
    if r < 0.75:
        forms = ["-0.000000", "+.5", "1e5", "2.5E-7", "-3e+0", "17", "0.1", "9007199254740992", "1.25e22", "4e-22",
                 "123456.789012", "0000.0001", "3.4028235e38"]
        return forms[int(rng.integers(len(forms)))]
    if r < 0.97:
        nd = int(rng.integers(1, 17))
        s = "".join(str(d) for d in rng.integers(0, 10, nd))
        p = int(rng.integers(0, nd))
        return ("-" if rng.random() < 0.5 else "") + s[:p] + "." + s[p:] + ("e%d" % rng.integers(-12, 12)
                                                                           if rng.random() < 0.3 else "")
    bad = ["nan", "inf", "1_0", "1.", "9007199254740993", "1e23", "0.12345678901234567", "1e-23"]
    return bad[int(rng.integers(len(bad)))]


def _corpus(rng, ncol, delim, nfiles):
    """Files of random lines: mostly in the grammar, some with one line of each kind outside it, some long enough
    that lines cross the kernel's 8 KB tiles, with "\\r\\n" or "\\n" and with or without a final terminator."""
    sep = "," if delim == T.COMMA else " "
    files = []
    for k in range(nfiles):
        n = int(rng.choice([2, 3, 50, 200, 700, 3000]))
        kind = k % 8
        odd = 0.05 if kind in (4, 6) else 0.0  # fields of every form, some outside the grammar or the exact path
        lines = []
        for _ in range(n):
            vals = [_field(rng) if rng.random() < odd else "%.6f" % rng.uniform(-2, 2) for _ in range(ncol)]
            line = sep.join(vals)
            if delim == T.WHITESPACE and rng.random() < 0.05:
                line = " \t" + line.replace(" ", "\t ") + "  "
            lines.append(line)
        if kind == 1 and n > 2:  # one line outside the grammar somewhere
            i = int(rng.integers(0, n))
            lines[i] = [lines[i] + sep + "1.0", "", lines[i].replace(sep, sep + "# ", 1),
                        lines[i][:-1] + "\r" + lines[i][-1:], sep.join(["1e-30"] * ncol),
                        lines[i].replace(sep, sep + sep, 1)][int(rng.integers(0, 6))]
        eol = "\r\n" if kind in (2, 5) else "\n"
        text = eol.join(lines) + ("" if kind in (3, 5) else eol)
        files.append(text.encode())
    return files


def _device_verdicts(blobs, ncol, delim, keep):
    lib = _lib.load()
    off = np.zeros(len(blobs) + 1, np.int64)
    np.cumsum([len(b) for b in blobs], out=off[1:])
    text = torch.from_numpy(np.frombuffer(b"".join(blobs) or b"\0", np.uint8).copy()).to(DEV)
    file_off = torch.from_numpy(off).to(DEV)
    rows = torch.empty(len(blobs), dtype=torch.int64, device=DEV)
    status = torch.empty(len(blobs), dtype=torch.int32, device=DEV)
    s = stream_ptr(DEV)
    _lib.check(lib.pn2_text_rows_scan(len(blobs), ptr(text), ptr(file_off), int(off[-1]), ncol, delim, ptr(rows),
                                      ptr(status), s), "scan")
    rows_h, status_h = rows.cpu().numpy(), status.cpu().numpy()
    kept = np.where(status_h == 0, np.minimum(rows_h, keep), 0)
    row_off = np.zeros(len(blobs) + 1, np.int64)
    np.cumsum(kept, out=row_off[1:])
    out = torch.full((int(row_off[-1]) + 1, ncol), 7.0, device=DEV)  # one guard row past the end
    _lib.check(lib.pn2_text_rows_parse(len(blobs), ptr(text), ptr(file_off), int(off[-1]), ncol, delim, ptr(status),
                                       keep, ptr(torch.from_numpy(row_off).to(DEV)), ptr(out), int(row_off[-1]), s),
               "parse")
    out_h = out.cpu().numpy()
    assert (out_h[-1] == 7.0).all()
    return rows_h, status_h, [out_h[row_off[i]:row_off[i + 1]] for i in range(len(blobs))]


def _loadtxt(blob, delim, tmp_path):
    p = tmp_path / "f.txt"
    p.write_bytes(blob)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        return np.loadtxt(str(p), delimiter="," if delim == T.COMMA else None).astype(np.float32)


@pytest.mark.parametrize("delim,ncol", [(T.COMMA, 6), (T.WHITESPACE, 7), (T.COMMA, 1), (T.WHITESPACE, 3)])
def test_device_parser_equals_loadtxt_and_the_grammar(delim, ncol, tmp_path):
    rng = np.random.default_rng(100 + 10 * delim + ncol)
    blobs = _corpus(rng, ncol, delim, 96) + [b"", b"1" + b",1" * (ncol - 1) + b"\n" if delim == T.COMMA else
                                             b" ".join([b"1"] * ncol)]
    for keep in (1 << 40, 100):
        rows, status, tables = _device_verdicts(blobs, ncol, delim, keep)
        on_device = 0
        for i, blob in enumerate(blobs):
            want_status, want_rows = T.classify_file(blob, ncol, delim)
            assert status[i] == want_status, (i, status[i], want_status)
            if status[i] != T.OK:
                continue
            on_device += 1
            assert rows[i] == len(want_rows)
            assert np.array_equal(_bits(tables[i]), _bits(want_rows[:keep]))
            if len(want_rows) >= 1:
                ref = _loadtxt(blob, delim, tmp_path).reshape(len(want_rows), ncol)
                assert np.array_equal(_bits(tables[i]), _bits(ref[:keep])), i
        assert on_device >= len(blobs) // 2  # a parser that leaves everything to the host fails here
        assert (status != T.OK).sum() >= 6


def test_tile_boundaries_and_long_lines(tmp_path):
    """Lines ending exactly at, just before and just after a tile boundary, and one line longer than a tile."""
    blobs = []
    for pad in (0, 1, 2, 7, 8, 9):
        line = "1.500000," + "0" * (8192 - 12 - pad) + "1,2"  # the first '\n' near byte 8192
        blobs.append((line + "\n" + "3,4,5\n" * 50).encode())
    blobs.append((",".join(["1.25"] * 3) + "\n").encode() * 3000)
    blobs.append(("1" + "0" * 20000 + "e-20000,2,3\n4,5,6").encode())  # inexact: M has more than 16 digits
    rows, status, tables = _device_verdicts(blobs, 3, T.COMMA, 1 << 40)
    for i, blob in enumerate(blobs):
        s, want = T.classify_file(blob, 3, T.COMMA)
        assert status[i] == s
        if s == T.OK:
            assert np.array_equal(_bits(tables[i]), _bits(_loadtxt(blob, T.COMMA, tmp_path)))
    assert status[-1] == T.INEXACT and (status[:-1] == T.OK).all()


def _write(tmp_path, blobs):
    paths = []
    for i, b in enumerate(blobs):
        p = tmp_path / f"f{i:03d}.txt"
        p.write_bytes(b)
        paths.append(str(p))
    return paths


def _table_ok(blob, tmp_path):
    try:
        return _loadtxt(blob, T.COMMA, tmp_path).ndim == 2
    except ValueError:
        return False


def test_streaming_over_many_chunks_and_a_file_larger_than_a_chunk(tmp_path):
    rng = np.random.default_rng(5)
    blobs = [b for b in _corpus(rng, 6, T.COMMA, 60) if _table_ok(b, tmp_path)]
    big = ("\n".join(",".join("%.6f" % v for v in row) for row in rng.uniform(-1, 1, (4000, 6))) + "\n").encode()
    blobs.insert(7, big)
    paths = _write(tmp_path, blobs)
    for keep in (1 << 40, 64):
        stats = {}
        got = datasets._read_tables(paths, 6, datasets.DELIM_COMMA, keep=keep, chunk_bytes=64 << 10, stats=stats)
        assert stats["chunks"] >= 5 and len(big) > 64 << 10
        assert stats["fallback"] == sum(T.classify_file(b, 6, T.COMMA)[0] != T.OK for b in blobs) > 0
        for p, g in zip(paths, got):
            want = np.loadtxt(p, delimiter=",").astype(np.float32)[:keep]
            assert g.shape == want.shape and np.array_equal(_bits(g), _bits(want)), p
    # a chunk whose files are all the host's: nothing to convert on the device
    host_only = _write(tmp_path, [b"1,2,3,4,5,6\n# c\n7,8,9,10,11,12\n"] * 3)
    got = datasets._read_tables(host_only, 6, datasets.DELIM_COMMA)
    assert all(np.array_equal(g, np.float32([[1, 2, 3, 4, 5, 6], [7, 8, 9, 10, 11, 12]])) for g in got)


def test_empty_and_one_row_files_are_refused_by_name(tmp_path):
    good = b"1,2,3,4,5,6\n" * 3
    for bad in (b"", b"1,2,3,4,5,6\n", b"1,2,3,4,5,6", b"1, 2,3,4,5,6\n", b"\n"):
        paths = _write(tmp_path, [good, bad])
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            with pytest.raises(ValueError, match="f001.txt"):
                datasets._read_tables(paths, 6, datasets.DELIM_COMMA)


@pytest.fixture(scope="module")
def trees(tmp_path_factory):
    return D.write_trees(str(tmp_path_factory.mktemp("datasets")))


def test_load_modelnet_equals_the_reference(trees):
    g = np.load(os.path.join(GOLDEN, "dataset_modelnet.npz"))
    for tag, (split, npoints, normalize, normal_channel, m10) in D.MODELNET_CASES.items():
        s, names = datasets.load_modelnet(trees["modelnet"], split, npoints, normalize, normal_channel, m10)
        pts, off = g[f"{tag}_points"], g[f"{tag}_offsets"]
        assert np.array_equal(s.offsets.cpu().numpy(), off), tag
        assert np.array_equal(s.label.cpu().numpy(), g[f"{tag}_label"]), tag
        assert np.array_equal(_bits(s.xyz.cpu().numpy()), _bits(pts[:, :3])), tag
        if normal_channel:
            assert np.array_equal(_bits(s.normals.cpu().numpy()), _bits(pts[:, 3:6])), tag
        else:
            assert s.normals is None
        assert s.num_class == len(names) == (2 if m10 else 4)
        batch = sample_shapes(s, torch.arange(len(s), device=s.device), 3, npoints=256, with_normals=normal_channel)
        assert (batch.lengths.cpu().numpy() == np.minimum(np.diff(off), 256)).all()


def test_load_shapenet_part_equals_the_reference(trees):
    g = np.load(os.path.join(GOLDEN, "dataset_shapenet.npz"))
    for tag, (split, normalize) in D.SHAPENET_CASES.items():
        s, names = datasets.load_shapenet_part(trees["shapenet"], split, normalize)
        assert names == list(g["categories"])
        assert np.array_equal(s.offsets.cpu().numpy(), g[f"{tag}_offsets"]), tag
        assert np.array_equal(s.label.cpu().numpy(), g[f"{tag}_label"]), tag
        assert np.array_equal(_bits(s.xyz.cpu().numpy()), _bits(g[f"{tag}_xyz"])), tag
        assert np.array_equal(_bits(s.normals.cpu().numpy()), _bits(g[f"{tag}_normal"])), tag
        assert np.array_equal(s.part.cpu().numpy(), g[f"{tag}_part"]), tag
        batch = sample_shapes(s, torch.arange(len(s), device=s.device), 4, npoints=512, subset="random",
                              rotate=False, perturb=False, scale=None, shift=0.0, jitter=None, with_normals=True)
        assert batch.part is not None and (batch.lengths.cpu().numpy() >= 1).all()


def test_load_scannet_builds_the_pickled_scenes(trees):
    for split, (seed, k) in (("train", (13, 4)), ("test", (14, 2))):
        ss = datasets.load_scannet(trees["scannet"], split)
        pts, labs = D.scannet_arrays(seed, k)
        assert len(ss) == k and ss.num_class == 21
        assert np.array_equal(ss.xyz.cpu().numpy(), np.concatenate(pts))
        assert np.array_equal(ss.label.cpu().numpy(), np.concatenate(labs))
        # scannet_dataset.py:17-24 over the pickled labels
        hist = sum(np.histogram(seg, range(22))[0] for seg in labs).astype(np.float32)
        want = 1 / np.log(1.2 + hist / np.sum(hist))
        assert np.array_equal(ss.train_label_weights().cpu().numpy(), want.astype(np.float32))
        crops = sample_crops(ss, torch.arange(k, device=ss.device), 9, ss.train_label_weights(), npoints=1024)
        assert (crops.lengths.cpu().numpy() >= 1).all()
