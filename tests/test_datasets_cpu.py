"""CPU tests of the dataset loaders (pointnet2_b200.datasets, DESIGN.md §6.18): the device grammar's exact
conversion restated and checked against Python's correctly rounded float(), the reference's file-list logic against
the recorded goldens, the ScanNet unpickler, and the text parser's argument checks."""
import ctypes
import os
import pickle
import sys

import numpy as np
import pytest

from oracle import dataset_ref as D
from pointnet2_b200 import _lib, datasets, nets

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import text_oracle as T  # noqa: E402

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _expect(s):
    return np.float32(float(s))


def _same(a, b):
    return np.asarray(a, np.float32).view(np.uint32) == np.asarray(b, np.float32).view(np.uint32)


def test_exact_conversion_matches_float_then_float32():
    rng = np.random.default_rng(2024)
    strings = []
    for _ in range(100_000):
        nd = int(rng.integers(1, 18))
        digits = "".join(str(d) for d in rng.integers(0, 10, nd))
        point = int(rng.integers(0, nd + 1))
        s = digits[:point] + ("." + digits[point:] if point < nd else "")
        if s.startswith("."):
            s = s if rng.random() < 0.5 else "0" + s
        if rng.random() < 0.4:
            s += "eE"[int(rng.integers(0, 2))] + ["", "+", "-"][int(rng.integers(0, 3))] + str(int(rng.integers(0, 30)))
        strings.append(("-" if rng.random() < 0.3 else "") + s)
    # float32 ties and their neighbours: odd integers in [2^24, 2^31) sit halfway between two float32 values
    for k in rng.integers(1 << 23, 1 << 30, 3000):
        t = 2 * int(k) + 1
        strings += [str(t), f"{t}.000001", f"{t - 1}.999999", f"{t}e0", f"{t}0e-1"]
    # the edges of the exact path: M at 2^53 +- 1, E at +-22 and +-23
    m53 = 2 ** 53
    for m in (m53 - 1, m53, m53 + 1):
        for e in (-23, -22, -1, 0, 1, 22, 23):
            strings.append(f"{m}e{e}")
    strings += ["1e22", "1e23", "1e-22", "1e-23", "0e23", "0.0000000000000000000001", "-0.000000", "-0", "+.5"]
    converted = 0
    for s in strings:
        v = T.convert(s)
        if v is None:
            continue
        converted += 1
        assert _same(v, _expect(s)), (s, v, _expect(s))
    assert converted >= 100_000
    # the rule's own edges
    assert T.convert(f"{m53}e22") is not None and T.convert(f"{m53 + 1}") is None
    assert T.convert("1e-23") is None and T.convert("1e23") is None
    assert np.signbit(T.convert("-0.000000"))


@pytest.mark.parametrize("line,delim,ncol,want", [
    ("1.5,-2,3e-2", T.COMMA, 3, T.OK),
    (".5,+0.25,-.125", T.COMMA, 3, T.OK),
    ("  1\t2   3 \t", T.WHITESPACE, 3, T.OK),
    ("1, 2,3", T.COMMA, 3, T.SYNTAX),
    ("1.,2,3", T.COMMA, 3, T.SYNTAX),
    ("nan,2,3", T.COMMA, 3, T.SYNTAX),
    ("inf 2 3", T.WHITESPACE, 3, T.SYNTAX),
    ("1_0,2,3", T.COMMA, 3, T.SYNTAX),
    ("1,,3", T.COMMA, 3, T.SYNTAX),
    ("1e,2,3", T.COMMA, 3, T.SYNTAX),
    ("1,2", T.COMMA, 3, T.FIELDS),
    ("1,2,3,4", T.COMMA, 3, T.FIELDS),
    ("1,2,3,", T.COMMA, 3, T.FIELDS),
    ("", T.COMMA, 3, T.BLANK),
    (" \t ", T.WHITESPACE, 3, T.BLANK),
    ("1,2\r,3", T.COMMA, 3, T.CR),
    ("# 1 2 3", T.WHITESPACE, 3, T.COMMENT),
    ("1 2 # c", T.WHITESPACE, 3, T.COMMENT),
    ("0.12345678901234567,2,3", T.COMMA, 3, T.INEXACT),
    ("1.5e-30 2 3", T.WHITESPACE, 3, T.INEXACT),
])
def test_grammar_classifies_lines(line, delim, ncol, want):
    assert T.parse_line(line, ncol, delim)[0] == want


def test_file_verdicts_terminators():
    assert T.classify_file(b"1,2\r\n3,4\r\n", 2, T.COMMA)[0] == T.OK
    assert T.classify_file(b"1,2\n3,4", 2, T.COMMA)[1].shape == (2, 2)
    assert T.classify_file(b"1,2\n3,4\r", 2, T.COMMA)[0] == T.CR  # a last "\r" is not a "\r\n"
    assert T.classify_file(b"1,2\r3,4\n", 2, T.COMMA)[0] == T.CR
    assert T.classify_file(b"1,2\n\n3,4\n", 2, T.COMMA)[0] == T.BLANK
    assert T.classify_file(b"", 2, T.COMMA)[1].shape == (0, 2)


@pytest.fixture(scope="module")
def trees(tmp_path_factory):
    return D.write_trees(str(tmp_path_factory.mktemp("datasets")))


def test_modelnet_file_lists_match_the_reference(trees):
    g = np.load(os.path.join(GOLDEN, "dataset_modelnet.npz"))
    for tag, (split, _, _, _, m10) in D.MODELNET_CASES.items():
        paths, labels, names = datasets.modelnet_files(trees["modelnet"], split, m10)
        assert [os.path.relpath(p, trees["modelnet"]) for p in paths] == list(g[f"{tag}_files"])
        assert labels == list(g[f"{tag}_label"])
        assert len(names) == (2 if m10 else 4)
    with pytest.raises(ValueError, match="split"):
        datasets.modelnet_files(trees["modelnet"], "val")


def test_shapenet_file_lists_match_the_reference(trees):
    g = np.load(os.path.join(GOLDEN, "dataset_shapenet.npz"))
    for tag, (split, _) in D.SHAPENET_CASES.items():
        paths, labels, names = datasets.shapenet_part_files(trees["shapenet"], split)
        assert [os.path.relpath(p, trees["shapenet"]) for p in paths] == list(g[f"{tag}_files"])
        assert labels == list(g[f"{tag}_label"])
        assert names == list(g["categories"])
    with pytest.raises(ValueError, match="split"):
        datasets.shapenet_part_files(trees["shapenet"], "all")


def test_part_categories_are_in_the_order_part_offsets_assume():
    names = [n for n, _ in D.PART_CATEGORIES]
    assert names == sorted(names) and len(names) == nets.NUM_CATEGORIES == len(nets.PART_OFFSETS) - 1
    # each category's part range in the reference's seg_classes (part_dataset_all_normal.py:75)
    first = {"Airplane": 0, "Bag": 4, "Cap": 6, "Car": 8, "Chair": 12, "Earphone": 16, "Guitar": 19, "Knife": 22,
             "Lamp": 24, "Laptop": 28, "Motorbike": 30, "Mug": 36, "Pistol": 38, "Rocket": 41, "Skateboard": 44,
             "Table": 47}
    assert [first[n] for n in names] == list(nets.PART_OFFSETS[:-1])


def test_py2_pickle_loads_to_the_arrays(tmp_path):
    pts, labs = D.scannet_arrays(5, 3)
    raw = D.py2_pickle_list(pts) + D.py2_pickle_list(labs)
    assert b"T" in raw or b"U" in raw  # array bytes as (SHORT_)BINSTRING, as Python 2 wrote them
    p = tmp_path / "scannet_train.pickle"
    p.write_bytes(raw)
    got_p, got_l = datasets.read_scannet_pickle(str(p))
    assert len(got_p) == len(got_l) == 3
    for a, b in zip(got_p + got_l, pts + labs):
        assert a.dtype == b.dtype and a.shape == b.shape and np.array_equal(a, b)


_CALLED = []


def _trap(*args):
    _CALLED.append(args)
    return 0


def test_unpickler_refuses_other_globals_without_calling_them(tmp_path):
    evil = b"\x80\x02" + D._p2_global(__name__, "_trap") + D._p2_str(b"x") + b"\x85R."
    p = tmp_path / "scannet_train.pickle"
    p.write_bytes(evil)
    with pytest.raises(pickle.UnpicklingError, match="refusing"):
        datasets.read_scannet_pickle(str(p))
    assert not _CALLED
    assert pickle.loads(evil) == 0 and _CALLED  # the same bytes do call it through the unrestricted unpickler
    p.write_bytes(b"\x80\x02" + D._p2_global("os", "system") + D._p2_str(b"true") + b"\x85R.")
    with pytest.raises(pickle.UnpicklingError, match="os.system"):
        datasets.read_scannet_pickle(str(p))


def test_text_entries_refuse_bad_arguments_without_a_launch():
    lib = _lib.load()
    P = ctypes.c_void_p(256)  # never dereferenced: every call below is refused before a launch
    before = _lib.launch_count()
    bad_scan = [(0, P, P, 10, 6, 1, P, P), (1, None, P, 10, 6, 1, P, P), (1, P, None, 10, 6, 1, P, P),
                (1, P, P, -1, 6, 1, P, P), (1, P, P, 10, 0, 1, P, P), (1, P, P, 10, 65, 1, P, P),
                (1, P, P, 10, 6, 2, P, P), (1, P, P, 10, 6, 1, None, P), (1, P, P, 10, 6, 1, P, None)]
    for args in bad_scan:
        assert lib.pn2_text_rows_scan(*args, None) == 1, args
    bad_parse = [(0, P, P, 10, 6, 1, P, 5, P, P, 5), (1, P, P, 10, 6, -1, P, 5, P, P, 5),
                 (1, P, P, 10, 6, 1, None, 5, P, P, 5), (1, P, P, 10, 6, 1, P, -1, P, P, 5),
                 (1, P, P, 10, 6, 1, P, 5, None, P, 5), (1, P, P, 10, 6, 1, P, 5, P, None, 5),
                 (1, P, P, 10, 6, 1, P, 5, P, P, -1), (1, P, P, 10, 65, 1, P, 5, P, P, 5)]
    for args in bad_parse:
        assert lib.pn2_text_rows_parse(*args, None) == 1, args
    assert _lib.launch_count() == before
