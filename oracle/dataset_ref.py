"""The dataset loaders' checker (TEST INFRASTRUCTURE ONLY, like the rest of oracle/): seeded fixture trees in the
reference's three dataset layouts, and the recorder of what the reference's own readers make of them.

* ``write_modelnet_tree`` — modelnet40_normal_resampled/: shape_names.txt, modelnet10_shape_names.txt, the four
  modelnet{40,10}_{train,test}.txt lists and class/id.txt files of 6 comma-separated columns.
* ``write_shapenet_tree`` — shapenetcore_partanno_segmentation_benchmark_v0_normal/: synsetoffset2category.txt (the
  benchmark's 16 categories), the three train_test_split/shuffled_*_file_list.json lists and synset/token.txt files
  of 7 blank-separated columns (xyz, normal, part).
* ``write_scannet_tree`` — scannet_{train,test}.pickle as Python 2 wrote them: protocol 2, array bytes as BINSTRING.

The text trees hold files with "\\r\\n" endings, without a final newline, with fewer and more rows than the
recorded npoints, and one file for each reason the device parser leaves a file to np.loadtxt.

    python oracle/dataset_ref.py DIR    # record DIR/dataset_*.npz from the reference's readers (CPU only)
    cp DIR/dataset_*.npz tests/golden/  # then commit

Only tests/ and tools/ may import this module.
"""
from __future__ import annotations

import contextlib
import importlib.util
import io
import json
import os
import struct
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))

# (split, npoints, normalize, normal_channel, modelnet10) of each recorded ModelNet load
MODELNET_CASES = {
    "m40_train_1024": ("train", 1024, True, False, False),
    "m40_test_64_raw_normals": ("test", 64, False, True, False),
    "m40_train_5000": ("train", 5000, True, False, False),
    "m10_test_512_normals": ("test", 512, True, True, True),
    "m10_train_300_raw": ("train", 300, False, False, True),
}
# (split, normalize) of each recorded ShapeNet-part load
SHAPENET_CASES = {
    "trainval": ("trainval", True),
    "train": ("train", True),
    "val": ("val", True),
    "test": ("test", True),
    "test_raw": ("test", False),
}
PART_CATEGORIES = [("Airplane", "02691156"), ("Bag", "02773838"), ("Cap", "02954340"), ("Car", "02958343"),
                   ("Chair", "03001627"), ("Earphone", "03261776"), ("Guitar", "03467517"), ("Knife", "03624134"),
                   ("Lamp", "03636649"), ("Laptop", "03642806"), ("Motorbike", "03790512"), ("Mug", "03797390"),
                   ("Pistol", "03948459"), ("Rocket", "04004475"), ("Skateboard", "04225987"), ("Table", "04379243")]
# a line of each kind the device grammar refuses but np.loadtxt reads (pn2_api.h PN2_TEXT_*), by reason
FALLBACK_KINDS = ("syntax", "fields", "blank", "cr", "comment", "inexact")


def _rows_text(a: np.ndarray, sep: str, fmt: str = "%.6f") -> list:
    return [sep.join(fmt % v for v in row) for row in a]


def _fallback_lines(lines: list, kind: str, sep: str) -> tuple:
    """lines with one change np.loadtxt reads the same way but the device grammar does not; (lines, eol)."""
    lines = list(lines)
    if kind == "syntax":  # a field "1." and, in comma files, a blank after a separator
        first, rest = lines[3].split(sep, 1)
        lines[3] = first.split(".")[0] + "." + sep + rest
        if sep == ",":
            lines[2] = lines[2].replace(",", ", ", 1)
    elif kind == "fields":  # one more column in every line (a ModelNet file of it sits in train lists only)
        lines = [ln + sep + "0.500000" for ln in lines]
    elif kind == "blank":
        lines.insert(len(lines) // 2, "")
    elif kind == "comment":
        lines.insert(1, "# a comment line")
    elif kind == "inexact":  # 17 significant digits; an exponent beyond 22
        a = lines[2].split(sep)
        a[0] = "0.12345678901234567"
        a[1] = "1.5e-30"
        lines[2] = sep.join(a)
    if kind == "cr":
        return lines, "\r"
    return lines, "\n"


def _write_text(path: str, lines: list, eol: str = "\n", final_eol: bool = True) -> None:
    os.makedirs(os.path.dirname(path), exist_ok=True)
    with open(path, "wb") as f:
        f.write((eol.join(lines) + (eol if final_eol else "")).encode())


def _odd_values(rng, a: np.ndarray) -> list:
    """Values in every form of the grammar, replacing some of a's formatted ones: signs, -0, .5, exponents."""
    forms = ["-0.000000", "+0.250000", ".500000", "-.125000", "1.5e-3", "2E+2", "-3e0", "0.000001", "12345678",
             "0.1", "7", "-0.999999"]
    idx = rng.choice(a.size, size=min(len(forms), a.size), replace=False)
    out = [["%.6f" % v for v in row] for row in a]
    for k, i in enumerate(idx):
        out[i // a.shape[1]][i % a.shape[1]] = forms[k]
    return out


def write_modelnet_tree(root: str, seed: int = 7) -> None:
    rng = np.random.default_rng(seed)
    classes = ["airplane", "night_stand", "chair", "flower_pot"]
    m10 = ["night_stand", "chair"]
    os.makedirs(root, exist_ok=True)
    _write_text(os.path.join(root, "shape_names.txt"), classes)
    _write_text(os.path.join(root, "modelnet10_shape_names.txt"), m10)
    lists = {("modelnet40", "train"): [], ("modelnet40", "test"): [], ("modelnet10", "train"): [],
             ("modelnet10", "test"): []}
    kinds = list(FALLBACK_KINDS) + ["crlf", "no_final_eol", "odd_values"] + ["plain"] * 9
    for k, kind in enumerate(kinds):
        cls = classes[k % len(classes)]
        sid = f"{cls}_{k + 1:04d}"
        n = int(rng.choice([40, 300, 700, 1100, 2600]))
        a = rng.uniform(-1.5, 1.5, (n, 6))
        a[:, 3:] = a[:, 3:] / np.linalg.norm(a[:, 3:], axis=1, keepdims=True)
        lines = _rows_text(a, ",")
        eol, final = "\n", True
        if kind in FALLBACK_KINDS:
            lines, eol = _fallback_lines(lines, kind, ",")
        elif kind == "crlf":
            eol = "\r\n"
        elif kind == "no_final_eol":
            final = False
        elif kind == "odd_values":
            lines = [",".join(r) for r in _odd_values(rng, a)]
        _write_text(os.path.join(root, cls, sid + ".txt"), lines, eol, final)
        split = "test" if k % 3 == 2 else "train"
        lists[("modelnet40", split)].append(sid)
        if cls in m10:
            lists[("modelnet10", split)].append(sid)
    for (tag, split), ids in lists.items():
        _write_text(os.path.join(root, f"{tag}_{split}.txt"), ids)


def write_shapenet_tree(root: str, seed: int = 11) -> None:
    rng = np.random.default_rng(seed)
    os.makedirs(os.path.join(root, "train_test_split"), exist_ok=True)
    _write_text(os.path.join(root, "synsetoffset2category.txt"), [f"{n}\t{s}" for n, s in PART_CATEGORIES])
    for _, syn in PART_CATEGORIES:
        os.makedirs(os.path.join(root, syn), exist_ok=True)
    used = [PART_CATEGORIES[i] for i in (0, 4, 8, 15)]  # Airplane, Chair, Lamp, Table
    offsets = dict(zip([n for n, _ in PART_CATEGORIES], (0, 4, 6, 8, 12, 16, 19, 22, 24, 28, 30, 36, 38, 41, 44, 47)))
    splits = {"train": [], "val": [], "test": []}
    kinds = list(FALLBACK_KINDS) + ["crlf", "no_final_eol", "odd_values", "unlisted"] + ["plain"] * 10
    for k, kind in enumerate(kinds):
        name, syn = used[k % len(used)]
        token = "%032x" % int(rng.integers(0, 1 << 62))
        n = int(rng.choice([30, 200, 900, 2800]))
        a = np.empty((n, 7))
        a[:, :3] = rng.uniform(-0.8, 0.8, (n, 3))
        a[:, 3:6] = rng.normal(size=(n, 3))
        a[:, 3:6] /= np.linalg.norm(a[:, 3:6], axis=1, keepdims=True)
        a[:, 6] = offsets[name] + rng.integers(0, 3, n)
        lines = [" ".join(r) for r in (_odd_values(rng, a[:, :6]) if kind == "odd_values" else
                                       [["%.6f" % v for v in row[:6]] for row in a])]
        lines = [ln + " %.6f" % p for ln, p in zip(lines, a[:, 6])]
        eol, final = "\n", True
        if kind in FALLBACK_KINDS:
            lines, eol = _fallback_lines(lines, kind, " ")
        elif kind == "crlf":
            eol = "\r\n"
        elif kind == "no_final_eol":
            final = False
        if k % 5 == 3:  # leading and trailing blanks, tabs between fields
            lines = ["  " + ln.replace(" ", "\t", 2) + " \t" if ln else ln for ln in lines]
        _write_text(os.path.join(root, syn, token + ".txt"), lines, eol, final)
        if kind != "unlisted":
            splits[("train", "train", "val", "test")[k % 4]].append(f"shape_data/{syn}/{token}")
    for s, lst in splits.items():
        with open(os.path.join(root, "train_test_split", f"shuffled_{s}_file_list.json"), "w") as f:
            json.dump(lst, f)


# ---- Python 2 pickles: protocol 2 as cPickle wrote numpy arrays, the array bytes as a BINSTRING ----------------------
def _p2_str(s: bytes) -> bytes:
    return (b"U" + bytes([len(s)]) + s) if len(s) < 256 else (b"T" + struct.pack("<i", len(s)) + s)


def _p2_int(v: int) -> bytes:
    return b"K" + bytes([v]) if 0 <= v < 256 else b"J" + struct.pack("<i", v)


def _p2_global(module: str, name: str) -> bytes:
    return b"c" + module.encode() + b"\n" + name.encode() + b"\n"


def py2_array_ops(a: np.ndarray) -> bytes:
    """The opcodes numpy 1.x under Python 2 emits for ndarray.__reduce__: _reconstruct(ndarray, (0,), 'b') then
    BUILD with (1, shape, dtype, is_fortran, raw bytes)."""
    a = np.ascontiguousarray(a)
    order = "|" if a.dtype.itemsize == 1 else "<"
    dt = (_p2_global("numpy", "dtype") + _p2_str(a.dtype.str[1:].encode()) + _p2_int(0) + _p2_int(1) + b"\x87R"
          + b"(" + _p2_int(3) + _p2_str(order.encode()) + b"NNN" + b"J\xff\xff\xff\xffJ\xff\xff\xff\xff" + _p2_int(0)
          + b"tb")
    shape = b"(" + b"".join(_p2_int(d) for d in a.shape) + b"t"
    return (_p2_global("numpy.core.multiarray", "_reconstruct") + _p2_global("numpy", "ndarray") + _p2_int(0)
            + b"\x85" + _p2_str(b"b") + b"\x87R" + b"(" + _p2_int(1) + shape + dt + b"\x89"
            + _p2_str(a.astype(a.dtype.newbyteorder("<")).tobytes()) + b"tb")


def py2_pickle_list(arrays) -> bytes:
    """One protocol-2 pickle of a list of arrays, as Python 2's cPickle.dump(lst, fp, 2) lays it out."""
    return b"\x80\x02]" + b"(" + b"".join(py2_array_ops(a) for a in arrays) + b"e."


def scannet_arrays(seed: int, scenes: int):
    rng = np.random.default_rng(seed)
    pts, labs = [], []
    for _ in range(scenes):
        n = int(rng.integers(3000, 6000))
        size = rng.uniform(2.0, 5.0, 3)
        pts.append((rng.uniform(0.0, 1.0, (n, 3)) * size).astype(np.float32))
        labs.append(rng.integers(0, 21, n).astype(np.int32))
    return pts, labs


def write_scannet_tree(root: str, seed: int = 13) -> None:
    os.makedirs(root, exist_ok=True)
    for split, (s, k) in {"train": (seed, 4), "test": (seed + 1, 2)}.items():
        pts, labs = scannet_arrays(s, k)
        with open(os.path.join(root, f"scannet_{split}.pickle"), "wb") as f:
            f.write(py2_pickle_list(pts) + py2_pickle_list(labs))


def write_trees(root: str) -> dict:
    dirs = {"modelnet": os.path.join(root, "modelnet40_normal_resampled"),
            "shapenet": os.path.join(root, "shapenetcore_partanno_segmentation_benchmark_v0_normal"),
            "scannet": os.path.join(root, "scannet")}
    write_modelnet_tree(dirs["modelnet"])
    write_shapenet_tree(dirs["shapenet"])
    write_scannet_tree(dirs["scannet"])
    return dirs


# ---- the recorder: the reference's own readers, CPU only ------------------------------------------------------------
def _ref_root() -> str:
    spec = importlib.util.spec_from_file_location("pn2_oracle_build", os.path.join(HERE, "build.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod.REF_ROOT


def _ref_modelnet(ref: str):
    sys.modules.setdefault("h5py", types.ModuleType("h5py"))  # utils/provider.py imports it; the text reader never uses it
    sys.path[:0] = [ref, os.path.join(ref, "utils")]
    spec = importlib.util.spec_from_file_location("ref_modelnet_dataset", os.path.join(ref, "modelnet_dataset.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod.ModelNetDataset


def _ref_part(ref: str):
    src = open(os.path.join(ref, "part_seg", "part_dataset_all_normal.py")).read()
    src = src[:src.index("if __name__ == '__main__':")]  # the rest is Python 2
    ns = {"__name__": "ref_part_dataset_all_normal"}
    exec(compile(src, "part_dataset_all_normal.py", "exec"), ns)
    return ns["PartNormalDataset"]


def _packed(arrays):
    off = np.zeros(len(arrays) + 1, np.int64)
    np.cumsum([len(a) for a in arrays], out=off[1:])
    return np.concatenate(arrays), off


def record(outdir: str) -> None:
    """Write outdir/dataset_modelnet.npz and dataset_shapenet.npz: per case the files in the reader's order (relative
    to the tree), their labels and the exact rows the reader caches."""
    import tempfile
    ref = _ref_root()
    os.makedirs(outdir, exist_ok=True)
    with tempfile.TemporaryDirectory() as tmp:
        dirs = write_trees(tmp)
        ModelNetDataset, PartNormalDataset = _ref_modelnet(ref), _ref_part(ref)
        arrs = {}
        for tag, (split, npoints, normalize, normal_channel, m10) in MODELNET_CASES.items():
            d = ModelNetDataset(dirs["modelnet"], npoints=npoints, split=split, normalize=normalize,
                                normal_channel=normal_channel, modelnet10=m10)
            items = [d._get_item(i) for i in range(len(d))]
            arrs[f"{tag}_files"] = np.array([os.path.relpath(p, dirs["modelnet"]) for _, p in d.datapath])
            arrs[f"{tag}_label"] = np.array([int(c[0]) for _, c in items], np.int32)
            arrs[f"{tag}_points"], arrs[f"{tag}_offsets"] = _packed([p for p, _ in items])
        np.savez_compressed(os.path.join(outdir, "dataset_modelnet.npz"), **arrs)
        arrs = {}
        for tag, (split, normalize) in SHAPENET_CASES.items():
            with contextlib.redirect_stdout(io.StringIO()):
                d = PartNormalDataset(dirs["shapenet"], split=split, normalize=normalize)
                for i in range(len(d)):
                    d[i]
            items = [d.cache[i] for i in range(len(d))]
            arrs[f"{tag}_files"] = np.array([os.path.relpath(p, dirs["shapenet"]) for _, p in d.datapath])
            arrs[f"{tag}_label"] = np.array([int(c[0]) for _, _, _, c in items], np.int32)
            arrs[f"{tag}_xyz"], arrs[f"{tag}_offsets"] = _packed([p for p, _, _, _ in items])
            arrs[f"{tag}_normal"] = np.concatenate([n for _, n, _, _ in items])
            arrs[f"{tag}_part"] = np.concatenate([s for _, _, s, _ in items])
        arrs["categories"] = np.array(list(d.cat))
        np.savez_compressed(os.path.join(outdir, "dataset_shapenet.npz"), **arrs)
    print("wrote", os.path.join(outdir, "dataset_modelnet.npz"), os.path.join(outdir, "dataset_shapenet.npz"))


if __name__ == "__main__":
    if len(sys.argv) != 2:
        sys.exit("usage: python oracle/dataset_ref.py OUTDIR")
    record(sys.argv[1])
