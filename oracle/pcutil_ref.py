"""The voxel and pillar grouping's checker (TEST INFRASTRUCTURE ONLY, like the rest of oracle/): the recorder of what the
reference's own utils/pc_util.py makes of seeded inputs, and the loader tools/pc_util_bench.py times it through.

pc_util imports eulerangles and plyfile, which the conversions never use: both are stubbed.  It calls np.lib.pad,
which numpy 2 no longer has: np.pad is put there before the calls.  Only cells of at most num_sample points are
recorded, where the reference draws nothing at random.

    python oracle/pcutil_ref.py DIR     # record DIR/pcutil_*.npz from the reference's functions (CPU only)
    cp DIR/pcutil_*.npz tests/golden/   # then commit

``build_pcutil_ref()`` (run by build()) byte-compiles the reference's pc_util.py into oracle/_ref/, which stays out
of git, so that the timing tool can load it where the reference checkout is absent.  Only tests/ and tools/ may
import this module.
"""
from __future__ import annotations

import importlib.machinery
import importlib.util
import os
import py_compile
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
PYC = os.path.join(HERE, "_ref", "pc_util.pyc")


def _ref_root() -> str:
    spec = importlib.util.spec_from_file_location("pn2_oracle_build", os.path.join(HERE, "build.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod.REF_ROOT


def build_pcutil_ref() -> str | None:
    """Byte-compile the reference's utils/pc_util.py into oracle/_ref/pc_util.pyc (when the checkout is present)."""
    src = os.path.join(_ref_root(), "utils", "pc_util.py")
    if not os.path.exists(src):
        return PYC if os.path.exists(PYC) else None
    if not os.path.exists(PYC) or os.path.getmtime(PYC) < os.path.getmtime(src):
        os.makedirs(os.path.dirname(PYC), exist_ok=True)
        py_compile.compile(src, cfile=PYC, doraise=True)
    return PYC


def load_pc_util():
    """The reference's pc_util module, from the checkout or from oracle/_ref/pc_util.pyc; None when neither exists."""
    for name, attrs in (("eulerangles", ("euler2mat",)), ("plyfile", ("PlyData", "PlyElement"))):
        if name not in sys.modules:
            stub = types.ModuleType(name)
            for a in attrs:
                setattr(stub, a, None)
            sys.modules[name] = stub
    if not hasattr(np.lib, "pad"):
        np.lib.pad = np.pad
    src = os.path.join(_ref_root(), "utils", "pc_util.py")
    if os.path.exists(src):
        spec = importlib.util.spec_from_file_location("ref_pc_util", src)
    elif os.path.exists(PYC):
        spec = importlib.util.spec_from_loader("ref_pc_util", importlib.machinery.SourcelessFileLoader("ref_pc_util", PYC))
    else:
        return None
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


# ---- inputs -------------------------------------------------------------------------------------------------------
def edge_values(vsize: int, radius: float, ulps: int = 2) -> np.ndarray:
    """float32 coordinates on and around every cell edge: the float32 nearest k * voxel - radius and ``ulps`` float32
    steps either side, for k = 0 .. vsize (k = 0: quotients in (-1, 0) below it; k = vsize: the grid's far face)."""
    r32, v32 = np.float32(radius), np.float32(2 * radius / float(vsize))
    out = []
    for k in range(vsize + 1):
        x = np.float32(np.float32(k) * v32 - r32)
        lo = hi = x
        out.append(x)
        for _ in range(ulps):
            lo, hi = np.nextafter(lo, np.float32(-np.inf)), np.nextafter(hi, np.float32(np.inf))
            out += [lo, hi]
    return np.array(out, np.float32)


def case_inputs(vsize: int, radius: float, n: int, seed: int) -> np.ndarray:
    """(2, n, 3) float32: cloud 0 from the edge values (every axis), cloud 1 uniform in the grid with a quarter of its
    rows duplicated and some quotients in (-1, 0); in both an eighth of the rows have a coordinate beyond the grid or
    NaN."""
    rs = np.random.RandomState(seed)
    e = edge_values(vsize, radius)
    voxel = 2 * radius / vsize
    c0 = rs.choice(e, (n, 3)).astype(np.float32)
    c1 = rs.uniform(-radius, radius, (n, 3)).astype(np.float32)
    c1[: n // 4] = c1[n // 4: n // 2]                                          # duplicates
    c1[n // 2: n // 2 + n // 8, 0] = rs.uniform(-radius - 0.999 * voxel, -radius, n // 8)  # quotient in (-1, 0)
    for c in (c0, c1):
        k = rs.choice(n, n // 8, replace=False)
        c[k, rs.randint(0, 3, len(k))] = rs.choice([-2 * radius, -radius - 1.01 * voxel, radius, 3 * radius, np.nan], len(k))
    return np.stack([c0, c1]).astype(np.float32)


# (vsize, radius, n, num_sample, seed) per recorded case; num_sample covers every cell's count
VOLUME_CASES = {"v12_r1": (12, 1.0, 300, 16, 1), "v7_r0.7": (7, 0.7, 300, 16, 2), "v1_r1": (1, 1.0, 40, 48, 3)}
IMAGE_CASES = {"i8_r1": (8, 1.0, 300, 32, 4), "i13_r0.7": (13, 0.7, 300, 16, 5), "i1_r1": (1, 1.0, 40, 48, 6)}


def _in_grid(pts, vsize, radius, dims):
    q = (pts[:, :dims] + np.float32(radius)) / np.float32(2 * radius / float(vsize))
    with np.errstate(invalid="ignore"):
        return q, np.all((q > -1) & (q < vsize), axis=1)


def _max_count(xyz, vsize, radius, dims):
    best = 0
    for pts in xyz:
        q, ok = _in_grid(pts, vsize, radius, dims)
        _, c = np.unique(q[ok].astype(np.int64), axis=0, return_counts=True)
        best = max(best, int(c.max()) if len(c) else 0)
    return best


def _inside(xyz, vsize, radius):
    """xyz with every point outside the grid moved to the origin: point_cloud_to_volume raises or wraps on those."""
    out = xyz.copy()
    for pts in out:
        pts[~_in_grid(pts, vsize, radius, 3)[1]] = 0
    return out


def record(outdir: str) -> None:
    """Write outdir/pcutil_volume.npz and outdir/pcutil_image.npz: per case the inputs, the parameters and the
    reference's point_cloud_to_volume_batch (in-grid points only), point_cloud_to_volume_v2_batch and
    point_cloud_to_image_batch outputs."""
    pc = load_pc_util()
    if pc is None:
        raise SystemExit("the reference's utils/pc_util.py is not available")
    os.makedirs(outdir, exist_ok=True)
    arrs = {}
    with np.errstate(invalid="ignore"):
        for tag, (vsize, radius, n, s, seed) in VOLUME_CASES.items():
            xyz = case_inputs(vsize, radius, n, seed)
            assert _max_count(xyz, vsize, radius, 3) <= s, tag
            inside = _inside(xyz, vsize, radius)
            arrs[f"{tag}_params"] = np.array([vsize, radius, s], np.float64)
            arrs[f"{tag}_xyz"] = xyz
            arrs[f"{tag}_v2"] = pc.point_cloud_to_volume_v2_batch(xyz, vsize, radius, s)
            arrs[f"{tag}_inside"] = inside
            arrs[f"{tag}_vol"] = pc.point_cloud_to_volume_batch(inside, vsize, radius, True)
        np.savez_compressed(os.path.join(outdir, "pcutil_volume.npz"), **arrs)
        arrs = {}
        for tag, (isize, radius, n, s, seed) in IMAGE_CASES.items():
            xyz = case_inputs(isize, radius, n, seed)
            assert _max_count(xyz, isize, radius, 2) <= s, tag
            arrs[f"{tag}_params"] = np.array([isize, radius, s], np.float64)
            arrs[f"{tag}_xyz"] = xyz
            arrs[f"{tag}_img"] = pc.point_cloud_to_image_batch(xyz, isize, radius, s)
        np.savez_compressed(os.path.join(outdir, "pcutil_image.npz"), **arrs)
    print("wrote", os.path.join(outdir, "pcutil_volume.npz"), os.path.join(outdir, "pcutil_image.npz"))


if __name__ == "__main__":
    if len(sys.argv) != 2:
        sys.exit("usage: python oracle/pcutil_ref.py OUTDIR")
    record(sys.argv[1])
