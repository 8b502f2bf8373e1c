"""The point viewer's checker (TEST INFRASTRUCTURE ONLY, like the rest of oracle/): its build recipe, its ctypes
front-end and the recorder of its fixtures.

* ``oracle/librender_oracle.so``  <- oracle/render_oracle.c, the C restatement ``oracle_render_ball`` (always built).
* ``oracle/_ref/libref_render.so`` <- utils/render_balls_so.cpp of the reference checkout that oracle/build.py uses,
  unmodified, with the reference's own flags (utils/compile_render_balls_so.sh: g++ -std=c++11 -O2 -shared -fPIC
  -D_GLIBCXX_USE_CXX11_ABI=0).  Without a checkout, a library an earlier build left in oracle/_ref/ is used.

    python oracle/render_ref.py DIR    # record DIR/render_*.npz from the reference's render_ball (CPU only)
    cp DIR/render_*.npz tests/golden/  # then commit

Only tests/ and tools/render_bench.py may import this module.
"""
from __future__ import annotations

import ctypes
import importlib.util
import os
import subprocess
import sys
from ctypes import c_int, c_void_p

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ORACLE_SRC = os.path.join(HERE, "render_oracle.c")
ORACLE_LIB = os.path.join(HERE, "librender_oracle.so")


def _oracle_build():
    spec = importlib.util.spec_from_file_location("pn2_oracle_build", os.path.join(HERE, "build.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _newer(target: str, *sources: str) -> bool:
    return os.path.exists(target) and all(os.path.getmtime(s) <= os.path.getmtime(target) for s in sources)


def build_render_oracle(force: bool = False) -> str:
    if force or not _newer(ORACLE_LIB, ORACLE_SRC, __file__):
        tmp = ORACLE_LIB + f".tmp{os.getpid()}"
        subprocess.run(["gcc", "-O2", "-std=c11", "-fPIC", "-shared", "-ffp-contract=off", "-fno-fast-math", "-o", tmp,
                        ORACLE_SRC, "-lm"], check=True)
        os.replace(tmp, ORACLE_LIB)
    return ORACLE_LIB


def ref_render_path() -> str:
    return os.path.join(_oracle_build().REF_OUT, "libref_render.so")


def build_render_ref(force: bool = False) -> str | None:
    """Compile the reference's render_balls_so.cpp into oracle/_ref/.  Returns its path, or None where there is neither
    a reference checkout nor an earlier build."""
    ob = _oracle_build()
    out = ref_render_path()
    src = os.path.join(ob.REF_ROOT, "utils", "render_balls_so.cpp")
    if not os.path.exists(src):
        return out if os.path.exists(out) else None
    os.makedirs(ob.REF_OUT, exist_ok=True)
    if force or not _newer(out, src, __file__):
        subprocess.run(["g++", "-std=c++11", "-O2", "-shared", "-fPIC", "-D_GLIBCXX_USE_CXX11_ABI=0", "-o", out, src],
                       check=True)
    return out


_lib = None
_ref = None


def _args(ixyz, colors, height, width, background):
    ixyz = np.ascontiguousarray(ixyz, np.int32).reshape(-1, 3)
    n = ixyz.shape[0]
    colors = np.full((n, 3), 255, np.float32) if colors is None else np.asarray(colors, np.float32).reshape(n, 3)
    chans = [np.ascontiguousarray(colors[:, k]) for k in range(3)]
    show = np.empty((height, width, 3), np.uint8)
    show[:] = np.asarray(background, np.uint8)
    return ixyz, chans, show


def _call(fn, ixyz, colors, height, width, radius, background):
    ixyz, chans, show = _args(ixyz, colors, height, width, background)
    p = [a.ctypes.data_as(c_void_p) for a in (show, ixyz, *chans)]
    fn(c_int(height), c_int(width), p[0], c_int(ixyz.shape[0]), p[1], p[2], p[3], p[4], c_int(radius))
    return show


def oracle_render_ball(ixyz, colors, height: int, width: int, radius: int, background=(0, 0, 0)):
    """render_ball (utils/render_balls_so.cpp) restated: cloud ixyz (n, 3) int32, colors (n, 3) float32 = c0, c1, c2
    (None: 255), on a (height, width, 3) uint8 canvas filled with ``background``.  Returns the canvas."""
    global _lib
    if _lib is None:
        _lib = ctypes.CDLL(build_render_oracle())
    return _call(_lib.oracle_render_ball, ixyz, colors, height, width, radius, background)


def have_refrender() -> bool:
    return os.path.exists(ref_render_path())


def refrender_ball(ixyz, colors, height: int, width: int, radius: int, background=(0, 0, 0)):
    """The reference's own render_ball (oracle/_ref/libref_render.so), arguments as oracle_render_ball."""
    global _ref
    if _ref is None:
        path = build_render_ref()
        if path is None:
            raise FileNotFoundError("oracle/_ref/libref_render.so: no reference checkout and no earlier build")
        _ref = ctypes.CDLL(path)
    return _call(_ref.render_ball, ixyz, colors, height, width, radius, background)


def render_cases():
    """render_ball inputs: name -> (ixyz (n,3) int32, colors (n,3) float32 or None, h, w, r, background)."""
    rng = np.random.RandomState(160)
    cases = {}

    def cloud(n, h, w, zlo, zhi, margin):
        return np.stack([rng.randint(-margin, h + margin, n), rng.randint(-margin, w + margin, n),
                         rng.randint(zlo, zhi, n)], 1).astype(np.int32)
    for r in (0, 1, 2, 8, 25):
        cases[f"render_r{r}"] = (cloud(400, 96, 128, -60, 60, 30), (rng.rand(400, 3) * 255).astype(np.float32), 96, 128,
                                 r, (0, 0, 0))
    # non-square canvases down to 1 x 1, points off the canvas on every side and at negative z
    cases["render_1x1"] = (cloud(50, 1, 1, -20, 5, 6), (rng.rand(50, 3) * 255).astype(np.float32), 1, 1, 3, (0, 0, 0))
    cases["render_1x37"] = (cloud(80, 1, 37, -30, -1, 4), (rng.rand(80, 3) * 255).astype(np.float32), 1, 37, 2, (9, 0, 3))
    cases["render_53x7"] = (cloud(120, 53, 7, -100, 100, 10), None, 53, 7, 4, (0, 0, 0))
    # duplicate points and equal-depth ties: every duplicate carries its own colour, so the winner is visible
    xyz = cloud(60, 40, 40, -3, 3, 0)
    xyz = np.concatenate([xyz, xyz[rng.randint(0, 60, 140)]])
    xyz[:, 2] = rng.randint(-1, 2, len(xyz))
    cases["render_ties"] = (xyz, (rng.rand(len(xyz), 3) * 255).astype(np.float32), 40, 40, 5, (0, 0, 0))
    # fractional colours near integers, where rounding shade x colour to float before the double product matters
    frac = (rng.randint(0, 256, (300, 3)) + rng.choice([0.0, 0.5, 0.999, 1e-3], (300, 3))).astype(np.float32)
    cases["render_fractional"] = (cloud(300, 64, 64, -40, 40, 5), frac, 64, 64, 10, (0, 0, 0))
    # a non-zero background
    cases["render_background"] = (cloud(200, 70, 90, 0, 50, 15), (rng.rand(200, 3) * 255).astype(np.float32), 70, 90,
                                  8, (17, 128, 250))
    return cases


def record(outdir: str) -> None:
    """Write outdir/render_*.npz: each case's inputs and what the reference's render_ball drew."""
    os.makedirs(outdir, exist_ok=True)
    for name, (xyz, col, h, w, r, bg) in render_cases().items():
        out = refrender_ball(xyz, col, h, w, r, bg)
        arrs = dict(xyz=xyz, h=np.int32(h), w=np.int32(w), r=np.int32(r), background=np.array(bg, np.uint8), out=out)
        if col is not None:
            arrs["colors"] = col
        np.savez_compressed(os.path.join(outdir, name + ".npz"), **arrs)
        print("wrote", name)


if __name__ == "__main__":
    if len(sys.argv) != 2:
        sys.exit("usage: python oracle/render_ref.py OUTDIR")
    record(sys.argv[1])
