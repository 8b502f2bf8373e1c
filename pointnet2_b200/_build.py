"""Build libpn2_b200.so in-tree with nvcc for sm_90a (and nothing else).

Used by ``pointnet2_b200._lib`` (lazy build on first import when the library is missing or stale)
and by ``__graft_entry__.build()``.  The built ``.so`` is git-ignored.
"""
from __future__ import annotations

import concurrent.futures as cf
import os
import shutil
import subprocess

PKG_DIR = os.path.dirname(os.path.abspath(__file__))
REPO_ROOT = os.path.dirname(PKG_DIR)
CSRC = os.path.join(PKG_DIR, "csrc")
INCLUDE = os.path.join(REPO_ROOT, "include")
BUILD_DIR = os.path.join(PKG_DIR, "build")
LIB_PATH = os.path.join(PKG_DIR, "libpn2_b200.so")

SOURCES = ["api.cu", "fps.cu", "ball_query.cu", "ball_query_grid.cu", "sa_fused.cu", "knn.cu", "group.cu", "interpolate.cu", "scatter_det.cu", "prob_sample.cu", "masked_bn.cu", "sa_mlp.cu", "fp_mlp.cu", "scene.cu", "crops.cu", "shapes.cu", "vscan.cu", "render.cu", "textparse.cu"]
HEADERS = [os.path.join(CSRC, "pn2_common.cuh"), os.path.join(CSRC, "mlp_tile.cuh"), os.path.join(CSRC, "knn_warp.cuh"), os.path.join(INCLUDE, "pn2_api.h")]

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-std=c++17", "-lineinfo",
    # no implicit mul+add contraction anywhere (front end AND ptxas): every fused multiply-add in
    # this library is written explicitly, because bit-exactness with the reference depends on where
    # the roundings are
    "-fmad=false",
    "-Xcompiler", "-fPIC",
    "-I", INCLUDE, "-I", CSRC,
]


def nvcc_path() -> str:
    p = os.environ.get("NVCC") or shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(p):
        raise RuntimeError("nvcc not found: libpn2_b200.so cannot be built (there is no CPU fallback)")
    return p


def is_stale() -> bool:
    if not os.path.exists(LIB_PATH):
        return True
    t = os.path.getmtime(LIB_PATH)
    deps = [os.path.join(CSRC, s) for s in SOURCES] + HEADERS + [__file__]
    return any(os.path.getmtime(d) > t for d in deps)


def source_signature() -> str:
    """Names the state of the sources a library is built from (newest modification time + file count)."""
    deps = [os.path.join(CSRC, s) for s in SOURCES] + HEADERS + [__file__]
    return f"{max(os.path.getmtime(d) for d in deps):.6f}:{len(deps)}"


def _compile_one(nvcc: str, src: str, verbose: bool) -> str:
    obj = os.path.join(BUILD_DIR, os.path.splitext(src)[0] + ".o")
    srcp = os.path.join(CSRC, src)
    if os.path.exists(obj) and all(os.path.getmtime(obj) >= os.path.getmtime(d) for d in [srcp, __file__] + HEADERS):
        return obj
    cmd = [nvcc] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-c", srcp, "-o", obj]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"nvcc failed for {src}:\n{r.stdout}\n{r.stderr}")
    if verbose:
        print(r.stderr)
    return obj


def build(force: bool = False, verbose: bool = False) -> str:
    """Compile every CUDA source for sm_90a and link libpn2_b200.so. Returns its path."""
    if not force and not is_stale():
        return LIB_PATH
    nvcc = nvcc_path()
    os.makedirs(BUILD_DIR, exist_ok=True)
    if force:
        for f in os.listdir(BUILD_DIR):
            if f.endswith(".o"):
                os.remove(os.path.join(BUILD_DIR, f))
    with cf.ThreadPoolExecutor(max_workers=len(SOURCES)) as ex:
        objs = list(ex.map(lambda s: _compile_one(nvcc, s, verbose), SOURCES))
    tmp = LIB_PATH + f".tmp{os.getpid()}"
    cmd = [nvcc, "-shared", "-gencode", "arch=compute_90a,code=sm_90a", "-o", tmp] + objs
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    os.replace(tmp, LIB_PATH)
    return LIB_PATH


if __name__ == "__main__":
    import sys
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
