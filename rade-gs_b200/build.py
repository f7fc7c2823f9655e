"""In-tree build of the H100 rasterizer (sm_90a only).

Produces, next to the Python packages so they travel with the source tree:
  rade-gs_b200/rade_gs_b200/librgs_b200.so              -- the C-ABI library (include/rgs_b200.h), no torch dependency
  rade-gs_b200/diff_gaussian_rasterization/_C.so        -- torch/pybind11 glue exporting the reference's four symbols

Usage:  python rade-gs_b200/build.py [--force] [--no-glue] [-v]
"""
from __future__ import annotations

import os
import subprocess
import sys
import sysconfig
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CSRC = os.path.join(HERE, "csrc")
OBJ = os.path.join(HERE, "build")
LIB = os.path.join(HERE, "rade_gs_b200", "librgs_b200.so")
GLUE = os.path.join(HERE, "diff_gaussian_rasterization", "_C.so")
NVCC = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "nvcc")

CORE_SOURCES = ["rgs_api.cu", "rgs_preprocess.cu", "rgs_binning.cu", "rgs_render_fwd.cu", "rgs_render_bwd.cu", "rgs_preprocess_bwd.cu", "rgs_activation.cu", "rgs_image_loss.cu", "rgs_integrate.cu", "rgs_exchange.cu", "rgs_knn.cu"]
HEADERS = ["rgs_common.cuh", "rgs_geom.cuh", "rgs_render_common.cuh", os.path.join(ROOT, "include", "rgs_b200.h")]
# per-file extra flags: backward-preprocess is pure gradient arithmetic with a 1e-3 tolerance -> approximate float
# division / sqrt (2-3 instructions instead of ~10 with a slow-path call); the eigen-solver inside it uses explicit IEEE
# intrinsics.  Forward preprocess keeps IEEE division: its expression chain decides the tile keys bit-exactly.
EXTRA_FLAGS = {"rgs_preprocess_bwd.cu": ["-prec-div=false", "-prec-sqrt=false"]}
NVCC_FLAGS = ["-std=c++17", "-O3", "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-Xcompiler", "-fPIC",
              "--expt-relaxed-constexpr", "-Xcudafe", "--diag_suppress=177"]


def _mtime(path: str) -> float:
    return os.path.getmtime(path) if os.path.exists(path) else 0.0


def _run(cmd, verbose):
    if verbose:
        print(" ".join(cmd), flush=True)
    subprocess.run(cmd, check=True)


def build_core(force=False, verbose=False) -> str:
    os.makedirs(OBJ, exist_ok=True)
    hdr_time = max(_mtime(h if os.path.isabs(h) else os.path.join(CSRC, h)) for h in HEADERS)
    hdr_time = max(hdr_time, _mtime(__file__))

    def one(src):
        s = os.path.join(CSRC, src)
        o = os.path.join(OBJ, src + ".o")
        if force or _mtime(o) < max(_mtime(s), hdr_time):
            print("[build] nvcc", src, flush=True)
            _run([NVCC, "-c", s, "-o", o] + NVCC_FLAGS + EXTRA_FLAGS.get(src, []) + (["-Xptxas", "-v"] if verbose else []), verbose)
            return o, True
        return o, False

    with ThreadPoolExecutor(max_workers=6) as ex:
        res = list(ex.map(one, CORE_SOURCES))
    objs = [o for o, _ in res]
    if force or any(ch for _, ch in res) or not os.path.exists(LIB):
        tmp = LIB + ".tmp"   # link to a temporary name and rename: a snapshot of the tree never sees a half-written library
        _run([NVCC, "-shared", "-o", tmp] + objs + ["-gencode", "arch=compute_90a,code=sm_90a", "-cudart", "shared"], verbose)
        os.replace(tmp, LIB)
        print("[build] wrote", LIB, flush=True)
    return LIB


def build_glue(force=False, verbose=False) -> str:
    src = os.path.join(CSRC, "torch_glue.cpp")
    if not force and _mtime(GLUE) >= max(_mtime(src), _mtime(os.path.join(ROOT, "include", "rgs_b200.h")), _mtime(__file__)):
        return GLUE
    from torch.utils import cpp_extension as ce

    incs = ce.include_paths() + [sysconfig.get_paths()["include"], os.path.join(ROOT, "include"), "/usr/local/cuda/include"]
    libdirs = ce.library_paths()
    o = os.path.join(OBJ, "torch_glue.o")
    print("[build] g++ torch_glue.cpp", flush=True)
    _run(["g++", "-c", src, "-o", o, "-std=c++17", "-O2", "-fPIC", "-DTORCH_EXTENSION_NAME=_C", "-DTORCH_API_INCLUDE_EXTENSION_H", "-w"]
         + ["-I" + i for i in incs], verbose)
    libdir = os.path.dirname(LIB)
    tmp = GLUE + ".tmp"
    _run(["g++", "-shared", "-o", tmp, o, "-L" + libdir, "-lrgs_b200"] + ["-L" + d for d in libdirs] +
         ["-L/usr/local/cuda/lib64", "-lc10", "-lc10_cuda", "-ltorch_cpu", "-ltorch_cuda", "-ltorch", "-ltorch_python", "-lcudart",
          "-Wl,-rpath,$ORIGIN/../rade_gs_b200"] + ["-Wl,-rpath," + d for d in libdirs], verbose)
    os.replace(tmp, GLUE)
    print("[build] wrote", GLUE, flush=True)
    return GLUE


def build_all(force=False, verbose=False, glue=True):
    build_core(force, verbose)
    if glue:
        build_glue(force, verbose)


if __name__ == "__main__":
    build_all(force="--force" in sys.argv, verbose="-v" in sys.argv, glue="--no-glue" not in sys.argv)
