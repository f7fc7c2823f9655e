"""Build the UNMODIFIED reference rasterizer (CUDA) as a checker:  oracle/_ref/ref_dgr_C.so

TEST INFRASTRUCTURE ONLY -- nothing in the product path imports this.

The sources are compiled from where they lie in a RaDe-GS checkout (never copied into the repo): $RADE_GS_REFERENCE when it is
set, else the checkout this repository is developed beside, `reference/` next to the repository's root directory:
    submodules/diff-gaussian-rasterization/{cuda_rasterizer/{forward,backward,rasterizer_impl}.cu,
                                            rasterize_points.cu, ext.cpp}
with two non-source workarounds (SURVEY.md section 0):
  * `-I oracle/glm_shim`  -- third_party/glm is an empty directory in the checkout; the shim is our own
    header restating the glm operators the reference uses;
  * `-include cstdint`    -- cuda_rasterizer/rasterizer_impl.h uses std::uintptr_t without including it.
Flags otherwise follow the reference's setup.py (no fast-math, default -fmad) plus the sm_90a gencode.

The module is exported under the name `ref_dgr_C` (the reference's own name is
`diff_gaussian_rasterization._C`, which the product occupies) and exposes the reference's four pybind
symbols unchanged.  Outputs go only to oracle/_ref/ (git-ignored).

Usage:  python oracle/build_ref.py [--force]
"""
from __future__ import annotations

import os
import subprocess
import sys
import sysconfig
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
REF_CHECKOUT = os.environ.get("RADE_GS_REFERENCE") or os.path.join(os.path.dirname(os.path.dirname(HERE)), "reference")
REF_ROOT = os.path.join(REF_CHECKOUT, "submodules", "diff-gaussian-rasterization")
OUT_DIR = os.path.join(HERE, "_ref")
OBJ_DIR = os.path.join(HERE, "_build", "ref")
MODULE = "ref_dgr_C"
SOURCES = [
    "cuda_rasterizer/rasterizer_impl.cu",
    "cuda_rasterizer/forward.cu",
    "cuda_rasterizer/backward.cu",
    "rasterize_points.cu",
    "ext.cpp",
]


def available() -> bool:
    return os.path.isdir(REF_ROOT)


def target() -> str:
    return os.path.join(OUT_DIR, MODULE + ".so")


def build(force: bool = False, verbose: bool = True) -> str | None:
    """Returns the path of the built module, or None when the reference checkout is absent and nothing is prebuilt."""
    out = target()
    if not available():
        return out if os.path.exists(out) else None
    srcs = [os.path.join(REF_ROOT, s) for s in SOURCES]
    shim = os.path.join(HERE, "glm_shim", "glm", "glm.hpp")
    newest = max(os.path.getmtime(p) for p in srcs + [shim, __file__])
    if not force and os.path.exists(out) and os.path.getmtime(out) >= newest:
        return out

    from torch.utils import cpp_extension as ce  # noqa: E402  (slow import, only when building)

    os.makedirs(OUT_DIR, exist_ok=True)
    os.makedirs(OBJ_DIR, exist_ok=True)
    incs = [os.path.join(HERE, "glm_shim"), REF_ROOT] + ce.include_paths() + [sysconfig.get_paths()["include"]]
    common = ["-std=c++17", "-O3", "-DTORCH_EXTENSION_NAME=" + MODULE, "-DTORCH_API_INCLUDE_EXTENSION_H",
              "-include", "cstdint"] + ["-I" + i for i in incs]
    nvcc = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "nvcc")

    def compile_one(src: str) -> str:
        obj = os.path.join(OBJ_DIR, os.path.basename(src) + ".o")
        if src.endswith(".cu"):
            cmd = [nvcc, "-c", src, "-o", obj, "-gencode", "arch=compute_90a,code=sm_90a",
                   "--expt-relaxed-constexpr", "-Xcompiler", "-fPIC", "-w"] + common
        else:
            cmd = ["g++", "-c", src, "-o", obj, "-fPIC", "-w"] + common
        if verbose:
            print("[build_ref]", os.path.basename(src), flush=True)
        subprocess.run(cmd, check=True)
        return obj

    with ThreadPoolExecutor(max_workers=5) as ex:
        objs = list(ex.map(compile_one, srcs))

    libdirs = ce.library_paths()
    link = ["g++", "-shared", "-o", out] + objs + ["-L" + d for d in libdirs] + \
           ["-L/usr/local/cuda/lib64", "-lc10", "-lc10_cuda", "-ltorch_cpu", "-ltorch_cuda", "-ltorch", "-ltorch_python",
            "-lcudart"] + ["-Wl,-rpath," + d for d in libdirs]
    subprocess.run(link, check=True)
    if verbose:
        print("[build_ref] wrote", out, flush=True)
    return out


def load():
    """Import the prebuilt reference module.  Raises if it was never built."""
    import importlib.util

    import torch  # noqa: F401  (libtorch must be loaded before the extension)

    path = target()
    if not os.path.exists(path):
        raise FileNotFoundError(path + " missing: run `python oracle/build_ref.py` with a RaDe-GS checkout at " + REF_CHECKOUT +
                                " (or named by $RADE_GS_REFERENCE)")
    spec = importlib.util.spec_from_file_location(MODULE, path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


if __name__ == "__main__":
    p = build(force="--force" in sys.argv)
    print(p if p else "reference sources absent and no prebuilt module")
