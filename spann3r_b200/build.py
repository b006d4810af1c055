"""In-tree build of libspann3r_b200.so (sm_90a, H100, only) with nvcc.

`python -m spann3r_b200.build` or `__graft_entry__.build()`.  nvcc cross-compiles without a GPU;
the resulting .so is git-ignored and rebuilt whenever a source or header is newer.
"""
from __future__ import annotations

import concurrent.futures as cf
import glob
import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OBJ = os.path.join(HERE, "build")
LIB = os.path.join(HERE, "libspann3r_b200.so")

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
    "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr",
]


def _nvcc() -> str:
    for c in (shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if c and os.path.exists(c):
            return c
    raise RuntimeError("nvcc not found: libspann3r_b200.so cannot be built (there is no CPU fallback)")


def _newer(src_list, target) -> bool:
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(s) > t for s in src_list)


def build(force: bool = False, verbose: bool = True, defines=(), lib: str = LIB, obj_dir: str = OBJ) -> str:
    """defines / lib / obj_dir: build an A/B variant next to the shipped library, e.g.
    `python -m spann3r_b200.build --variant NAME -DSOME_MACRO=1` -> ab/libspann3r_b200_NAME.so (git-ignored;
    select it with S3R_LIB=...).  The default build takes no defines."""
    return _build(force, verbose, tuple(defines), lib, obj_dir)


def _build(force, verbose, defines, LIB, OBJ) -> str:
    srcs = sorted(glob.glob(os.path.join(CSRC, "*.cu")))
    hdrs = sorted(glob.glob(os.path.join(CSRC, "*.cuh"))) + [os.path.join(os.path.dirname(HERE), "include", "spann3r_b200.h")]
    if not force and not _newer(srcs + hdrs, LIB):
        return LIB
    os.makedirs(OBJ, exist_ok=True)
    nvcc = _nvcc()

    def compile_one(src):
        obj = os.path.join(OBJ, os.path.basename(src)[:-3] + ".o")
        if force or _newer([src] + hdrs, obj):
            cmd = [nvcc] + NVCC_FLAGS + list(defines) + ["-c", src, "-o", obj]
            r = subprocess.run(cmd, capture_output=True, text=True)
            if r.returncode != 0:
                raise RuntimeError(f"nvcc failed for {src}:\n{r.stdout}\n{r.stderr}")
            if verbose:
                print("compiled", os.path.basename(src), flush=True)
        return obj

    with cf.ThreadPoolExecutor(max_workers=min(8, len(srcs))) as ex:
        objs = list(ex.map(compile_one, srcs))
    cmd = [nvcc, "-shared", "-o", LIB] + objs + ["-gencode", "arch=compute_90a,code=sm_90a"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    if verbose:
        print("linked", LIB, flush=True)
    return LIB


if __name__ == "__main__":
    if "--variant" in sys.argv:
        name = sys.argv[sys.argv.index("--variant") + 1]
        root = os.path.dirname(HERE)
        os.makedirs(os.path.join(root, "ab"), exist_ok=True)
        print(build(force=True, defines=[a for a in sys.argv if a.startswith("-D")],
                    lib=os.path.join(root, "ab", f"libspann3r_b200_{name}.so"), obj_dir=os.path.join(root, "ab", f"obj_{name}")))
    else:
        build(force="--force" in sys.argv)
