"""In-tree nvcc build of libgavatar_sm90.so (sm_90a only; no JIT cache, no multi-arch)."""
from __future__ import annotations

import glob
import os
import shutil
import subprocess
from concurrent.futures import ThreadPoolExecutor

_PKG = os.path.dirname(os.path.abspath(__file__))
_CSRC = os.path.join(_PKG, "csrc")
_OBJ = os.path.join(_PKG, "build")
LIB_PATH = os.path.join(_PKG, "libgavatar_sm90.so")

NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
              "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr"]


def _nvcc() -> str:
    for cand in (shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found; libgavatar_sm90.so cannot be built")


def _deps_mtime() -> float:
    hdrs = glob.glob(os.path.join(_CSRC, "*.cuh")) + glob.glob(os.path.join(_CSRC, "*.h")) + \
        glob.glob(os.path.join(os.path.dirname(_PKG), "include", "*.h"))
    return max([os.path.getmtime(h) for h in hdrs] + [0.0])


def build_library(force: bool = False, verbose: bool = False) -> str:
    """Compile every csrc/*.cu for sm_90a and link the shared library.  Incremental per translation unit."""
    nvcc = _nvcc()
    os.makedirs(_OBJ, exist_ok=True)
    srcs = sorted(glob.glob(os.path.join(_CSRC, "*.cu")))
    if not srcs:
        raise RuntimeError("no CUDA sources found under " + _CSRC)
    hdr_m = _deps_mtime()
    jobs, objs = [], []
    for s in srcs:
        o = os.path.join(_OBJ, os.path.basename(s)[:-3] + ".o")
        objs.append(o)
        if force or not os.path.exists(o) or os.path.getmtime(o) < max(os.path.getmtime(s), hdr_m):
            jobs.append([nvcc, *NVCC_FLAGS, "-c", s, "-o", o])

    def run(cmd):
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("nvcc failed: " + " ".join(cmd) + "\n" + r.stdout + r.stderr)
        if verbose and (r.stdout or r.stderr):
            print(r.stdout + r.stderr)

    if jobs:
        with ThreadPoolExecutor(max_workers=min(8, len(jobs))) as ex:
            list(ex.map(run, jobs))
    if jobs or not os.path.exists(LIB_PATH) or any(os.path.getmtime(o) > os.path.getmtime(LIB_PATH) for o in objs):
        run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-shared", "-o", LIB_PATH, *objs, "-lcudart"])
    return LIB_PATH


if __name__ == "__main__":
    import sys
    print(build_library(force="--force" in sys.argv, verbose=True))
