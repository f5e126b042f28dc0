"""Build libwispb200.so (hand-written sm_90a CUDA behind a C ABI) in-tree with nvcc.

    python kaolin-wisp_b200/build.py [--force]

The library lands in kaolin-wisp_b200/lib/ (git-ignored build output).
nvcc cross-compiles sm_90a without a GPU, so this also runs on a machine without one.
"""
from __future__ import annotations

import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIBDIR = os.path.join(HERE, "lib")
LIB = os.path.join(LIBDIR, os.environ.get("WB_LIB_NAME", "libwispb200.so"))      # WB_LIB_NAME + WB_EXTRA_NVCC_FLAGS: debug variants
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
FLAGS = ["-O3", "-std=c++17", "-lineinfo", "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr"]
FLAGS += os.environ.get("WB_EXTRA_NVCC_FLAGS", "").split()          # debug builds only


def sources():
    return sorted(f for f in os.listdir(CSRC) if f.endswith(".cu"))


def _deps_mtime():
    hdrs = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))]
    hdrs.append(os.path.join(os.path.dirname(HERE), "include", "wispb200.h"))
    return max(os.path.getmtime(h) for h in hdrs)


def build(force: bool = False, verbose: bool = False) -> str:
    os.makedirs(LIBDIR, exist_ok=True)
    objdir = os.path.join(LIBDIR, "obj" + ("_" + os.path.splitext(os.path.basename(LIB))[0] if "WB_LIB_NAME" in os.environ else ""))
    os.makedirs(objdir, exist_ok=True)
    hdr_m = _deps_mtime()
    jobs = []
    objs = []
    for src in sources():
        s = os.path.join(CSRC, src)
        o = os.path.join(objdir, src[:-3] + ".o")
        objs.append(o)
        if force or not os.path.exists(o) or os.path.getmtime(o) < max(os.path.getmtime(s), hdr_m):
            jobs.append([NVCC, *ARCH, *FLAGS, "-c", s, "-o", o])

    def run(cmd):
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("nvcc failed: %s\n%s\n%s" % (" ".join(cmd), r.stdout, r.stderr))
        if verbose and (r.stdout or r.stderr):
            print(r.stdout, r.stderr)

    with ThreadPoolExecutor(max_workers=min(8, max(1, len(jobs)))) as ex:
        list(ex.map(run, jobs))
    if jobs or force or not os.path.exists(LIB):
        run([NVCC, *ARCH, "-shared", "-o", LIB, *objs, "-lcudart"])
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
