#!/usr/bin/env python
"""Build oracle/_ref/libwisp_ref_kernels.so from the REFERENCE's own CUDA sources (TEST INFRASTRUCTURE; needs a kaolin-wisp checkout).

    python oracle/ref_kernels/build_ref.py        (also called by __graft_entry__.build() when the checkout exists)

Compiles, where they lie under the checkout's wisp/csrc, with nvcc for sm_90a against the installed torch headers:
    ops/hashgrid_interpolate.cpp, ops/hashgrid_interpolate_cuda.cu, ops/uniform_sample.cpp, ops/uniform_sample_cuda.cu,
    render/find_depth_bound.cpp, render/find_depth_bound_cuda.cu
plus oracle/ref_kernels/ref_shim.cpp (C entry points), and links them into oracle/_ref/ (git-ignored).  oracle/make_ref_golden.py runs them once
to store what tests/test_gpu_ref_kernels.py compares against under tests/golden/.
No reference source enters the repository.  One deviation, as SURVEY.md 8(c) found: hashgrid_interpolate_cuda.cu does not compile
against torch >= 2.x because `AT_DISPATCH_*(tensor.type(), ...)` no longer converts (lines 358, 375, 413, 433); the recipe compiles a
TEMPORARY copy (under /tmp, deleted afterwards) in which `.type()` inside those dispatch macros reads `.scalar_type()` -- a one-token
spelling change that alters no arithmetic.  Everything else is compiled byte for byte.  The reference's own build system (setup.py) is
not run."""
import os
import re
import subprocess
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
REF = "/root/reference/wisp/csrc"
OUT_DIR = os.path.join(ROOT, "oracle", "_ref")
OUT = os.path.join(OUT_DIR, "libwisp_ref_kernels.so")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")


def build(force: bool = False) -> str:
    if not os.path.isdir(REF):
        raise RuntimeError("the reference checkout is not present")
    srcs = ["ops/hashgrid_interpolate.cpp", "ops/hashgrid_interpolate_cuda.cu", "ops/uniform_sample.cpp", "ops/uniform_sample_cuda.cu",
            "render/find_depth_bound.cpp", "render/find_depth_bound_cuda.cu"]
    deps = [os.path.join(REF, s) for s in srcs] + [os.path.join(HERE, "ref_shim.cpp"), os.path.abspath(__file__)]
    if not force and os.path.exists(OUT) and os.path.getmtime(OUT) >= max(os.path.getmtime(d) for d in deps):
        return OUT
    import torch
    ti = os.path.join(os.path.dirname(torch.__file__), "include")
    tl = os.path.join(os.path.dirname(torch.__file__), "lib")
    flags = ["-gencode", "arch=compute_90a,code=sm_90a", "-std=c++17", "-O2", "-Xcompiler", "-fPIC", "-DWITH_CUDA",
             f"-D_GLIBCXX_USE_CXX11_ABI={int(torch._C._GLIBCXX_USE_CXX11_ABI)}", "-I", ti, "-I", os.path.join(ti, "torch", "csrc", "api", "include"),
             "-I", os.path.join(REF, "ops"), "-I", os.path.join(REF, "render"), "-w"]
    os.makedirs(OUT_DIR, exist_ok=True)
    with tempfile.TemporaryDirectory(prefix="wisp_ref_build_") as tmp:
        objs = []
        for s in srcs:
            src = os.path.join(REF, s)
            if s.endswith("hashgrid_interpolate_cuda.cu"):
                text = open(src).read()
                patched, n = re.subn(r"(AT_DISPATCH_[A-Z_]+\(\s*\w+)\.type\(\)", r"\1.scalar_type()", text)
                assert n == 4, f"expected 4 dispatch sites, found {n}"
                src = os.path.join(tmp, "hashgrid_interpolate_cuda_patched.cu")
                open(src, "w").write(patched)
            obj = os.path.join(tmp, os.path.basename(s).replace(".", "_") + ".o")
            subprocess.run([NVCC, *flags, "-x", "cu", "-c", src, "-o", obj], check=True)
            objs.append(obj)
        shim = os.path.join(tmp, "ref_shim.o")
        subprocess.run([NVCC, *flags, "-x", "cu", "-c", os.path.join(HERE, "ref_shim.cpp"), "-o", shim], check=True)
        subprocess.run([NVCC, "-shared", "-o", OUT, *objs, shim, "-L", tl, "-ltorch", "-ltorch_cpu", "-ltorch_cuda", "-lc10", "-lc10_cuda", "-lcudart",
                        "-Xlinker", f"-rpath={tl}"], check=True)
    return OUT


if __name__ == "__main__":
    print(build(force="--force" in sys.argv))
