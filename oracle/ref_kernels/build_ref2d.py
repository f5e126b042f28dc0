#!/usr/bin/env python
"""Build oracle/_ref/libwisp_ref_hashgrid2d.so: C entry points (oracle/ref_kernels/ref_shim2d.cpp) around the REFERENCE's own 2-D
hash-grid kernels (TEST INFRASTRUCTURE; needs a kaolin-wisp checkout).

    python oracle/ref_kernels/build_ref2d.py        (also called by __graft_entry__.build() when the checkout exists)

The reference operators themselves are the ones oracle/ref_kernels/build_ref.py compiles into oracle/_ref/libwisp_ref_kernels.so (built
first when missing or stale); this recipe compiles only the shim, with the same flags, and links it against that library (found next
to it at run time).  oracle/make_ref_golden2d.py runs it once to store what tests/test_gpu_ref_hashgrid2d.py compares against.
No reference source enters the repository."""
import importlib.util
import os
import subprocess
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))


def _build_ref():
    spec = importlib.util.spec_from_file_location("wisp_b200_build_ref", os.path.join(HERE, "build_ref.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def build(force: bool = False) -> str:
    br = _build_ref()
    base = br.build(force=force)
    out = os.path.join(br.OUT_DIR, "libwisp_ref_hashgrid2d.so")
    deps = [base, os.path.join(HERE, "ref_shim2d.cpp"), os.path.abspath(__file__)]
    if not force and os.path.exists(out) and os.path.getmtime(out) >= max(os.path.getmtime(d) for d in deps):
        return out
    import torch
    ti = os.path.join(os.path.dirname(torch.__file__), "include")
    tl = os.path.join(os.path.dirname(torch.__file__), "lib")
    flags = ["-gencode", "arch=compute_90a,code=sm_90a", "-std=c++17", "-O2", "-Xcompiler", "-fPIC", "-DWITH_CUDA",
             f"-D_GLIBCXX_USE_CXX11_ABI={int(torch._C._GLIBCXX_USE_CXX11_ABI)}", "-I", ti, "-I", os.path.join(ti, "torch", "csrc", "api", "include"), "-w"]
    with tempfile.TemporaryDirectory(prefix="wisp_ref2d_build_") as tmp:
        shim = os.path.join(tmp, "ref_shim2d.o")
        subprocess.run([br.NVCC, *flags, "-x", "cu", "-c", os.path.join(HERE, "ref_shim2d.cpp"), "-o", shim], check=True)
        subprocess.run([br.NVCC, "-shared", "-o", out, shim, "-L", br.OUT_DIR, "-l:" + os.path.basename(base), "-L", tl, "-ltorch", "-ltorch_cpu",
                        "-ltorch_cuda", "-lc10", "-lc10_cuda", "-lcudart", "-Xlinker", "-rpath=$ORIGIN", "-Xlinker", f"-rpath={tl}"], check=True)
    return out


if __name__ == "__main__":
    print(build(force="--force" in sys.argv))
