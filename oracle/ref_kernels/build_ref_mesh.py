#!/usr/bin/env python
"""Build oracle/_ref/libwisp_ref_mesh2sdf.so: the REFERENCE's mesh-to-SDF kernel (wisp/csrc/external/mesh2sdf_kernel.cu, compiled
unchanged) behind C entry points (oracle/ref_kernels/ref_shim_mesh.cpp).  TEST INFRASTRUCTURE; needs a kaolin-wisp checkout.

    python oracle/ref_kernels/build_ref_mesh.py        (also called by __graft_entry__.build() when the checkout exists)

Same flags as build_ref.py, plus the Python include directory: the kernel includes torch/extension.h, which includes Python.h.
oracle/make_ref_golden_mesh.py runs the result once to store what tests/test_gpu_mesh_sdf.py compares against.
No reference source enters the repository."""
import os
import subprocess
import sys
import sysconfig
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
SRC = "/root/reference/wisp/csrc/external/mesh2sdf_kernel.cu"
OUT_DIR = os.path.join(ROOT, "oracle", "_ref")
OUT = os.path.join(OUT_DIR, "libwisp_ref_mesh2sdf.so")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")


def build(force: bool = False) -> str:
    if not os.path.exists(SRC):
        raise RuntimeError("the reference checkout is not present")
    deps = [SRC, os.path.join(HERE, "ref_shim_mesh.cpp"), os.path.abspath(__file__)]
    if not force and os.path.exists(OUT) and os.path.getmtime(OUT) >= max(os.path.getmtime(d) for d in deps):
        return OUT
    import torch
    ti = os.path.join(os.path.dirname(torch.__file__), "include")
    tl = os.path.join(os.path.dirname(torch.__file__), "lib")
    flags = ["-gencode", "arch=compute_90a,code=sm_90a", "-std=c++17", "-O2", "-Xcompiler", "-fPIC", "-DWITH_CUDA",
             f"-D_GLIBCXX_USE_CXX11_ABI={int(torch._C._GLIBCXX_USE_CXX11_ABI)}", "-I", ti, "-I", os.path.join(ti, "torch", "csrc", "api", "include"),
             "-I", sysconfig.get_paths()["include"], "-w"]
    os.makedirs(OUT_DIR, exist_ok=True)
    with tempfile.TemporaryDirectory(prefix="wisp_ref_mesh_build_") as tmp:
        objs = [os.path.join(tmp, "mesh2sdf_kernel.o"), os.path.join(tmp, "ref_shim_mesh.o")]
        subprocess.run([NVCC, *flags, "-x", "cu", "-c", SRC, "-o", objs[0]], check=True)
        subprocess.run([NVCC, *flags, "-x", "cu", "-c", os.path.join(HERE, "ref_shim_mesh.cpp"), "-o", objs[1]], check=True)
        subprocess.run([NVCC, "-shared", "-o", OUT, *objs, "-L", tl, "-ltorch", "-ltorch_cpu", "-ltorch_cuda", "-lc10", "-lc10_cuda", "-lcudart",
                        "-Xlinker", f"-rpath={tl}"], check=True)
    return OUT


if __name__ == "__main__":
    print(build(force="--force" in sys.argv))
