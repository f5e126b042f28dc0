"""The decoder kernels compiled for the app/nerf geometry (TcShapeNerf64 in wb_shade_tc.cu) hold only the code that geometry runs
(no GPU needed: nvcc cross-compiles sm_90a).

The run-time kernels switch over every padded width 16 .. 128 in every layer; the TcShape instances must keep the pipelined wgmma
chains of test_wgmma_sass_cpu.py, use no HGMMA wider than the widest layer (N = 64) and stay far below the run-time kernels' size:
on sm_90a the fused backward went from 21 400 to 6 440 SASS instructions and the hash-grid forward from 5 984 to 3 352.
"""
import os
import re
import shutil
import subprocess

import pytest

from test_wgmma_sass_cpu import BUILD, SRC, check

SHAPE = "7TcShapeILi2ELi3E6TcListIJLi32ELi64ELi48ELi64ELi64EEES1_IJLi64ELi16ELi64ELi64ELi16EEEE"
# SASS instruction bounds of the TcShapeNerf64 instances, about 25 % above what nvcc 12.9 makes of them
MAX_INSTR = {"wb_mlp_bwd_tc_kernel": 8192, "wb_shade_fwd_tc_kernel": 4096}


def shape_report(sass):
    """{kernel: (SASS instructions, widest HGMMA N)} of the TcShapeNerf64 kernel instances in cuobjdump -sass output."""
    out = {}
    for body in re.split(r"\n\s*Function : ", sass)[1:]:
        name = body.split("\n", 1)[0].strip()
        if SHAPE not in name:
            continue
        widths = [int(n) for n in re.findall(r"\bHGMMA\.64x(\d+)x16", body)]
        out[name] = (len(re.findall(r"/\*[0-9a-f]{4,}\*/", body)), max(widths, default=0))
    return out


@pytest.mark.skipif(not os.path.exists(BUILD.NVCC) and shutil.which(BUILD.NVCC) is None, reason="needs nvcc")
def test_shape_kernels_straight_line(tmp_path):
    b = BUILD
    obj = str(tmp_path / "wb_shade_tc.o")
    r = subprocess.run([b.NVCC, *b.ARCH, *b.FLAGS, "-Xptxas", "-v", "-c", SRC, "-o", obj], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-4000:]
    cuobjdump = os.path.join(os.path.dirname(b.NVCC), "cuobjdump")
    sass = subprocess.run([cuobjdump, "-sass", obj], capture_output=True, text=True, check=True).stdout
    hg = check(r.stdout + r.stderr, sass)          # no C7520, no spills, gsb0 on at most half of the HGMMAs
    rep = shape_report(sass)
    assert sorted(k for k in hg if SHAPE in k) == sorted(rep)
    for kern, bound in MAX_INSTR.items():
        got = [(k, v) for k, v in rep.items() if kern in k]
        assert len(got) == 1, (kern, sorted(rep))
        k, (n, widest) = got[0]
        assert widest == 64, f"{k}: widest HGMMA N = {widest}"
        assert n <= bound, f"{k}: {n} SASS instructions (bound {bound})"
