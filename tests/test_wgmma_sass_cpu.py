"""The shade kernels' wgmma chains are pipelined in the machine code (no GPU needed: nvcc cross-compiles sm_90a).

ptxas serializes every wgmma of a kernel -- a WARPGROUP.ARRIVE before and a WARPGROUP.DEPBAR.LE gsb0, 0x0 after each HGMMA, so a
K-step waits for the previous one -- when it cannot prove the warpgroup converged around them (warning C7520) or when an
accumulator starts from a constant it tracks.  wb_shade_tc.cu is compiled exactly as build.py compiles it, plus -Xptxas -v.
"""
import importlib.util
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "kaolin-wisp_b200", "csrc", "wb_shade_tc.cu")
KERNELS = ("wb_shade_fwd_tc_kernel", "wb_mlp_bwd_tc_kernel")


def _build_module():
    spec = importlib.util.spec_from_file_location("wisp_b200_build_sass", os.path.join(ROOT, "kaolin-wisp_b200", "build.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _shade(name):
    return any(k in name for k in KERNELS)


def ptxas_report(text):
    """{kernel: {"c7520": bool, "spill": (stores, loads)}} of the shade kernels in ptxas -v output."""
    out = {}
    cur = None
    for line in text.splitlines():
        m = re.search(r"Compiling entry function '(\S+)'", line)
        if m:
            cur = m.group(1)
            if _shade(cur):
                out.setdefault(cur, {"c7520": False, "spill": None})
            continue
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and cur and _shade(cur):
            out[cur]["spill"] = (int(m.group(1)), int(m.group(2)))
        if "C7520" in line:
            for k in re.findall(r"function '(\S+?)'", line):
                if _shade(k):
                    out.setdefault(k, {"c7520": False, "spill": None})["c7520"] = True
    return out


def hgmma_report(sass):
    """{kernel: (HGMMAs, HGMMAs carrying gsb0, WARPGROUP.DEPBARs)} of the shade kernels in cuobjdump -sass output."""
    out = {}
    for body in re.split(r"\n\s*Function : ", sass)[1:]:
        name = body.split("\n", 1)[0].strip()
        if not _shade(name):
            continue
        out[name] = (len(re.findall(r"\bHGMMA\.", body)), len(re.findall(r"\bHGMMA\.[^;]*\bgsb0\b", body)),
                     len(re.findall(r"\bWARPGROUP\.DEPBAR", body)))
    return out


def check(ptxas_text, sass):
    """The assertions of the test, on a compile's ptxas -v output and SASS; returns the per-kernel HGMMA report."""
    rep = ptxas_report(ptxas_text)
    assert rep, "no shade kernel in the ptxas output"
    for k, r in rep.items():
        assert not r["c7520"], f"{k}: wgmma serialized (C7520)"
        assert r["spill"] == (0, 0), f"{k}: spills {r['spill']}"
    hg = hgmma_report(sass)
    assert set(hg) == set(rep), (sorted(hg), sorted(rep))
    for k, (n, g, dep) in hg.items():
        assert n > 0, k
        # gsb0 marks an HGMMA that a wait depends on: the last MMA of a chain, or every MMA of a serialized one
        assert 2 * g <= n, f"{k}: {g} of {n} HGMMAs carry gsb0 ({dep} DEPBARs): the chains are serialized"
    return hg


BUILD = _build_module()


@pytest.mark.skipif(not os.path.exists(BUILD.NVCC) and shutil.which(BUILD.NVCC) is None, reason="needs nvcc")
def test_shade_wgmma_chains_pipelined(tmp_path):
    b = BUILD
    obj = str(tmp_path / "wb_shade_tc.o")
    r = subprocess.run([b.NVCC, *b.ARCH, *b.FLAGS, "-Xptxas", "-v", "-c", SRC, "-o", obj], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-4000:]
    cuobjdump = os.path.join(os.path.dirname(b.NVCC), "cuobjdump")
    sass = subprocess.run([cuobjdump, "-sass", obj], capture_output=True, text=True, check=True).stdout
    hg = check(r.stdout + r.stderr, sass)
    assert any("wb_mlp_bwd_tc_kernel" in k for k in hg) and any("wb_shade_fwd_tc_kernel" in k for k in hg)
