"""CPU tests of the mesh-SDF route: the numpy restatement (tests/mesh_sdf_reference.py) against analytic shapes and against the
reference kernel's golden (tests/golden/ref_mesh_sdf.npz), the ctypes prototype of wb_mesh_sdf against the header, install()'s
patch of wisp.ops.mesh.compute_sdf on the unmodified reference module, and the missing CPU fallback."""
import ctypes as C
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

import mesh_sdf_reference as R
import wisp_b200 as W
from oracle import mesh_shapes as MS

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = "/root/reference/wisp"
GOLDEN = os.path.join(ROOT, "tests", "golden", "ref_mesh_sdf.npz")
MAX_PAIRS = 2 * 10 ** 6


def test_restatement_cube_is_exact():
    """The cube's mesh is the box itself: distances equal the analytic box distance to fp32 rounding, and every sign the
    restatement calls unambiguous is the analytic one."""
    V, F = MS.cube(0.5)
    P = np.concatenate([np.random.default_rng(0).uniform(-1.1, 1.1, (3000, 3)), MS.feature_points(V, F, 50, np.random.default_rng(1))])
    r = R.mesh_sdf(V[F].reshape(-1, 9), P)
    q = np.abs(P) - 0.5
    exact = np.linalg.norm(np.maximum(q, 0), axis=1) + np.minimum(q.max(1), 0)
    assert np.all(np.abs(np.abs(r["sdf"]) - np.abs(exact)) <= 4 * r["tol"] + 1e-12)
    ok = r["sign_ok"] & (np.abs(exact) > 1e-9)
    assert ok.mean() > 0.9 and np.array_equal(r["inside"][ok], exact[ok] < 0)


@pytest.mark.parametrize("shape", ["sphere", "torus"])
def test_restatement_curved_shapes(shape):
    """Sphere and torus meshes: distances within the chord error of the analytic surface, and the analytic inside/outside for every
    unambiguous point farther from the surface than that error."""
    rng = np.random.default_rng(2)
    if shape == "sphere":
        V, F = MS.icosphere(3, 0.6)
        P = rng.uniform(-1, 1, (1500, 3))
        exact = np.linalg.norm(P, axis=1) - 0.6
        chord = 0.6 * 0.02
    else:
        V, F = MS.torus(64, 32, 0.55, 0.2)
        P = rng.uniform(-1, 1, (800, 3))
        exact = np.hypot(np.hypot(P[:, 0], P[:, 1]) - 0.55, P[:, 2]) - 0.2
        chord = 0.75 * (1 - np.cos(np.pi / 64)) + 0.2 * (1 - np.cos(np.pi / 32))
    r = R.mesh_sdf(V[F].reshape(-1, 9), P)
    assert np.all(np.abs(np.abs(r["sdf"]) - np.abs(exact)) <= chord)
    ok = r["sign_ok"] & (np.abs(exact) > chord)
    assert ok.mean() > 0.8 and np.array_equal(r["inside"][ok], exact[ok] < 0)


def test_restatement_empty_mesh_and_nan():
    P = np.array([[0.0, 0.0, 0.0], [np.nan, 0.0, 0.0]])
    assert np.all(R.mesh_sdf(np.zeros((0, 9)), P)["sdf"] == np.inf)
    V, F = MS.cube()
    r = R.mesh_sdf(V[F].reshape(-1, 9), P)
    assert r["sdf"][0] == -0.5 and r["sdf"][1] == np.inf


@pytest.mark.parametrize("case", ["icosphere", "torus", "cube", "open", "noisy_sphere"])
def test_restatement_against_reference_kernel_golden(case):
    """On a seeded subsample: the reference kernel's distance inside the restatement's bound of its own value, and its sign on every
    point the restatement calls unambiguous."""
    g = np.load(GOLDEN)
    V, F, P, gold = (g[f"{case}_{k}"] for k in ("V", "F", "points", "sdf"))
    F, gold = F.astype(np.int64), gold.astype(np.float64)
    idx = np.sort(np.random.default_rng(11).choice(P.shape[0], min(P.shape[0], MAX_PAIRS // F.shape[0]), replace=False))
    r = R.mesh_sdf(V[F].reshape(-1, 9), P[idx])
    assert np.all(np.abs(np.abs(r["sdf"]) - np.abs(gold[idx])) <= r["tol"])
    ok = r["sign_ok"]
    assert ok.mean() > 0.5 and np.array_equal(r["inside"][ok], gold[idx][ok] < 0)


def test_reference_refuses_float32():
    """The reference kernel reads its inputs with data<double>(): the float32 tensors its callers pass are refused."""
    msg = str(np.load(GOLDEN)["f32_error"])
    assert "Double" in msg and "Float" in msg, msg


def test_mesh_sdf_prototype_matches_header():
    src = open(os.path.join(ROOT, "include", "wispb200.h")).read()
    m = re.search(r"\bint\s+wb_mesh_sdf\s*\(([^)]*)\)\s*;", src)
    assert m, "wb_mesh_sdf is not declared in include/wispb200.h"
    A = W._cabi
    ctype = {"const double*": C.c_void_p, "double*": C.c_void_p, "void*": C.c_void_p, "int64_t": C.c_int64, "wb_stream": C.c_void_p}
    params = [re.sub(r"\s+", " ", p.strip()) for p in m.group(1).split(",")]
    types = [re.sub(r"\s*\*\s*", "*", re.match(r"(.*?\*?)\s*\w+$", p).group(1)) for p in params]
    assert [ctype[t] for t in types] == A.MESH_SDF_ARGTYPES
    L = A.lib()
    assert L.wb_mesh_sdf.argtypes == A.MESH_SDF_ARGTYPES and L.wb_mesh_sdf.restype is C.c_int
    assert L.wb_mesh_sdf_workspace_bytes.restype is C.c_int64
    assert L.wb_mesh_sdf_workspace_bytes(0) > 0 and L.wb_mesh_sdf_workspace_bytes(-1) < 0
    if torch.cuda.is_available():          # the radix sort's scratch size is a query of the device
        assert L.wb_mesh_sdf_workspace_bytes(1000) > 1000 * 9 * 8


def test_no_cpu_fallback(monkeypatch):
    V, F = MS.cube()
    monkeypatch.setattr(torch.cuda, "is_available", lambda: False)
    with pytest.raises(W.WispB200Error):
        W.compute_sdf(torch.from_numpy(V), torch.from_numpy(F), torch.zeros(4, 3))


def test_bad_inputs_are_refused():
    V, F = MS.cube()
    for v, f, p in ((V[:, :2], F, np.zeros((2, 3))), (V, F.astype(np.float64), np.zeros((2, 3))), (V, F, np.zeros((2, 3), np.float16))):
        with pytest.raises(W.WispB200Error):
            W.compute_sdf(torch.from_numpy(v), torch.from_numpy(f), torch.from_numpy(p))


@pytest.mark.skipif(not os.path.isdir(REF), reason="needs the reference checkout")
def test_install_patches_reference_compute_sdf():
    """install() replaces wisp.ops.mesh.compute_sdf (what both SDF datasets call as mesh_ops.compute_sdf) with a function of the
    same signature that runs ops.compute_sdf; uninstall() restores the reference's."""
    code = r"""
import inspect, sys, warnings
warnings.filterwarnings("ignore")
sys.path.insert(0, ROOT)
import torch
from oracle import ref_import
ref_import.install()
import wisp.ops.mesh as mesh_ops
import wisp_b200 as W
from wisp_b200 import install as I
orig = mesh_ops.compute_sdf
assert I.install() is True
new = mesh_ops.compute_sdf
assert new is not orig and new.__wrapped__ is orig
assert list(inspect.signature(new).parameters) == list(inspect.signature(orig).parameters)
assert inspect.signature(new).parameters["split_size"].default == inspect.signature(orig).parameters["split_size"].default
calls = []
W.ops.compute_sdf = lambda V, F, points, split_size=10 ** 6: calls.append(split_size) or "native"
assert mesh_ops.compute_sdf(torch.zeros(3, 3), torch.zeros(1, 3, dtype=torch.long), torch.zeros(2, 3)) == "native" and calls == [10 ** 6]
I.uninstall()
assert mesh_ops.compute_sdf is orig
print("OK")
"""
    r = subprocess.run([sys.executable, "-c", code.replace("ROOT", repr(ROOT))], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "OK" in r.stdout, (r.stdout[-2000:], r.stderr[-4000:])
