"""CPU tests of the mesh-octree route: the reference's golden octrees (tests/golden/ref_mesh_octree.npz, recorded by
oracle/make_ref_golden_mesh_octree.py from the reference's own mesh_to_octree) against the float64 limit set of
tests/mesh_octree_reference.py, the draw-by-draw restatement of wb_mesh_octree_bits against the reference's distribution, install()'s
patch of wisp.ops.spc.mesh_to_octree on the unmodified reference modules, and the refusals of ops.mesh_to_octree without a GPU."""
import itertools
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import mesh_octree_reference as R
import wisp_b200 as W

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = "/root/reference/wisp"
GOLDEN = os.path.join(ROOT, "tests", "golden", "ref_mesh_octree.npz")
MESHES = ("noisy_sphere", "torus", "cube", "open")
N = {5: 2 * 10 ** 5, 7: 10 ** 6}
SEEDS = (0, 1, 2, 3)


def golden_case(name, level):
    """-> (V f32, F int64, [bool grid of each reference seed])."""
    g = np.load(GOLDEN)
    return g[f"{name}_V"], g[f"{name}_F"].astype(np.int64), [R.octree_cells(g[f"{name}_L{level}_s{s}"]) for s in SEEDS]


def tris_and_cdf(V, F):
    """The tris and cdf ops.mesh_to_octree hands the kernel, computed the same way on the CPU."""
    t = torch.from_numpy(V)[torch.from_numpy(F)]
    area = torch.norm(torch.cross(t[:, 0] - t[:, 1], t[:, 1] - t[:, 2], dim=1), p=2, dim=1) * 0.5
    cdf = torch.zeros(t.shape[0] + 1, dtype=torch.float64)
    cdf[1:] = torch.cumsum(area.double(), 0)
    return t.reshape(-1, 9).numpy(), cdf.numpy()


def bits_to_grid(bits, level):
    res = 2 ** level
    idx = np.nonzero(np.unpackbits(np.asarray(bits, np.uint32).view(np.uint8), bitorder="little"))[0]
    g = np.zeros(res ** 3, bool)
    g[idx[idx < res ** 3]] = True
    return g.reshape(res, res, res)


def distribution_bounds(refs):
    """(count low, count high, symmetric-difference bound) for a sampled octree against reference seeds `refs`: the count within
    6 sigma or 0.5 % of the reference mean; each symmetric difference at most 1.25 x the largest reference-to-reference one, or, where
    those are a handful of cells (a saturated level), that one plus 5 Poisson standard deviations and 5."""
    cnt = np.array([r.sum() for r in refs], np.float64)
    tol = max(6.0 * cnt.std(ddof=1), 0.005 * cnt.mean())
    m = max(int((a ^ b).sum()) for a, b in itertools.combinations(refs, 2))
    return cnt.mean() - tol, cnt.mean() + tol, max(1.25 * m, m + 5.0 * m ** 0.5 + 5.0)


@pytest.mark.parametrize("level", sorted(N))
@pytest.mark.parametrize("name", MESHES)
def test_golden_inside_limit_set(name, level):
    """Every cell the reference's sampler marked lies in the float64 limit set, which the sampler approaches but does not fill."""
    V, F, refs = golden_case(name, level)
    lim = R.limit_set(V, F, level)
    for r in refs:
        assert not (r & ~lim).any(), int((r & ~lim).sum())
        assert 0.5 * lim.sum() < r.sum() <= lim.sum()


def test_limit_set_cells():
    """A small triangle deep inside one cell: that cell alone; one on a cell face: both neighbours; one 0.3 cell inside the next cell:
    beyond the h = cell / 4 a grown box reaches past its face."""
    level, cell = 5, 2.0 / 32
    c = (np.array([10, 20, 5]) + 0.5) * cell - 1.0
    tri = np.array([c, c + [cell / 8, 0, 0], c + [0, cell / 8, 0]])
    g = R.limit_set(tri, np.array([[0, 1, 2]]), level)
    assert g.sum() == 1 and g[10, 20, 5]
    on_face = tri - [cell / 2, 0, 0]
    g = R.limit_set(on_face, np.array([[0, 1, 2]]), level)
    assert g.sum() == 2 and g[9, 20, 5] and g[10, 20, 5]
    g = R.limit_set(tri + [0.8 * cell, 0, 0], np.array([[0, 1, 2]]), level)
    assert not g[10, 20, 5] and g[11, 20, 5]


@pytest.mark.parametrize("case", [("noisy_sphere", 5), ("torus", 5), ("cube", 5), ("open", 5), ("torus", 7)])
def test_restatement_has_reference_distribution(case):
    """wb_mesh_octree_bits restated draw by draw (its stream, not torch's) gives octrees that cannot be told from the reference's:
    inside the limit set, the cell count within the reference seeds' spread, and symmetric differences like theirs."""
    name, level = case
    V, F, refs = golden_case(name, level)
    tris, cdf = tris_and_cdf(V, F)
    lim = R.limit_set(V, F, level)
    lo, hi, sd = distribution_bounds(refs)
    for seed in (101, 202):
        g = bits_to_grid(R.sample_bits(tris, cdf, N[level], level, seed), level)
        assert not (g & ~lim).any()
        assert lo <= g.sum() <= hi, (int(g.sum()), lo, hi)
        assert max(int((g ^ r).sum()) for r in refs) <= sd


def test_no_cpu_fallback(monkeypatch):
    monkeypatch.setattr(torch.cuda, "is_available", lambda: False)
    with pytest.raises(W.WispB200Error):
        W.mesh_to_octree(torch.zeros(3, 3), torch.tensor([[0, 1, 2]]), 5)


@pytest.mark.skipif(not os.path.isdir(REF), reason="needs the reference checkout")
def test_install_patches_reference_mesh_to_octree():
    """install() replaces wisp.ops.spc.mesh_to_octree (OctreeAS.from_mesh's name) and wisp.ops.spc.conversions.mesh_to_octree
    (mesh_to_spc's) with functions of the same signature that run ops.mesh_to_octree for levels 1..10 of float32 vertices; levels 0 and
    11 and float64 vertices reach the reference's own function (run here on the CPU); uninstall() restores both names."""
    code = r"""
import inspect, sys, warnings
warnings.filterwarnings("ignore")
sys.path.insert(0, ROOT)
import numpy as np, torch
from oracle import make_ref_golden_mesh_octree as G, mesh_shapes as MS
run = G.reference_mesh_to_octree()
import kaolin.ops.spc as kaolin_spc
import wisp.ops.spc as spc_ops
import wisp.ops.spc.conversions as conv
import wisp_b200 as W
from wisp_b200 import install as I
from wisp_b200 import spc as S
orig = conv.mesh_to_octree
assert spc_ops.mesh_to_octree is orig
assert I.install() is True
for mod in (spc_ops, conv):
    new = mod.mesh_to_octree
    assert new is not orig and new.__wrapped__ is orig
    assert list(inspect.signature(new).parameters) == list(inspect.signature(orig).parameters)
    assert inspect.signature(new).parameters["num_samples"].default == inspect.signature(orig).parameters["num_samples"].default
calls = []
W.ops.mesh_to_octree = lambda v, f, level, num_samples=10 ** 8: calls.append((level, num_samples)) or "native"
V, F = MS.cube()
V32, F64 = torch.from_numpy(V.astype(np.float32)), torch.from_numpy(F)
assert spc_ops.mesh_to_octree(V32, F64, 7) == "native" and conv.mesh_to_octree(V32, F64, 3, 50) == "native"
assert calls == [(7, 10 ** 8), (3, 50)]
# the fall-backs run the reference's body: on the CPU, with Tensor.cuda the identity and Kaolin's quantize_points supplied
cuda = torch.Tensor.cuda
torch.Tensor.cuda = lambda self, *a, **k: self
kaolin_spc.quantize_points = S.quantize_points
for v, level in ((V32, 0), (V32, 11), (V32.double(), 4)):
    for mod in (spc_ops, conv):
        torch.manual_seed(3)
        got = mod.mesh_to_octree(v, F64, level, 2000)
        torch.manual_seed(3)
        assert torch.equal(got, orig(v, F64, level, 2000)), (level, v.dtype)
torch.Tensor.cuda = cuda
assert len(calls) == 2
I.uninstall()
assert spc_ops.mesh_to_octree is orig and conv.mesh_to_octree is orig
print("OK")
"""
    r = subprocess.run([sys.executable, "-c", code.replace("ROOT", repr(ROOT))], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "OK" in r.stdout, (r.stdout[-2000:], r.stderr[-4000:])
