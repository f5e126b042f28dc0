"""wisp_b200.mesh_to_octree (wb_mesh_octree_bits + spc.points_to_octree) on the H100:
  - the kernel's bitmask word for word against its draw-by-draw restatement (tests/mesh_octree_reference.py);
  - every cell inside the float64 limit set, for every golden mesh and level, three seeds, at the default 10^8 samples;
  - the reference's distribution: cell counts and symmetric differences against the reference's own octrees (the golden);
  - a well-formed octree (scan_octree, generate_points, points_to_octree, OctreeAS query / raytrace); reproducibility by seed and
    by torch.manual_seed, through the install() replacement too; inputs on the host and int32 faces;
  - 2^32 samples in one call: the 64-bit sample counter, and a face of area share 2^-26 that a 24-bit uniform would never draw;
  - the refusals."""
import types

import numpy as np
import pytest
import torch

import mesh_octree_reference as R
import wisp_b200 as W
from test_mesh_octree_cpu import MESHES, N, bits_to_grid, distribution_bounds, golden_case
from wisp_b200 import _cabi as A
from wisp_b200 import install as I
from wisp_b200 import spc as S

pytestmark = pytest.mark.gpu


def kernel_bits(V, F, level, n, seed):
    """One wb_mesh_octree_bits call on the tris / cdf that ops.mesh_to_octree builds -> (bits as numpy uint32, tris, cdf)."""
    t = torch.from_numpy(V).cuda()[torch.from_numpy(F).cuda()]
    area = torch.norm(torch.cross(t[:, 0] - t[:, 1], t[:, 1] - t[:, 2], dim=1), p=2, dim=1) * 0.5
    cdf = torch.zeros(t.shape[0] + 1, dtype=torch.float64, device="cuda")
    cdf[1:] = torch.cumsum(area.double(), 0)
    tris = t.reshape(-1, 9).contiguous()
    bits = torch.zeros((8 ** level + 31) // 32, dtype=torch.int32, device="cuda")
    A.lib().wb_mesh_octree_bits(A.ptr(tris), A.ptr(cdf), tris.shape[0], n, level, seed, A.ptr(bits), A.stream())
    torch.cuda.synchronize()
    return bits.cpu().numpy().view(np.uint32), tris.cpu().numpy(), cdf.cpu().numpy()


def native(V, F, level, n, seed):
    return W.mesh_to_octree(torch.from_numpy(V).cuda(), torch.from_numpy(F).cuda(), level, n, seed=seed)


@pytest.mark.parametrize("case", [("noisy_sphere", 7, 1 << 20, 3), ("cube", 5, 300_001, 4), ("open", 7, 77_777, 0xFFFFFFFF)])
def test_bits_equal_restatement(case):
    name, level, n, seed = case
    V, F, _ = golden_case(name, level)
    bits, tris, cdf = kernel_bits(V, F, level, n, seed)
    assert np.array_equal(bits, R.sample_bits(tris, cdf, n, level, seed))


@pytest.mark.parametrize("level", sorted(N))
@pytest.mark.parametrize("name", MESHES)
def test_inside_limit_set_at_default_samples(name, level):
    V, F, refs = golden_case(name, level)
    lim = R.limit_set(V, F, level)
    for seed in (1, 2, 3):
        g = R.octree_cells(native(V, F, level, 10 ** 8, seed))
        assert not (g & ~lim).any(), int((g & ~lim).sum())
        assert g.sum() >= max(r.sum() for r in refs)          # 100 x more samples than the golden's: at least as many cells


@pytest.mark.parametrize("level", sorted(N))
@pytest.mark.parametrize("name", MESHES)
def test_reference_distribution(name, level):
    """At the golden's sample count the native octree cannot be told from the reference's (see distribution_bounds)."""
    V, F, refs = golden_case(name, level)
    lo, hi, sd = distribution_bounds(refs)
    for seed in (7, 8):
        g = R.octree_cells(native(V, F, level, N[level], seed))
        assert lo <= g.sum() <= hi, (int(g.sum()), lo, hi)
        assert max(int((g ^ r).sum()) for r in refs) <= sd, ([int((g ^ r).sum()) for r in refs], sd)


def test_well_formed_octree():
    V, F, _ = golden_case("torus", 7)
    level, n, seed = 7, 10 ** 6, 21
    octree = native(V, F, level, n, seed)
    assert octree.dtype == torch.uint8 and octree.is_cuda
    ml, pyramid, prefix = S.scan_octree(octree)
    assert ml == level
    pts = S.generate_points(octree, pyramid)
    finest = pts[int(pyramid[1, ml]):int(pyramid[1, ml]) + int(pyramid[0, ml])]
    g = bits_to_grid(kernel_bits(V, F, level, n, seed)[0], level)
    fn = finest.long().cpu().numpy()
    assert fn.shape[0] == g.sum() and g[fn[:, 0], fn[:, 1], fn[:, 2]].all()
    assert torch.equal(S.points_to_octree(finest, level), octree)
    blas = W.OctreeAS(octree)
    cells = (finest[:50].float() + 0.5) / 2 ** (level - 1) - 1.0
    pidx = blas.query(cells.cuda(), level).pidx
    assert torch.equal(pidx.long().cpu(), torch.arange(50) + int(pyramid[1, ml]))
    o = torch.tensor([[-3.0, 0.1, 0.05]], device="cuda").repeat(4, 1)
    d = torch.tensor([[1.0, 0.0, 0.0]], device="cuda").repeat(4, 1)
    rt = blas.raytrace(W.Rays(o, d, 0.0, 10.0), level)
    assert rt.ridx.numel() > 0


def test_reproducible():
    V, F, _ = golden_case("noisy_sphere", 5)
    a, b, c = native(V, F, 5, 10 ** 5, 9), native(V, F, 5, 10 ** 5, 9), native(V, F, 5, 10 ** 5, 10)
    assert torch.equal(a, b) and not torch.equal(a, c)
    # host inputs and int32 faces: the same octree
    assert torch.equal(W.mesh_to_octree(torch.from_numpy(V), torch.from_numpy(F).int(), 5, 10 ** 5, seed=9), a)
    # seed=None takes the seed from torch's default generator, and so does the install() replacement
    mod = types.ModuleType("wisp_b200_test_spc")
    fallback = []
    orig = lambda v, f, level, num_samples=100000000: fallback.append((level, v.dtype)) or "original"
    I._ORIG[(mod.__name__, "mesh_to_octree")] = (mod, orig)
    try:
        fn = I._mesh_to_octree(mod)
        outs = []
        for _ in range(2):
            torch.manual_seed(1234)
            outs.append(fn(torch.from_numpy(V).cuda(), torch.from_numpy(F).cuda(), 5, 10 ** 5))
        torch.manual_seed(1234)
        assert torch.equal(outs[0], outs[1]) and torch.equal(outs[0], W.mesh_to_octree(torch.from_numpy(V), torch.from_numpy(F), 5, 10 ** 5))
        for v, level in ((V, 0), (V, 11), (V.astype(np.float64), 5)):
            assert fn(torch.from_numpy(v).cuda(), torch.from_numpy(F).cuda(), level, 100) == "original"
        assert fallback == [(0, torch.float32), (11, torch.float32), (5, torch.float64)]
    finally:
        del I._ORIG[(mod.__name__, "mesh_to_octree")]


def test_64bit_counter_and_face_resolution():
    """2^32 samples in one call on two unit squares (total area 2) and an isolated triangle whose share is 2^-26, last in the CDF: its interval
    [1 - 2^-26, 1) holds no multiple of 2^-24, so only a uniform finer than 24 bits draws it (~64 expected draws, P(none) = e^-64).
    Its cell (deep inside one level-7 cell, far from the others) must be set, and no cell outside the limit set."""
    level = 7
    cell = 2.0 / 2 ** level
    c = (np.array([102, 101, 100]) + 0.5) * cell - 1.0
    leg = 2.0 ** -12                       # area leg^2 / 2 = 2^-25 against a total of 2: share 2^-26
    sq = np.array([[-0.5, -0.5, 0.0], [0.5, -0.5, 0.0], [-0.5, 0.5, 0.0], [0.5, 0.5, 0.0]])
    V = np.concatenate([sq + [0, 0, -0.2], sq + [0, 0, -0.6], [c, c + [leg, 0, 0], c + [0, leg, 0]]]).astype(np.float32)
    F = np.array([[0, 1, 2], [1, 3, 2], [4, 5, 6], [5, 7, 6], [8, 9, 10]])
    _, tris, cdf = kernel_bits(V, F, level, 1, 0)
    share = (cdf[5] - cdf[4]) / cdf[5]
    assert abs(share / 2 ** -26 - 1) < 1e-3 and np.floor((1 - share) * 2 ** 24) == 2 ** 24 - 1
    octree = native(V, F, level, 2 ** 32, 77)
    g = R.octree_cells(octree)
    assert g[102, 101, 100]
    assert not (g & ~R.limit_set(V, F, level)).any()
    assert not R.limit_set(V[:8], F[:4], level)[102, 101, 100]


def test_errors():
    V, F, _ = golden_case("cube", 5)
    v, f = torch.from_numpy(V).cuda(), torch.from_numpy(F).cuda()
    with pytest.raises(W.WispB200Error):
        W.mesh_to_octree(v, f[:0], 5)
    with pytest.raises(W.WispB200Error):
        W.mesh_to_octree(torch.zeros_like(v), f, 5)                # zero total area
    for level in (0, 11):
        with pytest.raises(W.WispB200Error):
            W.mesh_to_octree(v, f, level)
    with pytest.raises(W.WispB200Error):
        W.mesh_to_octree(v.double(), f, 5)
    with pytest.raises(W.WispB200Error):
        W.mesh_to_octree(v, f.float(), 5)
