"""GPU tests (-m gpu) of the kernels that decide which table rows and which cells a sample touches, through the C ABI and the
autograd functions, against tests/grid_index_reference.py:
  - wb_hashgrid_fwd bit for bit against the fp32 emulation (F 2 / 4 / 6 / 8, 1 to 16 levels, both sides of the dense / hashed
    boundary, coordinates on and beside the cube's faces, far outside, on cell faces and NaN, N*L around multiples of 256);
  - wb_hashgrid_bwd inside the float64 interval per table entry (heavy contention on one cell, skipped zero gradients,
    accumulation into a non-zero gradient table), and exactly the initial value where nothing is added;
  - wb_octree_build_bits / _coarse word for word against the exact masks, and the ensure_bits bounding box;
  - wb_prune_samples bit for bit (explicit u and the counter-based stream) and wb_prune_update with torch.max's NaN rule.
Each hash case prints one GRIDINDEX line: max |k - c| / r over the entries with r > 0 and the median radius."""
import ctypes as C
import zlib

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

import grid_index_reference as GR
import octree_reference as OR

f32 = np.float32


@pytest.fixture(scope="module")
def W():
    import wisp_b200
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return wisp_b200


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _special(res_list):
    """Coordinates at and beside +-1, far outside, NaN, and on the cell faces of every level (with their fp32 neighbours)."""
    one = f32(1.0)
    v = [0.0, -0.0, 1.0, -1.0, np.nextafter(one, f32(0)), np.nextafter(-one, f32(0)), np.nextafter(one, f32(2)),
         np.nextafter(-one, f32(-2)), 3.0, -3.0, 1e30, -1e30, np.nan]
    for r in res_list:
        k = np.arange(0, r + 1)
        faces = (2.0 * k / r - 1.0).astype(f32)
        v += list(faces[:: max(1, len(faces) // 16)]) + [faces[-2]]
    v = np.array(v, f32)
    v = np.concatenate([v, np.nextafter(v, f32(-2)), np.nextafter(v, f32(2))])
    return v


def _coords(rng, N, res_list):
    c = rng.uniform(-1.0, 1.0, (N, 3)).astype(f32)
    s = _special(res_list)
    m = min(N, 4 * len(s))
    c[:m] = s[rng.integers(0, len(s), (m, 3))]
    c[: min(N, len(s)), 0] = s[: min(N, len(s))]                       # every special value at least once on x
    return c


def _desc(W, table, res, bw, begin):
    return W._cabi.make_grid_desc(table, res, [int(b) for b in begin], 2 ** bw)


def _fwd(W, coords, table, res, bw, begin):
    A = W._cabi
    L, F = len(res), table.shape[1]
    c = dev(coords)
    feats = torch.full((c.shape[0], L * F), float("nan"), device="cuda")
    d = _desc(W, table, res, bw, begin)
    A.check(A.lib().wb_hashgrid_fwd(A.ptr(c), C.c_int64(c.shape[0]), C.byref(d), A.ptr(feats), A.stream()))
    torch.cuda.synchronize()
    return feats.cpu().numpy()


def _bwd(W, coords, go, table, gt0, res, bw, begin):
    A = W._cabi
    c, g, gt = dev(coords), dev(go), dev(gt0)
    d = _desc(W, table, res, bw, begin)
    A.check(A.lib().wb_hashgrid_bwd(A.ptr(c), C.c_int64(c.shape[0]), C.byref(d), A.ptr(g), A.ptr(gt), A.stream()))
    torch.cuda.synchronize()
    return gt.cpu().numpy()


def _report(tag, k, c, r):
    err = np.abs(k.astype(np.float64) - c)
    live = r > 0
    worst = float((err[live] / r[live]).max()) if live.any() else 0.0
    med = float(np.median(r[live])) if live.any() else 0.0
    print(f"GRIDINDEX {tag}: max|k-c|/r={worst:.3f} median_r={med:.3e} exact_entries={int((~live).sum())}")
    return worst


def _check_bwd(tag, got, gt0, c, r, k):
    assert np.isfinite(got).all()
    assert _report(tag, got, c, r) <= 1.0
    assert (np.abs(got.astype(np.float64) - c) <= r).all(), tag
    assert np.array_equal(got[k == 0].view(np.uint32), gt0[k == 0].view(np.uint32)), tag


def _geo(L, lo, hi):
    if L == 1:
        return [lo]
    b = np.exp((np.log(hi) - np.log(lo)) / (L - 1))
    return [int(np.floor(lo * b ** l)) for l in range(L)]


# name, resolutions, bitwidth, F, N
HASH = [
    ("f2_L16_bw19", _geo(16, 16, 512), 19, 2, 16 * 64 + 1),           # N*L = 256*64 + 16
    ("f2_L7_bw22", [16, 64, 128, 161, 162, 200, 512], 22, 2, 1463),  # 161 dense, 162 hashed; N*L = 256*40 + 1
    ("f4_L7_bw12", [2, 8, 15, 16, 17, 31, 64], 12, 4, 1),              # res 15 dense, 16^3 == 2^12 hashed
    ("f4_L7_bw12_big", [2, 8, 15, 16, 17, 31, 64], 12, 4, 37449),     # N*L = 262143 = 256*1024 - 1
    ("f6_L2_bw18", [63, 64], 18, 6, 128 * 51 + 1),                    # 63 dense, 64^3 == 2^18 hashed; N*L = 256*51 + 2
    ("f6_L16_bw8", _geo(16, 2, 40), 8, 6, 6000),                      # res 6 dense (216 < 256), 7 hashed
    ("f8_L1_bw8", [6], 8, 8, 256 * 7 + 1),                            # N*L = 256k + 1
    ("f8_L16_bw12", _geo(16, 4, 300), 12, 8, 8000),
    ("f2_L2_bw19_1M", [80, 81], 19, 2, (1 << 20) + 3),                # 80 dense, 81 hashed
]


@pytest.mark.parametrize("name,res,bw,F,N", HASH, ids=[h[0] for h in HASH])
def test_hashgrid_fwd_bit_exact_bwd_in_interval(W, name, res, bw, F, N):
    rng = np.random.default_rng(zlib.crc32(name.encode()))
    begin = GR.table_layout(res, bw)
    table = rng.standard_normal((int(begin[-1]), F)).astype(f32)
    coords = _coords(rng, N, res)
    got = _fwd(W, coords, dev(table), res, bw, begin)
    emu, cen, rad = GR.hashgrid_fwd(coords, table, res, bw)
    _report(name + " fwd", got, cen, rad)
    assert np.array_equal(got.view(np.uint32), emu.view(np.uint32)), name
    go = rng.standard_normal(emu.shape).astype(f32)
    go3 = go.reshape(N, len(res), F)
    go3[::5] = 0.0                                                    # whole rows zero: the float2 early exit / per-feature skip
    go3[1::7, :, 0] = 0.0                                             # one feature zero
    gt0 = np.zeros_like(table)
    gt0[::3] = rng.standard_normal(gt0[::3].shape).astype(f32)        # accumulate into a non-zero gradient table
    gt0[1::11] = -0.0
    got = _bwd(W, coords, go, dev(table), gt0, res, bw, begin)
    c, r, k = GR.hashgrid_bwd(coords, go, gt0, res, bw)
    _check_bwd(name + " bwd", got, gt0, c, r, k)


@pytest.mark.parametrize("F", [2, 4])
def test_hashgrid_bwd_one_cell_contention(W, F):
    """10^5 samples inside one cell of a dense level: 8 rows, 10^5 atomic adds each."""
    rng = np.random.default_rng(F)
    res, bw = [16], 14
    begin = GR.table_layout(res, bw)
    table = rng.standard_normal((int(begin[-1]), F)).astype(f32)
    lo = 2.0 * 5 / 16 - 1.0
    coords = (lo + rng.uniform(0.0, 2.0 / 16, (100000, 3))).astype(f32)
    coords = np.clip(coords, lo, np.nextafter(f32(lo + 2.0 / 16), f32(-2)))
    emu, cen, rad = GR.hashgrid_fwd(coords, table, res, bw)
    got = _fwd(W, coords, dev(table), res, bw, begin)
    assert np.array_equal(got.view(np.uint32), emu.view(np.uint32))
    go = rng.standard_normal(emu.shape).astype(f32)
    gt0 = np.zeros_like(table)
    got = _bwd(W, coords, go, dev(table), gt0, res, bw, begin)
    c, r, k = GR.hashgrid_bwd(coords, go, gt0, res, bw)
    assert (k > 0).sum() == 8 * F and k.max() == 100000
    _check_bwd(f"contention F={F}", got, gt0, c, r, k)


def test_hashgrid_dense_level_past_257_stays_in_range(W):
    """A dense level of res 258 (bitwidth 25): fl(res - 1 - 1e-5) == res - 1, so coordinates at +1 land on the last cell with
    weight 0 on its +1 corner.  The table is followed by NaN rows: a row read past the level would turn the feature into NaN."""
    rng = np.random.default_rng(258)
    res, bw, F = [258], 25, 2
    n = GR.level_rows(258, bw)
    assert GR.is_dense(258, bw) and n == 258 ** 3
    begin = GR.table_layout(res, bw)
    guard = 258 ** 2 + 258 + 2
    table = np.full((n + guard, F), np.nan, f32)
    table[:n] = rng.standard_normal((n, F)).astype(f32)
    ext = np.array([1.0, np.nextafter(f32(1), f32(0)), 2.0, np.nan, -1.0, 0.5], f32)
    coords = np.concatenate([np.stack(np.meshgrid(ext, ext, ext, indexing="ij"), -1).reshape(-1, 3), _coords(rng, 5000, res)])
    got = _fwd(W, coords, dev(table), res, bw, begin)
    emu, _, _ = GR.hashgrid_fwd(coords, table[:n], res, bw)
    assert np.isfinite(got).all()
    assert np.array_equal(got.view(np.uint32), emu.view(np.uint32))
    go = rng.standard_normal(emu.shape).astype(f32)
    gt0 = np.zeros((n + guard, F), f32)
    g = _bwd(W, coords, go, dev(table), gt0, res, bw, begin)
    assert np.array_equal(g[n:].view(np.uint32), gt0[n:].view(np.uint32))
    c, r, k = GR.hashgrid_bwd(coords, go, gt0[:n], res, bw)
    _check_bwd("dense res 258", g[:n], gt0[:n], c, r, k)


def test_hashgrid_interpolate_autograd(W):
    """ops.HashGridInterpolate end to end: forward bit for bit, table gradient in the interval, odd F and coords.requires_grad
    refused."""
    rng = np.random.default_rng(11)
    res, bw, F = [2, 8, 15, 16, 17, 31, 64], 12, 4
    begin = GR.table_layout(res, bw)
    table = rng.standard_normal((int(begin[-1]), F)).astype(f32)
    coords = _coords(rng, 3001, res)
    t = dev(table).requires_grad_(True)
    feats = W.ops.HashGridInterpolate.apply(dev(coords), torch.tensor(res), bw, len(res) - 1, t, torch.from_numpy(begin))
    emu, _, _ = GR.hashgrid_fwd(coords, table, res, bw)
    assert np.array_equal(feats.detach().cpu().numpy().view(np.uint32), emu.view(np.uint32))
    go = rng.standard_normal(emu.shape).astype(f32)
    feats.backward(dev(go))
    c, r, k = GR.hashgrid_bwd(coords, go, np.zeros_like(table), res, bw)
    _check_bwd("autograd", t.grad.cpu().numpy(), np.zeros_like(table), c, r, k)
    with pytest.raises(Exception, match="multiple of 2"):
        W.ops.HashGridInterpolate.apply(dev(coords), torch.tensor(res), bw, 0, dev(table[:, :3]), torch.from_numpy(begin))
    with pytest.raises(W._cabi.WispB200Error, match="coords"):
        W.ops.HashGridInterpolate.apply(dev(coords).requires_grad_(True), torch.tensor(res), bw, 0, t, torch.from_numpy(begin))


# ---- occupancy bitmasks ---------------------------------------------------------------------------------------------------
OCTREES = ["lego6", "corner_lo4", "corner_hi4", "corner_hi10", "dense3", "dense5", "checker4", "random8", "random10", "lines9",
           "lines10", "faces5"]


def _build_bits(W, pts, level, n=None):
    A = W._cabi
    bits = torch.zeros((8 ** level + 31) // 32, dtype=torch.int32, device="cuda")
    p = dev(pts.astype(np.int16))
    n = pts.shape[0] if n is None else n
    A.check(A.lib().wb_octree_build_bits(A.ptr(p), C.c_int64(n), C.c_int32(level), A.ptr(bits), A.stream()))
    return bits.cpu().numpy().view(np.uint32)


def _build_coarse(W, pts, level, cl, n=None):
    A = W._cabi
    cb = torch.zeros((8 ** cl + 31) // 32, dtype=torch.int32, device="cuda")
    p = dev(pts.astype(np.int16))
    n = pts.shape[0] if n is None else n
    A.check(A.lib().wb_octree_build_coarse(A.ptr(p), C.c_int64(n), C.c_int32(level), C.c_int32(cl), A.ptr(cb), A.stream()))
    return cb.cpu().numpy().view(np.uint32)


@pytest.mark.parametrize("name", OCTREES)
def test_octree_bits_and_coarse_are_exact(W, name):
    pts, level = OR.octree_points(name)
    assert np.array_equal(_build_bits(W, pts, level), GR.build_bits(pts, level)), name
    for cl in range(1, level):
        assert np.array_equal(_build_coarse(W, pts, level, cl), GR.build_coarse(pts, level, cl)), (name, cl)


def test_octree_bits_without_points(W):
    """num_points = 0 (an empty level slice of the points tensor, as ensure_bits passes it): nothing is set."""
    pts = np.full((1, 3), 3, np.int16)
    assert not _build_bits(W, pts, 4, n=0).any()
    assert not _build_coarse(W, pts, 4, 2, n=0).any()


@pytest.mark.parametrize("name", ["lego6", "corner_hi4", "random8", "faces5", "dense3"])
def test_ensure_bits_matches_exact(W, name):
    from oracle import oracle as O
    pts, level = OR.octree_points(name)
    spc = O.octree_to_spc(O.points_to_octree(pts, level))
    blas = W.OctreeAS(dev(spc.octree))
    t = W.ops.octree_tensors(blas)
    t.ensure_bits(level)
    torch.cuda.synchronize()
    s, c = int(t.pyramid[1, level]), int(t.pyramid[0, level])
    lvl = t.points[s:s + c].cpu().numpy()
    assert t.bits_level == level and np.array_equal(t.bits.cpu().numpy().view(np.uint32), GR.build_bits(lvl, level))
    cl = min(level - 1, W.ops.COARSE_LEVEL)
    if cl >= 2:
        assert t.coarse_level == cl and np.array_equal(t.coarse.cpu().numpy().view(np.uint32), GR.build_coarse(lvl, level, cl))
    lo, hi = GR.bbox(pts, level)
    assert t.bbox == (lo, hi)


# ---- prune ------------------------------------------------------------------------------------------------------------------
def _prune_samples(W, pts, level, u, seed):
    A = W._cabi
    N = pts.shape[0]
    p = dev(pts.astype(np.int16))
    uu = None if u is None else dev(u)
    samples = torch.empty((N, 3), device="cuda"); dirs = torch.empty((N, 3), device="cuda")
    rec_t = torch.full((N,), float("nan"), device="cuda"); rec_ray = torch.full((N,), -1, dtype=torch.int32, device="cuda")
    A.check(A.lib().wb_prune_samples(A.ptr(p), C.c_int64(N), C.c_int32(level), A.ptr(uu), C.c_uint32(seed), A.ptr(samples), A.ptr(dirs),
                                     A.ptr(rec_t), A.ptr(rec_ray), A.stream()))
    torch.cuda.synchronize()
    return samples.cpu().numpy(), dirs.cpu().numpy(), rec_t.cpu().numpy(), rec_ray.cpu().numpy()


@pytest.mark.parametrize("level", [1, 7, 15])
@pytest.mark.parametrize("N", [1, 256 * 41 + 1])
@pytest.mark.parametrize("seed", [0, 0xC0FFEE])
def test_prune_samples(W, level, N, seed):
    rng = np.random.default_rng(level * 7 + N)
    pts = rng.integers(0, 1 << level, (N, 3)).astype(np.int16)
    pts[0] = (1 << level) - 1
    stream = GR.prune_stream(seed, N)
    explicit = rng.random((N, 3)).astype(f32)
    explicit[-1] = np.nextafter(f32(1), f32(0))
    for u in (None, explicit):
        s, d, t, r = _prune_samples(W, pts, level, u, seed)
        want = GR.prune_samples(pts, level, stream[:, :3] if u is None else u)
        assert np.array_equal(s.view(np.uint32), want.view(np.uint32))
        assert (t == 0).all() and np.array_equal(r, np.arange(N))
        norm = np.linalg.norm(d.astype(np.float64), axis=1)
        assert (np.abs(norm - 1.0) <= 2 * 2.0 ** -23).all()
        assert np.array_equal(d[:, 2], (f32(1) - f32(2) * stream[:, 3]).astype(f32))      # z = 1 - 2 u0 of the same stream


def _prune_update(W, dens, occ0, decay, md):
    A = W._cabi
    N = dens.shape[0]
    shaded = np.zeros((N, 4), f32); shaded[:, 3] = dens
    sh, occ = dev(shaded), dev(occ0.copy())
    keep = torch.full((N,), 7, dtype=torch.uint8, device="cuda")
    A.check(A.lib().wb_prune_update(A.ptr(sh), C.c_int64(N), C.c_float(decay), C.c_float(md), A.ptr(occ), A.ptr(keep), A.stream()))
    torch.cuda.synchronize()
    return occ.cpu().numpy(), keep.cpu().numpy()


@pytest.mark.parametrize("decay", [0.0, 0.6, 1.0])
def test_prune_update(W, decay):
    nan, inf = np.nan, np.inf
    md = 0.01
    dens = np.array([nan, 0.3, nan, inf, -inf, -inf, md, 0.2, 0.5, 0.0, 1e-3, 0.7], f32)
    occ0 = np.array([0.9, nan, nan, 0.1, 0.9, 0.0, 0.0, 0.3, 0.5, 0.0, 0.02, 0.1], f32)
    rng = np.random.default_rng(1)
    N = 256 * 9 + 1
    d = np.concatenate([dens, rng.uniform(-0.1, 0.1, N).astype(f32)])
    o = np.concatenate([occ0, rng.uniform(0.0, 0.1, N).astype(f32)])
    got, keep = _prune_update(W, d, o, decay, md)
    want, wkeep = GR.prune_update(d, o, decay, md)
    assert np.array_equal(np.isnan(got), np.isnan(want))
    assert np.array_equal(got[~np.isnan(want)], want[~np.isnan(want)])
    assert np.array_equal(keep.astype(bool), wkeep) and set(np.unique(keep)) <= {0, 1}
    assert np.isnan(got[:3]).all() and not keep[:3].any()               # NaN density or occupancy: stored, not kept
    assert got[6] == f32(md) and not keep[6]                            # exactly min_density: not kept


def _prune_nef(W):
    import os
    from golden_util import load_case
    from gpu_util import nef_from_oracle
    g, onef, spc = load_case(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "prune.npz"))
    nef, _ = nef_from_oracle(onef, spc)
    nef.prune_density_decay, nef.prune_min_density = float(g["decay"]), float(g["min_density"])
    nef.grid.occupancy = torch.from_numpy(g["occupancy0"].copy())
    return nef, g


def test_prune_field_repeatable_and_nan_density(W):
    """prune_field twice from the same state with the same seed: the same occupancy bits and octree.  A NaN bias in the density
    decoder's output: the shade kernel's density activation fmaxf(sigma, 0) turns the NaN into 0 before wb_prune_update sees it
    (torch.relu would keep it, see DESIGN.md), so each cell's occupancy becomes max(0, occupancy * decay)."""
    a, g = _prune_nef(W)
    b, _ = _prune_nef(W)
    W.ops.prune_field(a, seed=9); W.ops.prune_field(b, seed=9)
    assert np.array_equal(a.grid.occupancy.cpu().numpy().view(np.uint32), b.grid.occupancy.cpu().numpy().view(np.uint32))
    assert np.array_equal(a.grid.blas.octree.cpu().numpy(), b.grid.blas.octree.cpu().numpy())
    c, _ = _prune_nef(W)
    with torch.no_grad():
        c.decoder_density.lout.bias[0] = float("nan")
    octree0 = c.grid.blas.octree.clone()
    W.ops.prune_field(c, seed=9)
    occ = c.grid.occupancy.cpu().numpy()
    want, keep = GR.prune_update(np.zeros_like(g["occupancy0"]), g["occupancy0"], float(g["decay"]), float(g["min_density"]))
    assert np.array_equal(occ, want)
    if not keep.any():
        assert torch.equal(c.grid.blas.octree, octree0)
