"""The VQAD codebook kernels (wb_codebook_rows_fwd / _bwd) through the C ABI, the unfused octree-grid forward
(wb_octree_interp_fwd) and CodebookOctreeGrid end to end, against the float64 references tests/codebook_reference.py and
oracle/sdf_reference.py.

Covers what the one small golden (K 16, F 4, <= 485 rows) cannot reach:
  - K = 1 .. 1024 on both sides of every instantiation boundary (KPL 8 / 32 at K 256 / 257, K below, at and above a warp), F 1 .. 32;
  - rows 1, 7, the forward's grid cap (8 rows x 16 CTAs x SMs) +- 1 and ~40 000 (a second grid-stride pass); for the backward
    several rows per warp past its cap (8 x 2 x SMs), so the per-warp dE row is reused;
  - logits N(0, 0.01) (nerf_codebook's init), N(0, 1), N(0, 30) (y underflows), exact ties in the same lane / another lane /
    another slot, rows of equal logits and rows at or below -3e38 (argmax 0 for equal rows, never out of [0, K));
  - argmax_out NULL and set, training and eval; E bit-exact dictionary[argmax] in both modes;
  - dE rows that are zero (skipped: g_logits stays 0), zero in feature 0 only, non-zero only in feature F-1, thousands of rows
    sharing one argmax, a pre-filled g_dictionary, both sides of the 48 KiB shared-memory opt-in;
  - wb_octree_interp_fwd bit-exact with sdf_reference.features (half_features on and off, F 1 .. 64, 'cat' / 'sum', every
    lod_idx, base_lod 0 and > 0, points outside the cube, on cell faces, in descents that stop early);
  - CodebookOctreeGrid at the nerf_codebook shape, bitwidth 8 and bitwidth 10 / F 32: features, logit and dictionary gradients.
Outputs are pre-filled with sentinels past `rows`.  Each interval check prints one CMPREPORT line: max|k - c| / r and the median
radius."""

import numpy as np
import pytest
import torch

import codebook_reference as CB
from oracle import sdf_reference as S
from sdf_shapes import case_of, points

pytestmark = pytest.mark.gpu
SENTINEL, ISENTINEL = 7.25, -5
KS = (1, 2, 16, 31, 32, 33, 255, 256, 257, 512, 1000, 1024)
FS = (1, 4, 5, 31, 32)


@pytest.fixture(scope="module")
def W():
    import wisp_b200
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return wisp_b200


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _sms():
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


def _check(name, k, c, r):
    k, c, r = np.broadcast_arrays(*(np.asarray(x, np.float64) for x in (k, c, r)))
    d = np.abs(k - c)
    ok = d <= r                                                          # NaN fails
    ratio = np.where(r > 0, d / np.where(r > 0, r, 1.0), np.where(d > 0, np.inf, 0.0))
    ratio = float(np.max(np.where(np.isnan(d), np.inf, ratio), initial=0.0))
    print(f"CMPREPORT {name}: max|k-c|/r={ratio:.3g} median_r={float(np.median(r)) if r.size else 0.0:.3g}")
    bad = np.argwhere(~ok)
    assert ok.all(), (name, int((~ok).sum()), bad[:4].tolist(), k[tuple(bad[0])], c[tuple(bad[0])], r[tuple(bad[0])])


def _fwd(W, lg, dc, training, with_am):
    """wb_codebook_rows_fwd on device logits [rows, K] / dictionary [K, F] -> (E, argmax or None) on the host."""
    A = W._cabi
    rows, K = lg.shape
    F = dc.shape[1]
    E = torch.full((rows + 3, F), SENTINEL, device="cuda")
    am = torch.full((rows + 3,), ISENTINEL, dtype=torch.int32, device="cuda") if with_am else None
    A.lib().wb_codebook_rows_fwd(A.ptr(lg), A.ptr(dc), rows, K, F, int(training),
                                 A.ptr(E), A.ptr(am), A.stream())
    assert bool((E[rows:] == SENTINEL).all()), "E rows past `rows` written"
    if am is not None:
        assert bool((am[rows:] == ISENTINEL).all()), "argmax_out past `rows` written"
    return E[:rows].cpu().numpy(), None if am is None else am[:rows].cpu().numpy()


def _bwd(W, lg, dc, dE, g0):
    """wb_codebook_rows_bwd with zeroed g_logits and g_dictionary = g0 -> (g_logits, g_dictionary) on the host."""
    A = W._cabi
    rows, K = lg.shape
    F = dc.shape[1]
    gl = torch.zeros((rows + 2, K), device="cuda"); gl[rows:] = SENTINEL
    gd = torch.full((K + 1, F), SENTINEL, device="cuda"); gd[:K] = dev(g0)
    A.lib().wb_codebook_rows_bwd(A.ptr(lg), A.ptr(dc), A.ptr(dev(dE)), rows, K, F,
                                 A.ptr(gl), A.ptr(gd), A.stream())
    assert bool((gl[rows:] == SENTINEL).all()) and bool((gd[K:] == SENTINEL).all()), "written past the buffers"
    return gl[:rows].cpu().numpy(), gd[:K].cpu().numpy()


def _fwd_all(W, name, L, D, modes=((0, 0), (0, 1), (1, 0), (1, 1))):
    lg, dc = dev(L), dev(D)
    am_ref = CB.first_max(L)
    for training, with_am in modes:
        E, am = _fwd(W, lg, dc, training, with_am)
        _check(f"{name} t{training} am{with_am} E", E, D[am_ref], 0.0)         # E = dictionary[argmax] bit for bit in both modes
        if am is not None:
            assert np.array_equal(am, am_ref), (name, training, np.flatnonzero(am != am_ref)[:4])


# ---- wb_codebook_rows_fwd --------------------------------------------------------------------------------------------------
EXTREME_KS = (1, 2, 16, 33, 256, 257, 1024)


@pytest.mark.parametrize("K", EXTREME_KS)
def test_rows_fwd_extreme_logits_training(W, K):
    """Rows at or below -3e38 in training mode with argmax_out set: the argmax is the first maximiser (0 for a row of equal
    logits) and E = dictionary[argmax], not NaN.  This path only compares k with the argmax, whatever its value."""
    rng = np.random.default_rng(K)
    L = CB.make_logits(300, K, "extreme", rng)
    D = rng.standard_normal((K, 5)).astype(np.float32)
    rf = CB.rows_fwd(L, D, True)
    eq = (L == L[:, :1]).all(1)
    assert eq.any() and np.all(rf.am[eq] == 0) and np.allclose(rf.y[eq], 1.0 / K, rtol=1e-6)
    _fwd_all(W, f"extreme K{K}", L, D, modes=((1, 1),))


@pytest.mark.parametrize("K", EXTREME_KS)
def test_rows_fwd_extreme_logits_eval(W, K):
    rng = np.random.default_rng(K)
    L = CB.make_logits(300, K, "extreme", rng)
    D = rng.standard_normal((K, 5)).astype(np.float32)
    _fwd_all(W, f"extreme K{K}", L, D)


@pytest.mark.parametrize("K", KS)
def test_rows_fwd(W, K):
    cap = 8 * CB.FWD_CTAS_PER_SM * _sms()
    rows = (1, 7, cap - 1, cap + 1, 40000 if K <= 256 else 300)
    ki = KS.index(K)
    for ri, regime in enumerate(("init", "unit", "wide", "ties", "equal")):
        R = rows[(ri + ki) % len(rows)]
        rng = np.random.default_rng(1000 * ki + ri)
        L = CB.make_logits(R, K, regime, rng)
        for F in FS:                                                     # argmax_out NULL at the first F, set at every F
            D = rng.standard_normal((K, F)).astype(np.float32)
            _fwd_all(W, f"K{K} F{F} R{R} {regime}", L, D, modes=((0, 0), (0, 1), (1, 0), (1, 1)) if F == FS[0] else ((0, 1), (1, 1)))


# ---- wb_codebook_rows_bwd --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("K", KS)
def test_rows_bwd(W, K):
    cap = 8 * CB.BWD_CTAS_PER_SM * _sms()
    ki = KS.index(K)
    for fi, F in enumerate(FS):
        if F < 31 and K <= 256:
            R = 3 * cap + 5                                              # three or four rows per warp
        elif F == 1:
            R = 2 * cap + 5
        elif K <= 64:
            R = cap + 33
        else:
            R = 7 if F in (4, 31) else 300
        regime = CB.REGIMES[(fi + ki) % len(CB.REGIMES)]
        rng = np.random.default_rng(100 * ki + fi)
        L = CB.make_logits(R, K, regime, rng)
        D = rng.standard_normal((K, F)).astype(np.float32)
        dE = CB.make_dE(R, F, rng)
        g0 = rng.standard_normal((K, F)).astype(np.float32) if fi % 2 else np.zeros((K, F), np.float32)
        gl, gd = _bwd(W, dev(L), dev(D), dE, g0)
        ref = CB.rows_bwd(L, D, dE, None, g0)
        name = f"K{K} F{F} R{R} {regime} smem{'>' if CB.bwd_smem(K, F) > CB.SMEM_DEFAULT else '<='}48K"
        assert np.all(gl[ref.skipped] == 0.0), name
        _check(f"{name} g_logits", gl, ref.g_logits, ref.g_logits_r)
        _check(f"{name} g_dict", gd, ref.g_dict, ref.g_dict_r)
        assert np.all(gd[ref.n == 0] == g0[ref.n == 0]), name            # entries no row selected keep their value exactly


# ---- wb_octree_interp_fwd --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("F", (1, 3, 5, 16, 32, 64))
@pytest.mark.parametrize("ms", ("cat", "sum"))
def test_octree_interp_fwd_bit_exact(W, F, ms):
    """OctreeGrid.interpolate = sdf_reference.features bit for bit (radius 0): base_lod 3 (level 5, 3 LODs) and base_lod 0
    (level 3, 4 LODs), half_features on and off, every lod_idx."""
    rng = np.random.default_rng(F)
    for level, nl in ((5, 3), (3, 4)):
        case = case_of(level, nl, 1, "sum")                              # the octree; features of width F drawn here
        feats = [(rng.standard_normal((f.shape[0], F)) * 0.05).astype(np.float32) for f in case["feats"]]
        blas = W.OctreeAS(dev(case["octree"]))
        grid = W.OctreeGrid(blas, feature_dim=F, num_lods=nl, multiscale_type=ms, feature_std=0.0).cuda()
        assert grid.base_lod == case["active_lods"][0] and np.array_equal(grid.trinkets.cpu().numpy(), case["trinkets"])
        with torch.no_grad():
            for f, ref in zip(grid.features, feats):
                f.copy_(dev(ref))
        coords, _ = points(case, 3000, seed=F + level)
        c = dev(coords)
        for half in (True, False):
            grid.half_features = half
            field = S.Field(case["spc"], case["trinkets"], feats, grid.base_lod, ms, [], [], 1, 0, half)
            for lod in range(nl):
                with torch.no_grad():
                    got = grid.interpolate(c, lod).cpu().numpy()
                fc, fr, _, _ = S.features(field, coords, lod + 1)
                assert not fr.any()
                _check(f"octree fwd F{F} {ms} base{grid.base_lod} half{int(half)} lod{lod}", got, fc, fr)


# ---- CodebookOctreeGrid end to end -------------------------------------------------------------------------------------------
# name: (octree level, num_lods, feature_dim, multiscale, codebook_bitwidth)
GRID_SHAPES = {"nerf_codebook": (6, 4, 5, "sum", 4), "bw8": (6, 4, 8, "cat", 8), "bw10_f32": (4, 3, 32, "cat", 10)}


@pytest.mark.parametrize("name", list(GRID_SHAPES))
def test_codebook_grid_end_to_end(W, name):
    level, nl, F, ms, bw = GRID_SHAPES[name]
    case = case_of(level, nl, 1, "sum")                                  # the octree only
    blas = W.OctreeAS(dev(case["octree"]))
    torch.manual_seed(0)
    grid = W.CodebookOctreeGrid(blas, feature_dim=F, num_lods=nl, multiscale_type=ms, feature_std=0.01, codebook_bitwidth=bw).cuda()
    base = grid.base_lod
    assert base == case["active_lods"][0] and np.array_equal(grid.trinkets.cpu().numpy(), case["trinkets"])
    logits = [f.detach().cpu().numpy() for f in grid.features]
    dicts = [d.detach().cpu().numpy() for d in grid.dictionary]
    coords, _ = points(case, 2000, seed=level)
    c = dev(coords)
    rng = np.random.default_rng(bw)
    for lod in ((1, nl - 1) if name == "nerf_codebook" else (nl - 1,)):
        tag = f"{name} lod{lod}"
        nlu = lod + 1
        # training: E from ops.CodebookRows (deterministic: no atomics, a fixed butterfly), the blend over it bit for bit
        grid.train()
        for p in list(grid.features) + list(grid.dictionary):
            p.grad = None
        feats = grid.interpolate(c, lod)
        E = [W.ops.CodebookRows.apply(grid.features[i], grid.dictionary[i], True).detach().cpu().numpy() for i in range(nlu)]
        for i in range(nlu):
            assert np.array_equal(E[i], CB.rows_fwd(logits[i], dicts[i], True).E), (tag, i)
        field = S.Field(case["spc"], case["trinkets"], E, base, ms, [], [], 1, 0, False)
        fc, fr, _, _ = S.features(field, coords, nlu)
        _check(f"{tag} train feats", feats.detach().cpu().numpy(), fc, fr)
        go = rng.standard_normal(tuple(feats.shape)).astype(np.float32)
        feats.backward(dev(go))
        dE = S.interp_backward(field, coords, go, lod)
        for i in range(nlu):
            ref = CB.rows_bwd(logits[i], dicts[i], *dE[i])
            _check(f"{tag} LOD{i} g_logits", grid.features[i].grad.cpu().numpy(), ref.g_logits, ref.g_logits_r)
            _check(f"{tag} LOD{i} g_dict", grid.dictionary[i].grad.cpu().numpy(), ref.g_dict, ref.g_dict_r)
        for i in range(nlu, nl):
            assert grid.features[i].grad is None and grid.dictionary[i].grad is None
        # eval: dictionary[argmax]; the dictionary gradient through index_add_, none for the logits
        grid.eval()
        for p in list(grid.features) + list(grid.dictionary):
            p.grad = None
        feats = grid.interpolate(c, lod)
        Ev = [CB.rows_fwd(logits[i], dicts[i], False).E for i in range(nlu)]
        field = S.Field(case["spc"], case["trinkets"], Ev, base, ms, [], [], 1, 0, False)
        fc, fr, _, _ = S.features(field, coords, nlu)
        _check(f"{tag} eval feats", feats.detach().cpu().numpy(), fc, fr)
        feats.backward(dev(go))
        dE = S.interp_backward(field, coords, go, lod)
        for i in range(nlu):
            assert grid.features[i].grad is None, (tag, i)
            ref = CB.rows_bwd(logits[i], dicts[i], *dE[i], with_logits=False)
            _check(f"{tag} LOD{i} eval g_dict", grid.dictionary[i].grad.cpu().numpy(), ref.g_dict, ref.g_dict_r)
