"""tests/codebook_reference.py on the CPU: with rounding off it is CodebookOctreeGrid's own float64 arithmetic (a torch autograd
restatement of codebook_grid.py:103-172 and, where the reference checkout exists, the reference class itself); its fp32 centre
reproduces tests/golden/codebook.npz; fp32 emulations of wb_codebook_rows_fwd / _bwd with any summation order and expf off by up
to 2 ulp land inside its intervals, mutated emulations outside; and the radii stay tight."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import codebook_reference as CB
from oracle import oracle as O
from oracle import octree_grid as OG
from oracle import sdf_reference as S
from sdf_shapes import case_of

REF_WISP = "/root/reference/wisp"
f64 = torch.float64


def _cells(spc, trinkets, base_lod, coords, nl, coef):
    """S.Cells with the trilinear coefficients of `coef(coords, points, level)`."""
    pidx = O.query(spc, coords, base_lod + nl - 1, with_parents=True)[:, base_lod:]
    ok, tk, cf = [], [], []
    for k in range(nl):
        o = pidx[:, k] >= 0
        p = pidx[o, k].astype(np.int64)
        ok.append(o); tk.append(trinkets[p].astype(np.int64))
        cf.append(np.asarray(coef(coords[o], spc.points[p], base_lod + k), np.float64))
    return S.Cells(ok, tk, cf)


def restatement(logits, dicts, cl, ms, training, go):
    """codebook_grid.py:103-172 in float64 torch, per (sample, corner): softmax, argmax of y_soft, scatter, straight-through keys,
    dictionary product (training) or dictionary[argmax] (eval), trilinear blend, 'cat' / 'sum' -> (feats, g_logits, g_dict)."""
    nl = len(cl.ok)
    N = cl.ok[0].shape[0]
    lg = [torch.tensor(np.asarray(l, np.float64), requires_grad=True) for l in logits]
    dc = [torch.tensor(np.asarray(d, np.float64), requires_grad=True) for d in dicts]
    F = dc[0].shape[1]
    feats = []
    for k in range(nl):
        idx = torch.from_numpy(cl.tk[k])
        if training:
            lo = lg[k][idx]
            y_soft = torch.softmax(lo, -1)
            index = y_soft.max(-1, keepdim=True)[1]
            y_hard = torch.zeros_like(lo).scatter_(-1, index, 1.0)
            keys = y_hard - y_soft.detach() + y_soft
            corner = (dc[k][None, None] * keys[..., None]).sum(-2)
        else:
            corner = dc[k][torch.max(lg[k][idx], dim=-1)[1]]
        blend = (corner * torch.from_numpy(cl.cf[k])[..., None]).sum(-2)
        fs = torch.zeros(N, F, dtype=f64).index_put((torch.from_numpy(cl.ok[k]),), blend)
        feats.append(fs)
    out = torch.stack(feats, -2).sum(-2) if (ms == "sum" and nl > 1) else torch.cat(feats, -1)
    (out * torch.from_numpy(np.asarray(go, np.float64))).sum().backward()
    grad = lambda t: np.zeros(t.shape) if t.grad is None else t.grad.numpy()
    return out.detach().numpy(), [grad(t) for t in lg], [grad(t) for t in dc], [t.grad is None for t in lg]


def pipeline(spc, trinkets, base_lod, logits, dicts, coords, ms, training, go, exact, cl=None):
    """The reference's route: rows_fwd per LOD, the blend (S.features) over E, S.interp_backward, rows_bwd."""
    nl = len(logits)
    rows = [CB.rows_fwd(l, d, training, exact) for l, d in zip(logits, dicts)]
    field = S.Field(spc, trinkets, [r.E for r in rows], base_lod, ms if nl > 1 else "cat", [], [], 1, 0, False)
    fc = S.features(field, coords, nl, exact, cl)[0]
    dE = S.interp_backward(field, coords, go, nl - 1, exact)
    bw = [CB.rows_bwd(l, d, c, r, exact=exact) for l, d, (c, r) in zip(logits, dicts, dE)]
    return rows, fc, dE, bw


def _close(a, b, what, tol=1e-12):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    scale = max(float(np.abs(b).max(initial=0.0)), 1e-300)
    err = float(np.abs(a - b).max(initial=0.0))
    assert err <= tol * scale, (what, err, scale)


def _case(K, ms, seed):
    c = case_of(4, 3, 4, ms)
    rng = np.random.default_rng(seed)
    F = 5
    logits = [rng.standard_normal((f.shape[0], K)) for f in c["feats"]]
    dicts = [rng.standard_normal((K, F)) for _ in c["feats"]]
    from sdf_shapes import points
    coords, _ = points(c, 240, seed=seed)
    return c, logits, dicts, coords.astype(np.float32)


@pytest.mark.parametrize("K", [1, 16, 256, 257, 1024])
@pytest.mark.parametrize("ms", ["sum", "cat"])
def test_exact_reference_is_the_float64_operation(K, ms):
    c, logits, dicts, coords = _case(K, ms, seed=K)
    spc, tr, base = c["spc"], c["trinkets"], c["active_lods"][0]
    for lod in (2, 0):
        nl = lod + 1
        cl = S.cells(S.Field(spc, tr, [np.zeros((1, 1))] * nl, base, ms, [], [], 1, 0, False), coords, nl)
        for training in (True, False):
            go = np.random.default_rng(lod).standard_normal((coords.shape[0], 5 if (ms == "sum" and nl > 1) else 5 * nl))
            rows, fc, _, bw = pipeline(spc, tr, base, logits[:nl], dicts[:nl], coords, ms, training, go, True, cl)
            out, g_lg, g_dc, none = restatement(logits[:nl], dicts[:nl], cl, ms, training, go)
            _close(fc, out, ("feats", K, ms, lod, training))
            for k in range(nl):
                _close(bw[k].g_dict, g_dc[k], ("g_dict", K, ms, lod, training, k))
                if training:
                    _close(bw[k].g_logits, g_lg[k], ("g_logits", K, ms, lod, training, k))
                    assert np.all(rows[k].y.argmax(1) == rows[k].am)
                else:
                    assert none[k]                                           # eval: the logits get no gradient


_REF_SCRIPT = r"""
import sys, warnings
warnings.filterwarnings("ignore")
sys.path.insert(0, ROOT)
import numpy as np, torch
from oracle import ref_import
ref_import.install()
from wisp.accelstructs import OctreeAS
from wisp.models.grids import CodebookOctreeGrid
torch.set_default_dtype(torch.float64)
a = np.load(IN)
out = {}
for ms in ("sum", "cat"):
    blas = OctreeAS(torch.from_numpy(a["octree"]))
    grid = CodebookOctreeGrid(blas, feature_dim=5, num_lods=3, interpolation_type='linear', multiscale_type=ms, feature_std=1.0,
                              codebook_bitwidth=int(a["bw"]))
    for i in range(3):
        grid.features[i].data = torch.from_numpy(a[f"logits{i}"]).clone(); grid.dictionary[i].data = torch.from_numpy(a[f"dict{i}"]).clone()
    coords = torch.from_numpy(a["coords"]).double()
    out[f"{ms}_trinkets"] = grid.trinkets.numpy(); out[f"{ms}_base"] = np.int64(grid.base_lod)
    for mode in ("train", "eval"):
        getattr(grid, mode)()
        for lod in (2, 0):
            for p in list(grid.features) + list(grid.dictionary):
                p.grad = None
            f = grid.interpolate(coords, lod)
            (f * torch.from_numpy(a[f"go_{ms}_{lod}"])).sum().backward()
            key = f"{ms}_{mode}_{lod}"
            out[key + "_feats"] = f.detach().numpy()
            for i in range(lod + 1):
                g = grid.features[i].grad
                out[key + f"_glogits{i}"] = np.zeros(0) if g is None else g.numpy()
                out[key + f"_gdict{i}"] = grid.dictionary[i].grad.numpy()
np.savez(OUT, **out)
print("REF-OK")
"""


@pytest.mark.skipif(not os.path.isdir(REF_WISP), reason="needs the reference checkout")
@pytest.mark.parametrize("bw", [0, 4, 8, 10])
def test_reference_class_in_float64(tmp_path, bw):
    """The unmodified CodebookOctreeGrid (imported on CPU through oracle/ref_import.py, in a subprocess because the import stubs
    are process-wide) run in float64 equals the restatement above to 1e-12, in training and eval mode, lod_idx 2 and 0."""
    g = np.load(os.path.join(os.path.dirname(__file__), "golden", "codebook.npz"))
    oct_np = g["octree"]
    spc = O.octree_to_spc(oct_np)
    _, pyr, trinkets, _ = OG.make_trilinear_spc(spc)
    level = int(g["level"]); base = level - 2
    rng = np.random.default_rng(bw)
    K = 2 ** bw
    inp = dict(octree=oct_np, bw=np.int64(bw), coords=g["sum_coords"].astype(np.float64))
    for i in range(3):
        inp[f"logits{i}"] = rng.standard_normal((int(pyr[0, base + i]) + 1, K)); inp[f"dict{i}"] = rng.standard_normal((K, 5))
    for ms in ("sum", "cat"):
        for lod in (2, 0):
            inp[f"go_{ms}_{lod}"] = rng.standard_normal((360, 5 if (ms == "sum" and lod > 0) else 5 * (lod + 1)))
    np.savez(tmp_path / "in.npz", **inp)
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    code = _REF_SCRIPT.replace("ROOT", repr(root)).replace("IN", repr(str(tmp_path / "in.npz"))).replace("OUT", repr(str(tmp_path / "out.npz")))
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "REF-OK" in r.stdout, (r.stdout[-500:], r.stderr[-2000:])
    out = np.load(tmp_path / "out.npz")
    coords = g["sum_coords"]
    for ms in ("sum", "cat"):
        assert np.array_equal(out[f"{ms}_trinkets"], trinkets) and int(out[f"{ms}_base"]) == base
        for mode in ("train", "eval"):
            for lod in (2, 0):
                nl = lod + 1
                cl = _cells(spc, trinkets, base, coords, nl, OG.trilinear_coeffs)
                logits, dicts = [inp[f"logits{i}"] for i in range(nl)], [inp[f"dict{i}"] for i in range(nl)]
                f, g_lg, g_dc, none = restatement(logits, dicts, cl, ms, mode == "train", inp[f"go_{ms}_{lod}"])
                key = f"{ms}_{mode}_{lod}"
                _close(out[key + "_feats"], f, key)
                for i in range(nl):
                    _close(out[key + f"_gdict{i}"], g_dc[i], (key, "gdict", i))
                    if mode == "train":
                        _close(out[key + f"_glogits{i}"], g_lg[i], (key, "glogits", i))
                    else:
                        assert out[key + f"_glogits{i}"].size == 0 and none[i]


@pytest.mark.parametrize("ms", ["sum", "cat"])
def test_centre_reproduces_golden(golden_dir, ms):
    """tests/golden/codebook.npz (the reference class in fp32 on CPU: per (sample, corner), torch's summation order, kaolin's
    coefficient rounding) against the fp32 centre: within the golden's own fp32 noise."""
    g = np.load(os.path.join(golden_dir, "codebook.npz"))
    spc = O.octree_to_spc(g["octree"])
    _, _, trinkets, _ = OG.make_trilinear_spc(spc)
    base = int(g["level"]) - 2
    logits, dicts = [g[f"{ms}_logits{i}"] for i in range(3)], [g[f"{ms}_dict{i}"] for i in range(3)]
    coords = g[f"{ms}_coords"]
    rows, fc, _, bw = pipeline(spc, trinkets, base, logits, dicts, coords, ms, True, g[f"{ms}_go"], False)
    np.testing.assert_allclose(fc, g[f"{ms}_feats_train"], atol=2e-5, rtol=1e-5)
    for i in range(3):
        for got, ref in ((bw[i].g_logits, g[f"{ms}_glogits{i}"]), (bw[i].g_dict, g[f"{ms}_gdict{i}"])):
            assert np.abs(got - ref).max() <= 2e-4 * max(np.abs(ref).max(), 1e-6), (ms, i)
    for lod, key in ((2, "feats_eval"), (0, "feats_eval_lod0")):
        rows, fc, _, _ = pipeline(spc, trinkets, base, logits[:lod + 1], dicts[:lod + 1], coords, ms, False,
                                  np.zeros_like(g[f"{ms}_go"][:, :(4 if ms == "sum" and lod else 4 * (lod + 1))]), False)
        np.testing.assert_allclose(fc, g[f"{ms}_{key}"], atol=2e-5, rtol=1e-5)


def _inside(name, k, c, r):
    k, c, r = (np.asarray(x, np.float64) for x in (k, c, r))
    d = np.abs(k - c)
    bad = ~(d <= r)
    ratio = float(np.max(np.where(r > 0, d / np.where(r > 0, r, 1.0), np.where(d > 0, np.inf, 0.0)), initial=0.0))
    print(f"{name}: max|k-c|/r={ratio:.3g} median_r={float(np.median(r)) if r.size else 0.0:.3g}")
    return int(bad.sum())


# (K, F, rows): the K / F pairs of the GPU tests that matter for the arithmetic (KPL 8 / 32, one feature, many features)
EMU_SHAPES = [(1, 4, 64), (2, 1, 64), (16, 5, 300), (33, 32, 200), (256, 8, 200), (257, 5, 150), (1024, 32, 60)]


def _emu_case(K, F, R, regime, seed):
    rng = np.random.default_rng(seed)
    L = CB.make_logits(R, K, regime, rng)
    D = rng.standard_normal((K, F)).astype(np.float32)
    dE = CB.make_dE(R, F, rng)
    g0 = rng.standard_normal((K, F)).astype(np.float32) if seed % 2 else None
    return L, D, dE, g0


@pytest.mark.parametrize("K,F,R", EMU_SHAPES)
def test_fp32_emulations_land_inside(K, F, R):
    for ri, regime in enumerate(CB.REGIMES):
        L, D, dE, g0 = _emu_case(K, F, R, regime, seed=K + ri)
        fw = {t: CB.rows_fwd(L, D, t) for t in (False, True)}
        bw = CB.rows_bwd(L, D, dE, None, g0)
        if regime == "extreme":
            assert np.all(fw[True].am == CB.first_max(L)) and np.all((fw[True].am >= 0) & (fw[True].am < K))
            eq = (L == L[:, :1]).all(1)
            np.testing.assert_allclose(fw[True].y[eq], 1.0 / K, rtol=1e-6)
            assert np.all(fw[True].am[eq] == 0)
        for trial in range(3):
            rng = np.random.default_rng(100 * trial + ri)
            for t in (False, True):
                am, E = CB.emulate_fwd(L, D, t, rng)
                assert np.array_equal(am, fw[t].am), (regime, t)
                assert np.array_equal(E, fw[t].E), (regime, t)                  # radius 0: bit-exact dictionary[argmax]
            g, gd = CB.emulate_bwd(L, D, dE, rng, g0)
            assert _inside(f"emu K{K} F{F} {regime} g_logits", g, bw.g_logits, bw.g_logits_r) == 0
            assert _inside(f"emu K{K} F{F} {regime} g_dict", gd, bw.g_dict, bw.g_dict_r) == 0
            assert np.all(g[bw.skipped] == 0)


@pytest.mark.parametrize("mutation", CB.MUTATIONS)
def test_mutated_emulations_land_outside(mutation):
    """Every mutation is caught at every shape where it can change a value (a tie-break needs ties, K > 1 everywhere)."""
    for K, F, R in EMU_SHAPES:
        if K == 1 or (mutation == "skip_lane0" and F == 1):
            continue
        bad = 0
        for ri, regime in enumerate(("ties", "unit", "init")):
            L, D, dE, g0 = _emu_case(K, F, R, regime, seed=K + ri)
            rng = np.random.default_rng(ri)
            if mutation == "tie_high":
                am, E = CB.emulate_fwd(L, D, True, rng, mutation)
                fw = CB.rows_fwd(L, D, True)
                bad += int((am != fw.am).sum()) + _inside(f"mut {mutation} K{K} E", E, fw.E, fw.E_r)
                if regime == "ties":
                    assert (am != fw.am).any(), (K, F)
            bw = CB.rows_bwd(L, D, dE, None, g0)
            g, gd = CB.emulate_bwd(L, D, dE, rng, g0, mutation)
            bad += _inside(f"mut {mutation} K{K} F{F} {regime} g_logits", g, bw.g_logits, bw.g_logits_r)
            bad += _inside(f"mut {mutation} K{K} F{F} {regime} g_dict", gd, bw.g_dict, bw.g_dict_r)
        assert bad > 0, (mutation, K, F)


def test_radii_are_tight():
    """Median radii relative to the median magnitude: a few ulps for g_logits, gamma(n + 1)-sized for the dictionary."""
    for K, F, R in EMU_SHAPES[2:]:
        L, D, dE, _ = _emu_case(K, F, R, "unit", seed=3)
        bw = CB.rows_bwd(L, D, dE)
        live = ~bw.skipped
        rl = float(np.median(bw.g_logits_r[live])) / float(np.median(np.abs(bw.g_logits[live])))
        touched = bw.n > 0
        rd = float(np.median(bw.g_dict_r[touched])) / float(np.median(np.abs(bw.g_dict[touched])))
        nmax = int(bw.n.max())
        print(f"K{K} F{F}: median g_logits r/|c| = {rl:.3g}, median g_dict r/|c| = {rd:.3g} (max rows per entry {nmax})")
        assert rl < 3e-5, (K, F, rl)
        assert rd < 4 * float(CB.g32(nmax + 1)), (K, F, rd)
        y, yr = CB.softmax(L)
        assert float(np.median(yr / y)) < 4e-6
