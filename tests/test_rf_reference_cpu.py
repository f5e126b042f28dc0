"""tests/rf_reference.py without a GPU: with rounding and accumulation off it is the float64 operation (torch's F.grid_sample,
the OctreeGrid blend and the NeuralRadianceField decoders, with autograd); fp32 emulations of the kernels, with random summation
orders, atomics in random order and sinf / cosf off by up to 2 ulp, land inside its intervals; it reproduces the triplanar golden;
and where the inputs are exact its gradient radii are at least 10x below the end-to-end tolerances the GPU tests replace."""
from types import SimpleNamespace

import numpy as np
import pytest
import torch
import torch.nn.functional as Fn

from oracle import octree_grid as OG
from oracle import oracle as O
from oracle import sdf_reference as S
from oracle import tc_decoders as T

import rf_reference as RF

TOL0_GRAD, TOL1_GRAD = 2e-3, 3e-2           # end-to-end gradient tolerances (of max) at precision 0 and 1


def special_coords(rng, n, sides):
    """Coordinates several periods outside [-1, 1], exactly +-1, and on texel lines of the given plane sides."""
    c = rng.uniform(-7.0, 7.0, (n, 3))
    lines = np.concatenate([2.0 * np.arange(s) / (s - 1) - 1.0 for s in sides] + [[-1.0, 1.0, 3.0, -5.0]])
    m = rng.random((n, 3)) < 0.3
    c[m] = rng.choice(lines, int(m.sum()))
    return c.astype(np.float32)


def triplanar(rng, C, sides, ms, nl=None):
    planes = [[(rng.standard_normal((C, s, s)) * 0.5).astype(np.float32) for _ in range(3)] for s in sides]
    return RF.Triplanar(planes, ms, nl or len(sides))


def torch_triplanar(tp, coords):
    """float64 TriplanarGrid.interpolate: F.grid_sample(align_corners=True, padding_mode='reflection') per plane."""
    leaves, outs = [], []
    x = torch.from_numpy(coords.astype(np.float64))
    pair = [(1, 2), (0, 2), (0, 1)]
    per_lod = []
    for l in range(tp.nl):
        row = []
        for p in range(3):
            pl = torch.from_numpy(tp.planes[l][p].astype(np.float64))[None].requires_grad_(True)
            leaves.append(pl)
            g = x[:, list(pair[p])][None, :, None, :]
            row.append(Fn.grid_sample(pl, g, mode="bilinear", padding_mode="reflection", align_corners=True)[0, :, :, 0].T)
        per_lod.append(torch.cat(row, 1))
    out = torch.cat(per_lod, 1) if tp.multiscale == "cat" else sum(per_lod)
    return out, leaves


@pytest.mark.parametrize("C,sides,ms", [(1, (2,), "cat"), (3, (3, 7), "sum"), (4, (5, 9, 17), "cat"), (8, (2, 513), "sum")])
def test_triplanar_exact_matches_grid_sample(C, sides, ms):
    rng = np.random.default_rng(C)
    tp = triplanar(rng, C, sides, ms)
    coords = special_coords(rng, 500, sides)
    out, leaves = torch_triplanar(tp, coords)
    fc, fr = RF.triplanar_features(tp, coords, exact=True)
    assert np.all(fr == 0)
    np.testing.assert_allclose(fc, out.detach().numpy(), rtol=0, atol=1e-12)
    go = rng.standard_normal(fc.shape)
    out.backward(torch.from_numpy(go))
    ref = RF.triplanar_scatter(tp, coords, go, np.zeros_like(go), exact=True)
    for i, leaf in enumerate(leaves):
        c, r = ref[i // 3][i % 3]
        assert np.all(r == 0)
        np.testing.assert_allclose(c, leaf.grad[0].numpy(), rtol=0, atol=1e-12)


def test_triplanar_reproduces_golden(golden_dir):
    import os
    g = np.load(os.path.join(golden_dir, "triplanar.npz"))
    for ms in ("sum", "cat"):
        planes = [[g[f"{ms}_plane{3 * l + p}"][0] for p in range(3)] for l in range(3)]
        tp = RF.Triplanar(planes, ms, 3)
        coords = g[f"{ms}_coords"]
        fc, fr = RF.triplanar_features(tp, coords)
        np.testing.assert_allclose(fc, g[f"{ms}_feats"].reshape(fc.shape), atol=2e-6, rtol=1e-4)
        lod0 = RF.triplanar_features(RF.Triplanar(planes, ms, 1), coords)[0]
        np.testing.assert_allclose(lod0, g[f"{ms}_feats_lod0"].reshape(lod0.shape), atol=2e-6, rtol=1e-4)
        go = g[f"{ms}_go"].reshape(fc.shape).astype(np.float64)
        ref = RF.triplanar_scatter(tp, coords, go, np.zeros_like(go))
        for i in range(9):
            np.testing.assert_allclose(ref[i // 3][i % 3][0], g[f"{ms}_gplane{i}"][0], atol=2e-5, rtol=1e-4)


def _emulate_sum(terms, rng, axis_len):
    """fp32 sum of terms [N, n] in a random order per row (each addition rounded)."""
    perm = np.argsort(rng.random(terms.shape), 1)
    t = np.take_along_axis(terms.astype(np.float32), perm, 1)
    acc = t[:, 0].copy()
    for j in range(1, axis_len):
        acc = (acc + t[:, j]).astype(np.float32)
    return acc


@pytest.mark.parametrize("C,sides,ms", [(2, (3, 5, 9), "sum"), (5, (2, 17), "cat")])
def test_triplanar_fp32_emulation_inside(C, sides, ms):
    rng = np.random.default_rng(11 + C)
    tp = triplanar(rng, C, sides, ms)
    coords = special_coords(rng, 2000, sides)
    fc, fr = RF.triplanar_features(tp, coords)
    emu = np.zeros(fc.shape, np.float32)
    for l in range(tp.nl):
        s = sides[l]
        for p in range(3):
            b = RF.tp_setup(coords, p, s)
            for c in range(C):
                pl = tp.planes[l][p][c].reshape(-1)
                terms = (pl[b.idx] * b.w.astype(np.float32)).astype(np.float32)
                v = _emulate_sum(terms, rng, 4)
                f = tp.col(l, p, c)
                emu[:, f] = (emu[:, f] + v).astype(np.float32)
    assert np.all(np.abs(emu - fc) <= fr)
    # scatter: one fp32 product per texel, atomics in random order
    gc = rng.standard_normal(fc.shape)
    gc = gc.astype(np.float32).astype(np.float64)
    ref = RF.triplanar_scatter(tp, coords, gc, np.zeros_like(gc))
    for l in range(tp.nl):
        for p in range(3):
            b = RF.tp_setup(coords, p, sides[l])
            for c in range(C):
                terms = (gc[:, tp.col(l, p, c)][:, None].astype(np.float32) * b.w.astype(np.float32)).reshape(-1)
                idx = b.idx.reshape(-1)
                order = rng.permutation(terms.size)
                acc = np.zeros(sides[l] ** 2, np.float32)
                for k in order:                                          # atomics one by one
                    acc[idx[k]] = np.float32(acc[idx[k]] + terms[k])
                cc, rr = ref[l][p]
                assert np.all(np.abs(acc - cc[c].reshape(-1)) <= rr[c].reshape(-1))


def octree_case(rng, F, ms, half, level=4, lods=3):
    spc = O.octree_to_spc(O.points_to_octree(O.lego_like_points(level), level))
    _, pyr, tr, _ = OG.make_trilinear_spc(spc)
    base = level - lods + 1
    feats = [(rng.standard_normal((int(pyr[0, base + k]), F)) * 0.5).astype(np.float32) for k in range(lods)]
    return RF.octree_field(spc, tr, feats, base, ms, half), tr, feats, base


@pytest.mark.parametrize("F,ms,half,nl", [(3, "sum", False, 3), (8, "cat", True, 2), (16, "sum", True, 1), (1, "cat", False, 3)])
def test_octree_reference(F, ms, half, nl):
    rng = np.random.default_rng(F)
    field, tr, feats, base = octree_case(rng, F, ms, half)
    coords = rng.uniform(-1.3, 1.3, (3000, 3)).astype(np.float32)
    # the reference's fp32 features against the independent restatement of OctreeGrid.interpolate (Kaolin's coefficient formula)
    fc, fr, cl = RF.octree_features(field, coords, nl)
    assert np.all(fr == 0)
    ref = OG.octree_grid_interpolate(field.spc, tr, feats, [base + k for k in range(len(feats))], coords, nl - 1, ms, half)
    np.testing.assert_allclose(fc, ref, atol=2e-3 if half else 2e-6, rtol=1e-4)
    assert (np.abs(fc) > 0).any(axis=1).mean() > 0.2 and (fc == 0).all(axis=1).mean() > 0.05       # hits and misses
    # exact: a float64 torch blend over the same cells, and its autograd
    ec, er, _ = RF.octree_features(field, coords, nl, exact=True)
    leaves = [torch.from_numpy(f.astype(np.float64)).requires_grad_(True) for f in feats[:nl]]
    blends = []
    for k in range(nl):
        b = torch.zeros((coords.shape[0], F), dtype=torch.float64)
        ok = torch.from_numpy(cl.ok[k])
        v = leaves[k][torch.from_numpy(cl.tk[k])]                               # [n, 8, F]
        b[ok] = (v * torch.from_numpy(cl.cf[k])[:, :, None]).sum(1)
        blends.append(b)
    out = sum(blends) if (ms == "sum" and nl > 1) else torch.cat(blends, 1)
    np.testing.assert_allclose(ec, out.detach().numpy(), rtol=0, atol=1e-12)
    go = rng.standard_normal(ec.shape)
    out.backward(torch.from_numpy(go))
    sc = RF.octree_scatter(field, cl, nl, go, np.zeros_like(go), exact=True)
    for k in range(nl):
        np.testing.assert_allclose(sc[k][0], leaves[k].grad.numpy(), rtol=0, atol=1e-12)
    # fp32 atomics in random order land inside
    gc = go.astype(np.float32).astype(np.float64)
    sc = RF.octree_scatter(field, cl, nl, gc, np.zeros_like(gc))
    for k in range(nl):
        cols = slice(0, F) if (ms == "sum" and nl > 1) else slice(k * F, (k + 1) * F)
        g = gc[cl.ok[k]][:, cols].astype(np.float32)
        acc = np.zeros(feats[k].shape, np.float32)
        terms = (g[:, None, :] * cl.cf[k].astype(np.float32)[:, :, None]).astype(np.float32)     # [n, 8, F]
        rows = cl.tk[k]
        for i in rng.permutation(rows.size):
            n_, j = divmod(int(i), 8)
            acc[rows[n_, j]] = (acc[rows[n_, j]] + terms[n_, j]).astype(np.float32)
        assert np.all(np.abs(acc - sc[k][0]) <= sc[k][1])


def _decoders(rng, dens, col, bias=True):
    def mlp(dims):
        Ws = [(rng.uniform(-1, 1, (o, i)) / np.sqrt(i)).astype(np.float32) for i, o in zip(dims[:-1], dims[1:])]
        bs = [(rng.uniform(-1, 1, o) / np.sqrt(i)).astype(np.float32) for i, o in zip(dims[:-1], dims[1:])] if bias else None
        return Ws, bs
    return T.Decoders(*mlp(dens), *mlp(col))


def torch_rgba(dec, x0, dirs, view):
    """float64 NeuralRadianceField.rgba's decoders: density stack, relu(density), colour stack on [density feats 1:, view], sigmoid."""
    leaves = []

    def stack(h, Ws, bs):
        for l, Wm in enumerate(Ws):
            w = torch.from_numpy(Wm.astype(np.float64)).requires_grad_(True); leaves.append(w)
            h = h @ w.T
            if bs is not None:
                b = torch.from_numpy(bs[l].astype(np.float64)).requires_grad_(True); leaves.append(b)
                h = h + b
            if l < len(Ws) - 1:
                h = torch.relu(h)
        return h
    x = torch.from_numpy(x0).requires_grad_(True)
    df = stack(x, dec.dens_W, dec.dens_b)
    n_dens = len(leaves)
    ve = torch.from_numpy(S._embed(SimpleNamespace(pos_mode=view[0], pos_freq=view[1]), dirs.astype(np.float64), True)[0])
    c3 = stack(torch.cat([df[:, 1:], ve], 1), dec.col_W, dec.col_b)
    out = torch.cat([torch.sigmoid(c3), torch.relu(df[:, :1])], 1)
    return out, x, leaves[:n_dens], leaves[n_dens:]


@pytest.mark.parametrize("dens,col,view,bias", [([16], [16, 16], (3, 2), True), ([], [], (1, 0), True), ([40, 24], [20, 36, 12], (2, 3), False)])
def test_decoders_exact_match_torch(dens, col, view, bias):
    rng = np.random.default_rng(len(dens) * 7 + len(col))
    I0, dout = 12, 9
    vd = 0 if view[0] == 0 else 3 if view[0] == 1 else 6 * view[1] + (3 if view[0] == 3 else 0)
    dec = _decoders(rng, [I0] + dens + [dout], [dout - 1 + vd] + col + [3], bias)
    S_ = 300
    x0 = rng.standard_normal((S_, I0))
    dirs = rng.standard_normal((S_, 3)).astype(np.float32)
    ref = RF.Shade0(dec, x0, np.zeros_like(x0), dirs, *view, exact=True)
    out, x, ld, lc = torch_rgba(dec, x0, dirs, view)
    c, r = ref.shaded()
    assert np.all(r == 0)
    np.testing.assert_allclose(c, out.detach().numpy(), rtol=0, atol=1e-12)
    go = rng.standard_normal((S_, 4)).astype(np.float32)
    out.backward(torch.from_numpy(go.astype(np.float64)))
    bw = ref.backward(go)
    np.testing.assert_allclose(bw["dx0"][0], x.grad.numpy(), rtol=0, atol=1e-12)
    for key, leaves in (("dens", ld), ("col", lc)):
        want = np.concatenate([l.grad.numpy().reshape(-1) for l in leaves])
        np.testing.assert_allclose(bw[key][0], want, rtol=0, atol=1e-12)
        assert np.all(bw[key][1] == 0)


def _sinf_embed(dirs, mode, freq, rng):
    """The view embedding with sinf / cosf off by up to 2 ulp."""
    c, _ = S._embed(SimpleNamespace(pos_mode=mode, pos_freq=freq), dirs.astype(np.float64), False)
    c = c.astype(np.float32)
    first = 3 if mode in (1, 3) else 0
    k = rng.integers(-2, 3, c[:, first:].shape)
    tr = c[:, first:]
    for _ in range(2):
        tr = np.where(k > 0, np.nextafter(tr, np.float32(np.inf)), np.where(k < 0, np.nextafter(tr, np.float32(-np.inf)), tr))
        k = k - np.sign(k)
    c[:, first:] = tr
    return c


def _fma_chain(x, W, b, rng=None):
    """fp32 fmaf chain per unit seeded with b over the inputs in ascending order (what wb_layer_fwd / wb_dgrad compute)."""
    s = np.broadcast_to(b.astype(np.float64), (x.shape[0], W.shape[0])).copy()
    for k in range(W.shape[1]):
        s = S.fma32(W[None, :, k].astype(np.float64), x[:, k:k + 1].astype(np.float64), s)
    return s.astype(np.float32)


def emulate_shade0(dec, x0, dirs, view, go, nt, rng):
    """fp32 emulation of wb_shade_fwd_kernel / wb_shade_bwd_kernel for one CTA per tile: in-order chains, sinf / cosf off by up to
    2 ulp, weight and bias gradients summed over the samples of a tile in a random order and the tiles added in a random order."""
    f32 = np.float32
    nd = len(dec.dens_W)
    layers = [(Wm, (dec.dens_b[l] if dec.dens_b else np.zeros(Wm.shape[0], f32))) for l, Wm in enumerate(dec.dens_W)] + \
             [(Wm, (dec.col_b[l] if dec.col_b else np.zeros(Wm.shape[0], f32))) for l, Wm in enumerate(dec.col_W)]
    h = x0.astype(f32)
    ins = []
    ve = _sinf_embed(dirs, *view, rng)
    for l, (Wm, b) in enumerate(layers):
        if l == nd:
            df = h
            h = np.concatenate([h[:, 1:], ve], 1)
        ins.append(h)
        a = _fma_chain(h, Wm, b)
        h = a if l in (nd - 1, len(layers) - 1) else np.maximum(a, f32(0))
    rgb = (f32(1) / (f32(1) + np.exp(-h, dtype=f32))).astype(f32)
    shaded = np.concatenate([rgb, np.maximum(df[:, :1], f32(0))], 1)
    g = ((go[:, :3] * rgb).astype(f32) * (f32(1) - rgb)).astype(f32)
    S_ = x0.shape[0]
    tiles = [np.arange(t, min(t + nt, S_)) for t in range(0, S_, nt)]
    grads = [None] * len(layers)
    for l in range(len(layers) - 1, -1, -1):
        Wm, b = layers[l]
        x = ins[l]
        gw, gb = np.zeros(Wm.shape, f32), np.zeros(Wm.shape[0], f32)
        for ti in rng.permutation(len(tiles)):
            acc, bacc = np.zeros(Wm.shape, f32), np.zeros(Wm.shape[0], f32)
            for si in rng.permutation(tiles[ti]):
                acc = (acc + (g[si][:, None] * x[si][None, :]).astype(f32)).astype(f32)
                bacc = (bacc + g[si]).astype(f32)
            gw = (gw + acc).astype(f32); gb = (gb + bacc).astype(f32)
        grads[l] = (gw, gb)
        n = _fma_chain(g, Wm.T, np.zeros(Wm.shape[1], f32))
        if l == nd:
            n = np.concatenate([np.where(df[:, :1] > 0, go[:, 3:4], f32(0)), n[:, :df.shape[1] - 1]], 1)
        elif l > 0:
            n = np.where(x > 0, n, f32(0))
        g = n
    packs = {}
    for key, ls, has_b in (("dens", range(nd), dec.dens_b is not None), ("col", range(nd, len(layers)), dec.col_b is not None)):
        packs[key] = np.concatenate([a.reshape(-1) for l in ls for a in (grads[l] if has_b else grads[l][:1])])
    return shaded, packs, g


@pytest.mark.parametrize("dens,col,view,bias", [([24], [24, 24], (3, 2), True), ([20, 12], [12, 28, 8], (2, 1), False)])
def test_shade0_fp32_emulation_inside(dens, col, view, bias):
    rng = np.random.default_rng(5 + len(col))
    I0, dout = 10, 6
    vd = 0 if view[0] == 0 else 3 if view[0] == 1 else 6 * view[1] + (3 if view[0] == 3 else 0)
    dec = _decoders(rng, [I0] + dens + [dout], [dout - 1 + vd] + col + [3], bias)
    S_, nt = 200, 64
    x0 = rng.standard_normal((S_, I0)).astype(np.float32)
    dirs = rng.standard_normal((S_, 3)).astype(np.float32)
    go = (rng.standard_normal((S_, 4)) * 1e-2).astype(np.float32)
    ref = RF.Shade0(dec, x0.astype(np.float64), np.zeros((S_, I0)), dirs, *view)
    bw = ref.backward(go, nt, -(-S_ // nt))
    for trial in range(2):
        shaded, packs, dx0 = emulate_shade0(dec, x0, dirs, view, go, nt, np.random.default_rng(trial))
        c, r = ref.shaded()
        assert np.all(np.abs(shaded - c) <= r)
        for key in ("dens", "col"):
            assert np.all(np.abs(packs[key] - bw[key][0]) <= bw[key][1]), key
        assert np.all(np.abs(dx0 - bw["dx0"][0]) <= bw["dx0"][1])


def test_radius_tightness_with_exact_inputs():
    """fp32-exact decoder inputs (octree features: bit-exact), no view embedding: the median gradient radius is 10x below the
    precision-0 end-to-end tolerance (2e-3 of max) for the decoders and the grid; the precision-1 scatter of fp16 planes 10x below 3e-2."""
    rng = np.random.default_rng(3)
    field, *_ = octree_case(rng, 8, "cat", True)
    coords = rng.uniform(-0.9, 0.9, (2000, 3)).astype(np.float32)
    fc, fr, cl = RF.octree_features(field, coords, 3)
    assert np.all(fr == 0)
    dec = _decoders(rng, [24, 64, 16], [15, 64, 64, 3])
    ref = RF.Shade0(dec, fc, fr, np.ones((2000, 3), np.float32), 0, 0)
    go = (rng.standard_normal((2000, 4)) * 1e-2).astype(np.float32)
    plan = RF.shade0_plan([24, 64, 16], [15, 64, 64, 3])
    bw = ref.backward(go, plan.nt_bwd, -(-2000 // plan.nt_bwd))
    for key in ("dens", "col"):
        c, r = bw[key]
        assert np.median(r) <= 0.1 * TOL0_GRAD * np.abs(c).max(), key
    sc = RF.octree_scatter(field, cl, 3, *bw["dx0"])
    for c, r in sc:
        assert np.median(r[c != 0]) <= 0.1 * TOL0_GRAD * np.abs(c).max()
    planes = T.f16(rng.standard_normal((2000, 24)) * 0.1)
    sc = RF.octree_scatter(field, cl, 3, planes, np.zeros_like(planes), RF.SCAN_LEVELS)
    for c, r in sc:
        assert np.median(r[c != 0]) <= 0.1 * TOL1_GRAD * np.abs(c).max()


def test_shade0_plan_tiles():
    """The tile sizes of wb_shade_{fwd,bwd}_launch for the decoder shapes the GPU tests use for NT 128 / 64 / 32."""
    assert RF.shade0_plan([42, 48, 16], [15 + 21, 48, 48, 3]).nt_bwd == 128
    p = RF.shade0_plan([35, 100, 60, 16], [42, 100, 36, 20, 3])
    assert (p.nt_fwd, p.nt_bwd) == (128, 64)
    p = RF.shade0_plan([16, 256, 16], [42, 256, 3])
    assert (p.nt_fwd, p.nt_bwd, p.per_sm) == (64, 32, 1)
    assert p.tiles_per_cta(2 * 132 * 32 + 1, 132) == 3
    assert RF.shade0_plan([16, 256, 256, 16], [42, 256, 3]) is None
