"""CPU checks of oracle/sdf_reference.py, the interval reference of the NeuralSDF(OctreeGrid) kernels (no GPU needed).

  - exact mode (no rounding, no accumulation error): the radius is 0 and the centre is a float64 torch NeuralSDF, its L2 loss and
    its autograd, for 1 and 3 hidden layers, every position-embedding mode, 'cat' and 'sum';
  - soundness: fp32 emulations that round at the kernels' points and sum in random orders (the decoder, the loss, the gradient
    accumulations; the feature blend keeps the order every kernel uses) land inside the intervals;
  - tightness: on the GPU tests' own fields the loss and decoder-gradient radii are 10x below the autograd comparison's
    tolerances wherever the decoder input is exact in fp32 (see test_radii_are_tight);
  - the reference trainer's own step 1 (tests/golden/sdf_train.npz): loss and decoder gradients, and grid gradients within the
    fp16 rounding of the reference's gradient.
"""
import os

import numpy as np
import pytest
import torch

from oracle import octree_grid as OG
from oracle import sdf_reference as S

import sdf_shapes as SH

LOSS_TOL, GRAD_TOL = 1e-5, 1e-4            # tests/test_gpu_sdf_step.py::test_sdf_step_fused_vs_autograd
_CASES = {}


def base_case(num_lods=3, F=8, multiscale="sum", level=5):
    key = (num_lods, F, multiscale, level)
    if key not in _CASES:
        _CASES[key] = OG.make_sdf_case(level=level, num_lods=num_lods, feature_dim=F, hidden_dim=16, multiscale=multiscale, res=4, seed=3,
                                       feature_std=0.05)
    return _CASES[key]


def make_field(pos_mode=1, pos_freq=0, multiscale="sum", layers=1, hidden=16, F=8, num_lods=3, half=True, seed=0, level=5):
    case = base_case(num_lods, F, multiscale, level)
    rng = np.random.default_rng(seed)
    feats = [(rng.standard_normal(f.shape) * 0.3).astype(np.float32) for f in case["feats"]]
    pd = S.Field(case["spc"], case["trinkets"], feats, 0, multiscale, [], [], pos_mode, pos_freq).pos_dim
    in_dim = pd + (F if multiscale == "sum" else F * num_lods)
    Ws, bs = S.random_decoder(rng, in_dim, pos_mode, hidden, layers, scale=1.0)
    return S.Field(case["spc"], case["trinkets"], feats, case["active_lods"][0], multiscale, Ws, bs, pos_mode, pos_freq, half), case


def points(case, n, seed=1):
    rng = np.random.default_rng(seed)
    spc, L = case["spc"], case["level"]
    pts = spc.points[spc.pyramid[1, L]: spc.pyramid[1, L] + spc.pyramid[0, L]].astype(np.float32)
    nn = (n + 1) // 2
    near = (pts[rng.integers(0, pts.shape[0], nn)] + rng.random((nn, 3)).astype(np.float32)) / (2.0 ** (L - 1)) - 1.0
    c = np.concatenate([near, rng.uniform(-1.1, 1.1, (n - nn, 3))]).astype(np.float32)[:n]
    gt = ((np.abs(c).sum(-1) - 0.5) / np.sqrt(3.0)).astype(np.float32)
    return c, gt


# ---------------------------------------------------------------------------------------------------------------
# exact mode against float64 torch + autograd
# ---------------------------------------------------------------------------------------------------------------
def torch_sdf_loss(field, coords, gt, lods):
    """float64 NeuralSDF.sdf + sum_lod sum_i (y - gt)^2 / N, written directly in torch; -> loss, [feature grads], packed decoder grad."""
    t = lambda a: torch.tensor(np.asarray(a, np.float64), requires_grad=True)
    feats = [t(f) for f in field.feats]
    Ws, bs = [t(W) for W in field.Ws], [t(b) for b in field.bs]
    x = torch.tensor(coords.astype(np.float64))
    N = coords.shape[0]
    if field.pos_mode == 0:
        pos = x[:, :0]
    elif field.pos_mode == 1:
        pos = x
    else:
        wind = (x[:, None, :] * (2.0 ** torch.arange(field.pos_freq, dtype=torch.float64))[None, :, None]).reshape(N, -1)
        pos = torch.cat(([x] if field.pos_mode == 3 else []) + [torch.sin(wind), torch.cos(wind)], -1)
    loss = 0.0
    for lod in lods:
        cl = S.cells(field, coords, lod + 1)
        blends = []
        for k in range(lod + 1):
            b = torch.zeros((N, field.F), dtype=torch.float64)
            ok = torch.tensor(cl.ok[k])
            cf = torch.tensor(cl.cf[k])
            v = (feats[k][torch.tensor(cl.tk[k])] * cf[:, :, None]).sum(1)
            blends.append(b.index_put((ok,), v))
        f = sum(blends) if field.multiscale == "sum" else torch.cat(blends, -1)
        h = torch.cat([pos, f], -1)
        for l, (W, b) in enumerate(zip(Ws, bs)):
            h = h @ W.T + b
            if l < len(Ws) - 1:
                h = torch.relu(h)
        loss = loss + ((h[:, 0] - torch.tensor(gt.astype(np.float64))) ** 2).sum() / N
    loss.backward()
    dec = torch.cat([a.grad.reshape(-1) for W, b in zip(Ws, bs) for a in (W, b)]).numpy()
    return float(loss.detach()), [f.grad.numpy() for f in feats], dec, h[:, 0].detach().numpy()


@pytest.mark.parametrize("pos_mode,pos_freq,multiscale,layers", [(0, 0, "sum", 1), (1, 0, "sum", 3), (2, 2, "cat", 1), (3, 3, "cat", 3),
                                                                   (3, 1, "sum", 1), (1, 0, "cat", 1)])
def test_exact_mode_is_float64_autograd(pos_mode, pos_freq, multiscale, layers):
    field, case = make_field(pos_mode, pos_freq, multiscale, layers)
    coords, gt = points(case, 300)
    lods = [field.num_lods - 1] if multiscale == "cat" else list(range(field.num_lods))
    ref_loss, ref_feats, ref_dec, ref_y = torch_sdf_loss(field, coords, gt, lods)
    fw = S.forward(field, coords, exact=True)
    assert np.all(fw.y_r == 0) and np.abs(fw.y - ref_y).max() <= 1e-12 * max(np.abs(ref_y).max(), 1.0)
    tr = S.train(field, coords, gt, lods, exact=True)
    assert tr.loss_r == 0 and abs(tr.loss - ref_loss) <= 1e-12 * ref_loss
    assert np.all(tr.dec_r == 0) and np.abs(tr.dec - ref_dec).max() <= 1e-12 * np.abs(ref_dec).max()
    for (c, r), g in zip(tr.grid, ref_feats):
        assert np.all(r == 0) and np.abs(c - g).max() <= 1e-12 * max(np.abs(g).max(), 1e-300)
    assert not tr.amb.any()


def test_interp_backward_exact():
    field, case = make_field(multiscale="cat")
    coords, _ = points(case, 200)
    go = np.random.default_rng(4).standard_normal((200, field.F * field.num_lods))
    feats = [torch.tensor(f.astype(np.float64), requires_grad=True) for f in field.feats]
    cl = S.cells(field, coords, field.num_lods)
    out = []
    for k in range(field.num_lods):
        v = (feats[k][torch.tensor(cl.tk[k])] * torch.tensor(cl.cf[k])[:, :, None]).sum(1)
        out.append(torch.zeros((200, field.F), dtype=torch.float64).index_put((torch.tensor(cl.ok[k]),), v))
    (torch.cat(out, -1) * torch.tensor(go)).sum().backward()
    for (c, r), f in zip(S.interp_backward(field, coords, go, field.num_lods - 1, exact=True), feats):
        assert np.all(r == 0) and np.abs(c - f.grad.numpy()).max() <= 1e-12 * np.abs(f.grad.numpy()).max()


# ---------------------------------------------------------------------------------------------------------------
# soundness: fp32 emulations with random summation orders
# ---------------------------------------------------------------------------------------------------------------
def _fsum(terms, rng, axis):
    """fp32 sum of `terms` (float64 values of exact products) along `axis` in a random order, one fp32 rounding per addition."""
    terms = np.moveaxis(terms, axis, 0)
    acc = np.zeros(terms.shape[1:], np.float32)
    for i in rng.permutation(terms.shape[0]):
        acc = (acc.astype(np.float64) + terms[i]).astype(np.float32)
    return acc.astype(np.float64)


def emulate(field, coords, gt, lods, rng):
    """The fused training step in fp32: kernel rounding points, random summation orders (one emulated kernel per call)."""
    N = coords.shape[0]
    r32 = lambda a: np.asarray(a, np.float64).astype(np.float32).astype(np.float64)
    inv = float(np.float32(1.0 / N))
    x64 = coords.astype(np.float64)
    if field.pos_mode in (2, 3):
        wind = np.concatenate([x64 * 2.0 ** f for f in range(field.pos_freq)], -1).astype(np.float32)
        ulp = lambda v: rng.integers(-2, 3, v.shape) * np.spacing(np.abs(v).astype(np.float32)).astype(np.float64)
        sc = [r32(fn(wind)) for fn in (np.sin, np.cos)]                     # sinf / cosf: any value within 2 ulp
        pos = np.concatenate(([x64] if field.pos_mode == 3 else []) + [v + ulp(v) for v in sc], -1)
    else:
        pos = x64 if field.pos_mode == 1 else x64[:, :0]
    loss_terms, dec = [], np.zeros(field.packed().size)
    grid = [np.zeros(f.shape) for f in field.feats]
    W0, b0, Wo, bo = [a.astype(np.float64) for a in (field.Ws[0], field.bs[0], field.Ws[-1], field.bs[-1])]
    for lod in lods:
        cl = S.cells(field, coords, lod + 1)
        blends = []
        for k in range(lod + 1):
            ft = field.feats[k].astype(np.float64)
            ft = S.f16(ft) if field.half else ft
            b = np.zeros((N, field.F))
            if cl.ok[k].any():                                             # the corner order every kernel uses
                v = np.zeros((cl.cf[k].shape[0], field.F))
                for j in range(8):
                    v = S.fma32(ft[cl.tk[k][:, j]], cl.cf[k][:, j:j + 1], v)
                b[cl.ok[k]] = S.f16(v) if field.half else v
            blends.append(b)
        if field.multiscale == "sum" and lod > 0:
            f = blends[0]
            for b in blends[1:]:
                f = r32(f + b)
        else:
            f = np.concatenate(blends, -1)
        x = np.concatenate([pos, f], -1)
        a = np.broadcast_to(b0, (N, W0.shape[0])).copy()                   # the kernels' order: bias, then the inputs in order
        for k in range(x.shape[1]):
            a = S.fma32(W0[None, :, k], x[:, k:k + 1], a)
        act = a > 0
        h = np.where(act, a, 0.0)
        y = np.broadcast_to(bo, (N, 1)).copy()
        for j in range(h.shape[1]):
            y = S.fma32(Wo[:, j], h[:, j:j + 1], y)
        y = y[:, 0]
        d = r32(y - gt)
        loss_terms.append(d * d)
        dy = r32(inv * (2 * d))
        G = _fsum((act * Wo)[:, :, None] * W0[None], rng, 1)
        da = r32(dy[:, None] * (act * Wo))
        gW0 = _fsum(da[:, :, None] * x[:, None, :], rng, 0)
        parts = [gW0.reshape(-1), _fsum(da, rng, 0), _fsum(dy[:, None] * h, rng, 0), _fsum(dy[:, None], rng, 0)]
        dec = r32(dec + np.concatenate(parts))
        gx = r32(dy[:, None] * G[:, field.pos_dim:])
        for k in range(lod + 1):
            ok, tk, cf = cl.ok[k], cl.tk[k], cl.cf[k]
            cols = slice(0, field.F) if field.multiscale == "sum" and lod > 0 else slice(k * field.F, (k + 1) * field.F)
            t = r32(gx[ok][:, None, cols] * cf[:, :, None])                   # [n, 8, F]
            rows, tt = tk.reshape(-1), t.reshape(-1, field.F)
            order = rng.permutation(rows.shape[0])
            g = grid[k].astype(np.float32)
            for i in order:
                g[rows[i]] = (g[rows[i]].astype(np.float64) + tt[i]).astype(np.float32)
            grid[k] = g.astype(np.float64)
    loss = float(r32(_fsum(np.concatenate(loss_terms), rng, 0) * inv))
    return loss, dec, grid


@pytest.mark.parametrize("pos_mode,pos_freq,multiscale,lods,half", [(1, 0, "sum", "last", True), (3, 2, "cat", "last", True),
                                                                     (2, 1, "sum", "all", False), (0, 0, "sum", "all", True)])
def test_fp32_emulation_inside_intervals(pos_mode, pos_freq, multiscale, lods, half):
    field, case = make_field(pos_mode, pos_freq, multiscale, 1, hidden=12, half=half, seed=2)
    coords, gt = points(case, 160, seed=3)
    lods = [field.num_lods - 1] if lods == "last" else list(range(field.num_lods))
    tr = S.train(field, coords, gt, lods, sms=1)            # two tiles on one SM: the any-order bounds of the sums over samples
    keep = ~tr.amb
    assert keep.mean() > 0.9
    coords, gt = coords[keep], gt[keep]
    tr = S.train(field, coords, gt, lods, sms=1)
    assert not tr.amb.any()
    rng = np.random.default_rng(9)
    for _ in range(3):
        loss, dec, grid = emulate(field, coords, gt, lods, rng)
        assert abs(loss - tr.loss) <= tr.loss_r
        assert np.all(np.abs(dec - tr.dec) <= tr.dec_r)
        for g, (c, r) in zip(grid, tr.grid):
            assert np.all(np.abs(g - c) <= r)


# ---------------------------------------------------------------------------------------------------------------
# tightness
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", sorted(SH.SHAPES))
def test_radii_are_tight(name):
    """The radii on tests/test_gpu_sdf_kernels.py's own fields and points (N = 1000: one tile per CTA, so every chain but the
    atomics is emulated in the kernel's order).  Where the decoder input is exact in fp32 (no sin/cos of a position already
    carrying raw x), the loss radius is 10x below the 1e-5 relative and the decoder-gradient radius 10x below the 1e-4 of max of
    the autograd comparison; sinf / cosf (2 ulp) of 3 + 6 f inputs leave up to 2e-5 / 3e-5.  Grid gradients are sums of one
    atomic per sample and corner in any order: below 1e-4 of max, 3e-4 on the 1-feature root level that every sample reaches."""
    field, case = SH.make_field(name)
    coords, gt = SH.points(case, 1000, seed=3)
    fw = S.forward(field, coords)
    assert fw.amb.mean() <= 0.01 and fw.y_r.max() <= 1e-6 * np.abs(fw.y).max()
    if len(field.Ws) > 2:
        return
    tr = S.train(field, coords, gt, [field.num_lods - 1])
    exact_inputs = field.pos_mode != 3
    assert tr.loss_r <= (0.1 * LOSS_TOL if exact_inputs else 2e-5) * tr.loss
    assert tr.dec_r.max() <= (0.1 * GRAD_TOL if exact_inputs else 3e-5) * np.abs(tr.dec).max()
    for c, r in tr.grid:
        assert r.max() <= (3 if field.F == 1 else 1) * GRAD_TOL * np.abs(c).max()


# ---------------------------------------------------------------------------------------------------------------
# the reference trainer's step 1
# ---------------------------------------------------------------------------------------------------------------
GOLDEN_GRID_TOL = 2e-2      # of max: the reference's grid gradient is fp16 (feats.half(), octree_grid.py:147); measured: <= 1.1e-2


@pytest.mark.parametrize("case", ["sum", "cat", "sum_all"])
def test_golden_step1(golden_dir, case):
    from oracle import oracle as O
    g = np.load(os.path.join(golden_dir, "sdf_train.npz"))
    spc = O.octree_to_spc(g["octree"])
    _, _, trinkets, _ = OG.make_trilinear_spc(spc)
    p = lambda n: g[f"{case}_init_{n}"]
    feats = [p(f"grid.features.{k}") for k in range(3)]
    field = S.Field(spc, trinkets, feats, int(g["level"]) - 2, str(g[f"{case}_multiscale"]),
                    [p("decoder.layers.0.weight"), p("decoder.lout.weight")], [p("decoder.layers.0.bias"), p("decoder.lout.bias")], 1, 0, True)
    lods = [int(l) for l in g[f"{case}_loss_lods"]]
    tr = S.train(field, g["coords"], g["sdf"].reshape(-1), lods)
    assert tr.amb.mean() < 0.02
    assert abs(tr.loss - g[f"{case}_losses"][0]) <= 1e-6 * tr.loss                 # measured: <= 1e-7
    ref_dec = np.concatenate([g[f"{case}_grad1_decoder.{n}"].reshape(-1) for n in ("layers.0.weight", "layers.0.bias", "lout.weight", "lout.bias")])
    assert np.abs(tr.dec - ref_dec).max() <= 1e-6 * np.abs(ref_dec).max()          # measured: <= 1.2e-7 of max
    for k, (c, r) in enumerate(tr.grid):
        ref = g[f"{case}_grad1_grid.features.{k}"]
        assert np.abs(c - ref).max() <= GOLDEN_GRID_TOL * np.abs(ref).max(), k
