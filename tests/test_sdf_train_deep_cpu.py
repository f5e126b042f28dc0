"""CPU checks of tests/sdf_deep_reference.py, the interval reference of wb_sdf_train for decoders with 2 to 4 hidden layers, as its
layer-by-layer kernel trains them (no GPU needed):
  - soundness: an fp32 emulation of that kernel (forward chains in the kernel's order; the backward's delta chains over units, the
    sums over samples and CTAs and the atomics in random orders) lands inside the rounded-mode intervals;
  - tightness: on tests/test_gpu_sdf_train_deep.py's fields the decoder-gradient radii are 10x and the loss radii 3x below the
    autograd comparison's tolerances wherever the decoder input is exact in fp32;
  - the reference trainer's own step 1 with deeper decoders (tests/golden/sdf_train_deep.npz);
  - the packed decoder order of ops.decoder_params, which SDFStep flattens into the kernel's parameter buffer."""
import os

import numpy as np
import pytest
import torch

from oracle import octree_grid as OG
from oracle import sdf_reference as S

import sdf_deep_reference as DR
import sdf_deep_shapes as DS
from test_sdf_reference import GOLDEN_GRID_TOL, GRAD_TOL, LOSS_TOL, _fsum
from test_sdf_reference import make_field as small_field
from test_sdf_reference import points as small_points


def emulate_deep(field, coords, gt, lods, rng):
    """wb_sdf_train_deep_kernel in fp32: the forward bit-exact in the kernel's order, every sum of the backward in a random order."""
    N = coords.shape[0]
    r32 = S.r32
    inv = float(np.float32(1.0 / N))
    x64 = coords.astype(np.float64)
    if field.pos_mode in (2, 3):
        wind = np.concatenate([x64 * 2.0 ** f for f in range(field.pos_freq)], -1).astype(np.float32)
        ulp = lambda v: rng.integers(-2, 3, v.shape) * np.spacing(np.abs(v).astype(np.float32)).astype(np.float64)
        sc = [r32(fn(wind)) for fn in (np.sin, np.cos)]
        pos = np.concatenate(([x64] if field.pos_mode == 3 else []) + [v + ulp(v) for v in sc], -1)
    else:
        pos = x64 if field.pos_mode == 1 else x64[:, :0]
    Ws = [W.astype(np.float64) for W in field.Ws]
    bs = [b.astype(np.float64) for b in field.bs]
    loss_terms, dec = [], np.zeros(field.packed().size)
    grid = [np.zeros(f.shape) for f in field.feats]
    for lod in lods:
        fc, _, _, cl = S.features(field, coords, lod + 1)
        x = np.concatenate([pos, fc], -1)
        hs = [x]
        for W, b in zip(Ws[:-1], bs[:-1]):                 # per unit: the bias, then the inputs in order
            a = np.broadcast_to(b, (N, W.shape[0])).copy()
            for k in range(W.shape[1]):
                a = S.fma32(W[None, :, k], hs[-1][:, k:k + 1], a)
            hs.append(np.maximum(a, 0.0))
        y = np.broadcast_to(bs[-1], (N, 1)).copy()
        for j in range(hs[-1].shape[1]):
            y = S.fma32(Ws[-1][:, j], hs[-1][:, j:j + 1], y)
        d = r32(y[:, 0] - gt)
        loss_terms.append(d * d)
        dy = r32(inv * (2 * d))
        parts = [None] * (2 * len(Ws))
        parts[-2] = _fsum(dy[:, None] * hs[-1], rng, 0)
        parts[-1] = _fsum(dy[:, None], rng, 0)
        delta = np.where(hs[-1] > 0, r32(dy[:, None] * Ws[-1][0][None]), 0.0)
        for l in range(len(Ws) - 2, -1, -1):
            parts[2 * l] = _fsum(delta[:, :, None] * hs[l][:, None, :], rng, 0).reshape(-1)
            parts[2 * l + 1] = _fsum(delta, rng, 0)
            back = _fsum(delta[:, :, None] * Ws[l][None], rng, 1)          # sum over the units of W_l[j, :] delta_l[j]
            delta = np.where(hs[l] > 0, back, 0.0) if l > 0 else back
        dec = r32(dec + np.concatenate(parts))
        gx = delta[:, field.pos_dim:]
        for k in range(lod + 1):
            ok, tk, cf = cl.ok[k], cl.tk[k], cl.cf[k]
            cols = slice(0, field.F) if field.multiscale == "sum" and lod > 0 else slice(k * field.F, (k + 1) * field.F)
            t = r32(gx[ok][:, None, cols] * cf[:, :, None])
            rows, tt = tk.reshape(-1), t.reshape(-1, field.F)
            g = grid[k].astype(np.float32)
            for i in rng.permutation(rows.shape[0]):
                g[rows[i]] = (g[rows[i]].astype(np.float64) + tt[i]).astype(np.float32)
            grid[k] = g.astype(np.float64)
    loss = float(r32(_fsum(np.concatenate(loss_terms), rng, 0) * inv))
    return loss, dec, grid


@pytest.mark.parametrize("pos_mode,pos_freq,multiscale,layers,lods,half", [(1, 0, "sum", 2, "last", True), (3, 2, "cat", 3, "last", True),
                                                                            (2, 1, "sum", 4, "all", False), (0, 0, "sum", 2, "all", True)])
def test_fp32_emulation_inside_intervals(pos_mode, pos_freq, multiscale, layers, lods, half):
    field, case = small_field(pos_mode, pos_freq, multiscale, layers, hidden=12, half=half, seed=2)
    coords, gt = small_points(case, 160, seed=3)
    lods = [field.num_lods - 1] if lods == "last" else list(range(field.num_lods))
    tr = DR.train(field, coords, gt, lods, sms=1)
    keep = ~tr.amb
    assert keep.mean() > 0.8
    coords, gt = coords[keep], gt[keep]
    tr = DR.train(field, coords, gt, lods, sms=1)
    assert not tr.amb.any()
    rng = np.random.default_rng(9)
    for _ in range(3):
        loss, dec, grid = emulate_deep(field, coords, gt, lods, rng)
        assert abs(loss - tr.loss) <= tr.loss_r
        assert np.all(np.abs(dec - tr.dec) <= tr.dec_r), np.max(np.abs(dec - tr.dec) - tr.dec_r)
        for g, (c, r) in zip(grid, tr.grid):
            assert np.all(np.abs(g - c) <= r)


@pytest.mark.parametrize("name", sorted(DS.DEEP_SHAPES))
def test_radii_are_tight(name):
    """N = 1000 on the GPU tests' fields, with the kernel's tile: where the decoder input is exact in fp32 the decoder-gradient
    radius is 10x below 1e-4 of max; the loss radius, an order-free bound (gamma of the tree height times the loss: the deep
    kernel's per-CTA partials are not emulated), stays 3x below 1e-5.  With sinf / cosf inputs (2 ulp): up to 2e-5 / 5e-5."""
    field, case = DS.make_field(name, seed=1)
    coords, gt = DS.points(case, 1000, seed=3)
    tr = DR.train(field, coords, gt, [field.num_lods - 1], tile=DS.tile_of(field))
    assert tr.amb.mean() <= 0.02
    exact_inputs = field.pos_mode != 3
    assert tr.loss_r <= (0.3 * LOSS_TOL if exact_inputs else 2e-5) * tr.loss
    assert tr.dec_r.max() <= (0.1 * GRAD_TOL if exact_inputs else 5e-5) * np.abs(tr.dec).max()
    for c, r in tr.grid:
        assert r.max() <= GRAD_TOL * np.abs(c).max()


def _golden_field(g, case):
    from oracle import oracle as O
    spc = O.octree_to_spc(g["octree"])
    _, _, trinkets, _ = OG.make_trilinear_spc(spc)
    p = lambda n: g[f"{case}_init_{n}"]
    feats = [p(f"grid.features.{k}") for k in range(3)]
    nh = len([k for k in g.files if k.startswith(f"{case}_init_decoder.layers.") and k.endswith(".weight")])
    names = [f"layers.{l}" for l in range(nh)] + ["lout"]
    field = S.Field(spc, trinkets, feats, int(g["level"]) - 2, str(g[f"{case}_multiscale"]),
                    [p(f"decoder.{n}.weight") for n in names], [p(f"decoder.{n}.bias") for n in names], 1, 0, True)
    return field, names


@pytest.mark.parametrize("case", ["sum", "cat", "sum_all"])
def test_golden_step1(golden_dir, case):
    g = np.load(os.path.join(golden_dir, "sdf_train_deep.npz"))
    field, names = _golden_field(g, case)
    assert len(field.Ws) - 1 == {"sum": 2, "cat": 3, "sum_all": 2}[case]
    lods = [int(l) for l in g[f"{case}_loss_lods"]]
    tr = DR.train(field, g["coords"], g["sdf"].reshape(-1), lods)
    assert tr.amb.mean() < 0.02
    assert abs(tr.loss - g[f"{case}_losses"][0]) <= 1e-6 * tr.loss
    ref_dec = np.concatenate([g[f"{case}_grad1_decoder.{n}.{w}"].reshape(-1) for n in names for w in ("weight", "bias")])
    assert np.abs(tr.dec - ref_dec).max() <= 1e-6 * np.abs(ref_dec).max()
    for k, (c, r) in enumerate(tr.grid):
        ref = g[f"{case}_grad1_grid.features.{k}"]
        assert np.abs(c - ref).max() <= GOLDEN_GRID_TOL * np.abs(ref).max(), k


@pytest.mark.parametrize("layers", [2, 3, 4])
def test_decoder_params_packed_order(layers):
    """ops.decoder_params lists [W0, b0, W1, b1, ..., Wout, bout], so SDFStep's flattened buffer is the kernel's packed layout;
    after the in-place flattening every parameter is a view of its slice."""
    import wisp_b200 as W
    from wisp_b200 import trainers
    from oracle import oracle as O
    from oracle.make_golden import octahedron_points
    blas = W.OctreeAS(torch.from_numpy(O.points_to_octree(octahedron_points(4), 4)))
    grid = W.OctreeGrid(blas, feature_dim=4, num_lods=2, multiscale_type='sum', feature_std=0.1)
    nef = W.NeuralSDF(grid, pos_embedder='none', position_input=True, hidden_dim=8, num_layers=layers)
    lin = list(nef.decoder.layers) + [nef.decoder.lout]
    assert len(lin) == layers + 1
    want = [t for l in lin for t in (l.weight, l.bias)]
    params = W.ops.decoder_params(nef.decoder)
    assert [id(p) for p in params] == [id(p) for p in want]
    packed = torch.cat([t.detach().reshape(-1) for t in want]).clone()
    flat = trainers._flatten_in_place(params)
    assert torch.equal(flat, packed)
    o = 0
    for t in want:
        assert t.data_ptr() == flat[o:o + t.numel()].data_ptr()
        o += t.numel()
    assert o == flat.numel() == 8 * 7 + 8 + (layers - 1) * (8 * 8 + 8) + 8 + 1          # in = 3 (position) + 4 (features)
