"""The hash-grid hook of the float64 interval reference (tests/sdf_hash_reference.py), without a GPU: its fp32 features are the
oracle's hashgrid_fwd bit for bit, with rounding off it is a float64 torch model of HashGrid.interpolate + NeuralSDF.sdf + the L2 loss
and its autograd, and it reproduces the reference trainer's step 1 (tests/golden/sdf_train_hash.npz).  The GPU kernels are checked
inside its intervals in tests/test_gpu_sdf_hash.py."""
import os

import numpy as np
import pytest
import torch

import sdf_hash_reference as H
from oracle import oracle as O
from oracle import sdf_reference as S
import sdf_deep_reference as D


def _field(rng, F=8, ms="cat", layers=1, hidden=16, pos_mode=1, pos_freq=0, bw=10, res=(4, 8, 16, 32), std=0.3):
    begin = O.table_layout(list(res), bw)
    table = (rng.standard_normal((int(begin[-1]), F)) * std).astype(np.float32)
    pd = 0 if pos_mode == 0 else 3 if pos_mode == 1 else 6 * pos_freq + (3 if pos_mode == 3 else 0)
    Ws, bs = S.random_decoder(rng, pd + (F if ms == "sum" else F * len(res)), pos_mode, hidden, layers, scale=0.5)
    return H.hash_field(table, begin, res, bw, ms, Ws, bs, pos_mode, pos_freq)


def _points(rng, n):
    """Points on a 2^-8 lattice below the last cell of the 4-cell level (every coefficient is exact in fp32 there), a few below -1
    (clamped to the first cell), exact -1, duplicates."""
    c = (rng.integers(-256, 128, (n, 3)) / 256.0)
    c[:8] = rng.uniform(-1.6, -1.0, (8, 3)).round(3)
    c[8] = -1.0
    c[-4:] = c[10:14]
    return c.astype(np.float32)


@pytest.mark.parametrize("F,ms", [(8, "cat"), (4, "sum"), (4, "cat"), (8, "sum")])
def test_features_are_oracle_hashgrid_fwd(F, ms):
    rng = np.random.default_rng(1)
    field = _field(rng, F, ms)
    c = np.concatenate([_points(rng, 300), rng.uniform(-1.3, 1.3, (300, 3)).astype(np.float32), [[1, 1, 1], [1, -1, 1]]]).astype(np.float32)
    raw = O.hashgrid_fwd(c, field.table(), field.resolutions, field.bitwidth)
    L = field.num_lods
    for nl in range(1, L + 1):
        got = H.features(field, c, nl)[0]
        if ms == "cat":
            ref = raw.copy(); ref[:, (nl - 1) * F:] = 0
        else:
            ref = np.zeros((c.shape[0], F), np.float32)
            for l in range(L):
                ref = (ref + raw[:, l * F:(l + 1) * F]).astype(np.float32)
        assert np.array_equal(got, ref.astype(np.float64)), nl


def _torch_model(field, c, gt, lods):
    """float64 torch HashGrid.interpolate (hash_grid.py:205-233, hashgrid_interpolate_cuda.cu:38-79) + NeuralSDF.sdf + the L2 loss."""
    table = torch.tensor(field.table(), dtype=torch.float64, requires_grad=True)
    Ws = [torch.tensor(W, dtype=torch.float64, requires_grad=True) for W in field.Ws]
    bs = [torch.tensor(b, dtype=torch.float64, requires_grad=True) for b in field.bs]
    x = torch.tensor(c, dtype=torch.float64)
    begin = O.table_layout(field.resolutions, field.bitwidth)
    T = 2 ** field.bitwidth
    loss = 0.0
    for lod in lods:
        per = []
        for l, res in enumerate(field.resolutions):
            p = (x * 0.5 + 0.5) * res
            p = p.clamp(0.0, float(np.float32(res - 1 - 1e-5)))
            i = torch.floor(p).long(); w = p - i
            f = 0.0
            for j in range(8):
                d = torch.tensor([(j >> 2) & 1, (j >> 1) & 1, j & 1])
                q = i + d
                if res ** 3 < T:
                    idx = q[:, 0] + q[:, 1] * res + q[:, 2] * res * res
                else:
                    idx = (q[:, 0] ^ ((q[:, 1] * H.P1) & 0xFFFFFFFF) ^ ((q[:, 2] * H.P2) & 0xFFFFFFFF)) & (T - 1)
                wt = torch.where(d.bool(), w, 1 - w).prod(-1, keepdim=True)
                f = f + table[int(begin[l]) + idx] * wt
            per.append(f)
        feats = torch.cat(per, -1)
        if field.multiscale == "cat":
            mask = torch.ones(feats.shape[-1], dtype=torch.float64); mask[lod * field.F:] = 0
            feats = feats * mask
        else:
            feats = feats.reshape(-1, field.num_lods, field.F).sum(-2)
        h = torch.cat([x, feats], -1) if field.pos_mode == 1 else feats
        for k in range(len(Ws)):
            h = h @ Ws[k].T + bs[k]
            if k < len(Ws) - 1:
                h = torch.relu(h)
        loss = loss + ((h[:, 0] - torch.tensor(gt, dtype=torch.float64)) ** 2).sum()
    loss = loss / c.shape[0]
    loss.backward()
    dec = torch.cat([t.grad.reshape(-1) for W, b in zip(Ws, bs) for t in (W, b)])
    return float(loss.detach()), dec.numpy(), table.grad.numpy()


@pytest.mark.parametrize("F,ms,layers,pos,lods", [(8, "cat", 1, 1, [3]), (4, "sum", 1, 1, [3]), (8, "cat", 2, 1, [0, 1, 2, 3]),
                                                  (4, "sum", 3, 0, [1]), (8, "cat", 4, 0, [2, 3])])
def test_exact_reference_is_the_float64_model(F, ms, layers, pos, lods):
    rng = np.random.default_rng(2)
    field = _field(rng, F, ms, layers, hidden=8, pos_mode=pos)
    c = _points(rng, 200)
    gt = rng.uniform(-0.5, 0.5, 200)
    tr = D.train(field, c, gt, lods, exact=True)
    loss, dec, tab = _torch_model(field, c, gt, lods)
    assert abs(tr.loss - loss) <= 1e-12 * max(abs(loss), 1)
    assert np.abs(tr.dec - dec).max() <= 1e-12 * max(np.abs(dec).max(), 1)
    assert np.abs(H.table_grad(tr)[0] - tab).max() <= 1e-12 * max(np.abs(tab).max(), 1)


@pytest.mark.parametrize("case", ["cat", "sum", "cat_all", "cat_l2"])
def test_reference_reproduces_hash_golden(golden_dir, case):
    """The reference on the golden's initial parameters reproduces the reference trainer's step-1 loss and decoder gradients to
    1e-6 (relative / of max) and its table gradient to 1e-5 of max."""
    g = np.load(os.path.join(golden_dir, "sdf_train_hash.npz"))
    res = [int(r) for r in g[f"{case}_resolutions"]]
    bw = int(g[f"{case}_codebook_bitwidth"])
    layers = int(g[f"{case}_num_layers"])
    names = [f"decoder.layers.{k}" for k in range(layers)] + ["decoder.lout"]
    Ws = [g[f"{case}_init_{n}.weight"] for n in names]
    bs = [g[f"{case}_init_{n}.bias"] for n in names]
    field = H.hash_field(g[f"{case}_init_grid.codebook.feats"], O.table_layout(res, bw), res, bw, str(g[f"{case}_multiscale"]), Ws, bs)
    lods = [int(l) for l in g[f"{case}_loss_lods"]]
    tr = D.train(field, g["coords"], g["sdf"], lods)
    assert abs(tr.loss - g[f"{case}_losses"][0]) <= 1e-6 * g[f"{case}_losses"][0]
    ref_dec = np.concatenate([g[f"{case}_grad1_{n}.{t}"].reshape(-1) for n in names for t in ("weight", "bias")])
    assert np.abs(tr.dec - ref_dec).max() <= 1e-6 * np.abs(ref_dec).max()
    ref_tab = g[f"{case}_grad1_grid.codebook.feats"]
    assert np.abs(H.table_grad(tr)[0] - ref_tab).max() <= 1e-5 * np.abs(ref_tab).max()
