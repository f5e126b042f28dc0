"""CPU checks of tests/sdf_tc_reference.py, the fp16-faithful reference of the precision-1 SDF training step: with rounding off it
is the float64 autograd gradient; its centre is a torch CPU emulation with explicit .half() casts at the rounding points; and the
footprint it documents is the library's wb_sdf_train_tc_smem_bytes, at the boundary too."""
import ctypes as C

import numpy as np
import pytest
import torch

import sdf_tc_reference as TR
from sdf_deep_shapes import make_field as make_deep
from sdf_shapes import make_field, points


def _torch_train(field, coords, gt, lod, dtype, half):
    """The decoder part of the step in torch autograd: x (position | features) is a leaf, so dL/dx is the feature gradient."""
    from oracle import sdf_reference as S
    pc, _ = S._embed(field, coords.astype(np.float64), not half)
    fc, _, _, _ = S.features(field, coords, lod + 1, exact=not half)
    cast = (lambda t: t.half().to(dtype)) if half else (lambda t: t)
    x = cast(torch.tensor(np.concatenate([pc, fc], -1), dtype=dtype)).requires_grad_(True)
    Ws = [torch.tensor(W, dtype=dtype, requires_grad=True) for W in field.Ws]
    bs = [torch.tensor(b, dtype=dtype, requires_grad=True) for b in field.bs]
    h = x
    for W, b in zip(Ws[:-1], bs[:-1]):
        h = cast(torch.relu(h @ cast(W).T + cast(b)))
    y = cast(h @ cast(Ws[-1]).T + cast(bs[-1]))[:, 0]
    loss = ((y - torch.tensor(gt, dtype=dtype)) ** 2).sum() / coords.shape[0]
    if half:
        # autocast's fp16 backward, with the kernel's power-of-two loss scale on dY and fp32 feature gradients
        scale = TR.loss_scale(1.0 / coords.shape[0])
        y.register_hook(lambda g: cast(g * scale))
        loss.backward()
        return float(loss.detach()), [p.grad.double().numpy() / scale for pair in zip(Ws, bs) for p in pair], x.grad.double().numpy()[:, field.pos_dim:] / scale
    loss.backward()
    return float(loss.detach()), [p.grad.double().numpy() for pair in zip(Ws, bs) for p in pair], x.grad.double().numpy()[:, field.pos_dim:]


@pytest.mark.parametrize("name,deep", [("config3", False), ("sum_pos3", False), ("cat_id", False), ("l2_h128", True), ("l2_h64", True)])
def test_rounding_off_is_float64_autograd(name, deep):
    field, case = (make_deep if deep else make_field)(name)
    coords, gt = points(case, 300)
    lod = field.num_lods - 1
    ref = TR.train_tc(field, coords, gt, [lod], rounding=False)
    loss, grads, dx = _torch_train(field, coords, gt, lod, torch.float64, False)
    assert abs(ref.loss - loss) <= 1e-12 * abs(loss)
    got = np.concatenate([g.reshape(-1) for g in grads])
    assert np.abs(ref.dec - got).max() <= 1e-12 * np.abs(got).max()
    assert np.abs(ref.dfeat[0][0] - dx).max() <= 1e-12 * max(np.abs(dx).max(), 1e-300)


@pytest.mark.parametrize("name,deep", [("config3", False), ("cat_id", False), ("l2_h128", True)])
def test_torch_half_emulation_inside_intervals(name, deep):
    """torch float32 on the CPU with .half() at every rounding point lies inside the intervals (samples whose relu mask the
    intervals leave open dropped)."""
    field, case = (make_deep if deep else make_field)(name)
    coords, gt = points(case, 500)
    lod = field.num_lods - 1
    ref = TR.train_tc(field, coords, gt, [lod], rounding=True)
    coords, gt = coords[~ref.amb], gt[~ref.amb]                         # a relu decision float32 may take either way
    ref = TR.train_tc(field, coords, gt, [lod], rounding=True)
    loss, grads, dx = _torch_train(field, coords, gt, lod, torch.float32, True)
    # the emulation is one more kernel of the contract (its fp32 sums are taller than the kernel's: 1e-4 of max on top)
    assert abs(ref.loss - loss) <= ref.loss_r + 1e-6 * abs(loss)
    got = np.concatenate([g.reshape(-1) for g in grads])
    assert (np.abs(ref.dec - got) <= ref.dec_r + 1e-4 * np.abs(got).max()).all()
    fc, fr = ref.dfeat[0]
    assert (np.abs(fc - dx) <= fr + 1e-4 * np.abs(dx).max()).all()
    exact = TR.train_tc(field, coords, gt, [lod], rounding=False)
    assert ref.loss != exact.loss                                        # the rounding points do something


def _desc(in_feat, F, ms, num_lods, pos_mode, pos_freq, H, nh):
    from wisp_b200 import _cabi as A
    d = A.SdfDesc()
    d.points = d.trinkets = d.params = 16                                # host-only: never dereferenced
    ptrs = (C.c_void_p * num_lods)(*([16] * num_lods))
    d.feats = ptrs
    d.feature_dim, d.num_lods, d.multiscale, d.base_lod, d.half_round = F, num_lods, ms, 2, 1
    d.pos_mode, d.pos_freq, d.num_layers, d.hidden_dim = pos_mode, pos_freq, nh, H
    return d, ptrs


@pytest.mark.parametrize("F,ms,L,pm,pf,H,nh", [
    (16, 1, 6, 1, 0, 128, 1),        # config 3: 19-128-1
    (16, 1, 6, 1, 0, 128, 2),        # 19-128-128-1: about 180 KB
    (16, 1, 6, 1, 0, 128, 3),        # three hidden layers of 128: over 227 KB
    (16, 1, 6, 1, 0, 96, 3),         # fits
    (16, 1, 6, 1, 0, 112, 3),        # the boundary of three layers at in 19
    (8, 0, 4, 1, 0, 128, 1),         # nglod_hash-like in 35
    (21, 0, 5, 3, 4, 128, 2),        # in 132 -> K 144
    (4, 1, 6, 0, 0, 30, 1),          # H padded to 32
    (16, 1, 6, 1, 0, 80, 2),         # Hp 80: the dY tile holds two 64-output passes (16 slabs)
    (4, 1, 6, 0, 0, 96, 1),          # Hp 96
])
def test_footprint_matches_library(F, ms, L, pm, pf, H, nh):
    from wisp_b200 import _cabi as A
    d, keep = _desc(None, F, ms, L, pm, pf, H, nh)
    pos = 0 if pm == 0 else 3 if pm == 1 else 6 * pf + (3 if pm == 3 else 0)
    feat = F if ms else F * L
    want = TR.footprint(pos + feat, pos, feat, H, nh)
    got = int(A.lib().wb_sdf_train_tc_smem_bytes(C.byref(d)))
    assert got == want, (got, want)
    if (F, H, nh) == (16, 128, 2):
        assert 170 * 1024 < got <= 227 * 1024
    if (H, nh) == (128, 3):
        assert got < 0


def test_rounding_off_has_zero_radius():
    field, case = make_deep("l2_h64")
    coords, gt = points(case, 200)
    ref = TR.train_tc(field, coords, gt, [field.num_lods - 1], rounding=False)
    assert ref.loss_r == 0 and not ref.dec_r.any() and not any(r.any() for _, r in ref.grid)


def test_footprint_boundary_is_exact():
    """The widest three-layer decoder at in 19 that fits, and the next multiple of 16 that does not."""
    fits = [H for H in range(16, 129, 16) if TR.footprint(19, 3, 16, H, 3) > 0]
    assert fits and fits[-1] < 128
    assert TR.footprint(19, 3, 16, fits[-1] + 16, 3) < 0


def test_loss_scale():
    for N in (1, 2, 3, 512, 1000, 65536, 1 << 20):
        s = TR.loss_scale(1.0 / N)
        assert 0.5 <= s / N < 1.0 and s == 2.0 ** round(np.log2(s))
