"""CPU tests of tests/composite_reference.py, the float64 interval reference of wb_composite_fwd / wb_composite_bwd /
wb_composite_bwd_loss and wb_adam_step:
  - with rounding off it IS the operation: float64 torch autograd of oracle/torch_twin.py's exponential_integration / sum_reduce
    formulas, torch's mse / l1 / smooth_l1 losses (d = 0 and |d| = 1 included) and torch.optim.Adam, to 1e-12;
  - fp32 restatements of the kernels with random summation orders and expf off by up to 2 ulp land inside its intervals, and
    the bit-exact Adam emulation lands inside the Adam interval;
  - a subtly wrong kernel (inclusive transmittance, carry dropped after the first chunk, T_k in place of T_{k+1}, no bg term in
    dL/dalpha, no inv_count, huber with the l1 gradient, Adam without the v bias correction, AdamW's decoupled decay) lands outside
    on at least one element at the shapes the GPU tests use;
  - the radii are tight: their medians stay below about twice what this file prints."""
import numpy as np
import pytest
import torch

from oracle import torch_twin as TT

import composite_reference as CR

f32 = np.float32


def _case(R=205, regime="mixed", seed=0):
    rng = np.random.default_rng(seed)
    return CR.make_case(CR.ray_lengths(R, rng), regime, seed)


def _grads(R, seed=1):
    rng = np.random.default_rng(seed)
    return (rng.standard_normal((R, 3)).astype(f32), rng.standard_normal(R).astype(f32), rng.standard_normal(R).astype(f32))


def _inside(k, c, r):
    return np.abs(np.asarray(k, np.float64) - c) <= r


# ---- rounding off == the float64 operation ------------------------------------------------------------------------------------
def _torch_composite(case, bg, g_rgb, g_depth, g_alpha):
    """float64 autograd of PackedRFTracer's compositing through torch_twin's formulas -> rgb, depth, alpha, dL/dshaded."""
    old = torch.get_default_dtype()
    torch.set_default_dtype(torch.float64)              # torch_twin.sum_reduce allocates with the default dtype
    try:
        return _torch_composite64(case, bg, g_rgb, g_depth, g_alpha)
    finally:
        torch.set_default_dtype(old)


def _torch_composite64(case, bg, g_rgb, g_depth, g_alpha):
    n = case["n"]
    sh = torch.tensor(case["shaded"], dtype=torch.float64, requires_grad=True)
    dl = torch.tensor(case["deltas"], dtype=torch.float64)[:, None]
    t = torch.tensor(case["depth"], dtype=torch.float64)[:, None]
    R = n.shape[0]
    rgb = torch.tensor(np.asarray(bg, np.float64)).expand(R, 3).clone()
    depth, alpha = torch.zeros(R, 1, dtype=torch.float64), torch.zeros(R, 1, dtype=torch.float64)
    hitr = torch.from_numpy(np.nonzero(n > 0)[0])
    if sh.shape[0]:
        ridx = torch.from_numpy(np.repeat(np.arange(R), n))
        boundary = torch.ones_like(ridx, dtype=torch.bool)
        boundary[1:] = ridx[1:] != ridx[:-1]
        tau = sh[:, 3:4] * dl
        ray_colors, w = TT.exponential_integration(sh[:, :3], tau, boundary)
        ray_depth = TT.sum_reduce(t * w, boundary)
        a = TT.sum_reduce(w, boundary)
        bgt = torch.tensor(np.asarray(bg, np.float64))
        rgb = rgb.index_put((hitr,), bgt * (1.0 - a) + ray_colors)
        depth = depth.index_put((hitr,), ray_depth)
        alpha = alpha.index_put((hitr,), a)
    L = (rgb * torch.from_numpy(g_rgb.astype(np.float64))).sum() + (depth[:, 0] * torch.from_numpy(g_depth.astype(np.float64))).sum() \
        + (alpha[:, 0] * torch.from_numpy(g_alpha.astype(np.float64))).sum()
    if sh.shape[0]:
        L.backward()
    g = sh.grad.numpy() if sh.grad is not None else np.zeros_like(case["shaded"], np.float64)
    return rgb.detach().numpy(), depth.detach().numpy()[:, 0], alpha.detach().numpy()[:, 0], g


def _close(a, b, tol=1e-12):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return np.abs(a - b).max(initial=0.0) <= tol * max(1.0, np.abs(b).max(initial=0.0))


@pytest.mark.parametrize("regime", ["mixed", "zero", "opaque", "huge", "delta0"])
def test_exact_reference_is_torch_autograd(regime):
    case = _case(R=70, regime=regime, seed=3)
    bg = (0.25, 0.5, 0.75)
    gr, gd, ga = _grads(70)
    rgb, depth, alpha, g = _torch_composite(case, bg, gr, gd, ga)
    fw = CR.forward(case["offsets"], case["shaded"], case["depth"], case["deltas"], bg, exact=True)
    assert _close(fw.rgb, rgb) and _close(fw.depth, depth) and _close(fw.alpha, alpha)
    bw = CR.backward(case["offsets"], case["shaded"], case["depth"], case["deltas"], bg, gr, gd, ga, exact=True)
    assert _close(bw.g, g)
    assert np.all(fw.rgb_r == 0) and np.all(bw.r == 0)


@pytest.mark.parametrize("loss_type", ["l2", "l1", "huber"])
def test_exact_loss_is_torch(loss_type):
    """dL/drgb and the loss value against torch's losses on a leaf rgb, with d = 0, +-1 exactly and |d| around 1."""
    rng = np.random.default_rng(5)
    R = 64
    rgb = (rng.integers(0, 1024, (R, 3)) / 1024.0).astype(f32)
    tgt = (rgb + rng.choice([0.0, 1.0, -1.0, 0.5, -2.0, 0.999, 1.001], (R, 3))).astype(f32)
    inv = 1.0 / (3 * R)
    x = torch.tensor(rgb, dtype=torch.float64, requires_grad=True)
    y = torch.tensor(tgt, dtype=torch.float64)
    l = {"l2": lambda: torch.nn.functional.mse_loss(x, y, reduction='none'), "l1": lambda: torch.abs(x - y),
         "huber": lambda: torch.nn.functional.smooth_l1_loss(x, y, reduction='none')}[loss_type]()
    val = l.sum() * inv
    val.backward()
    t = CR.LOSS_TYPES[loss_type]
    assert _close(CR.loss_grad(rgb, tgt, t, inv, exact=True), x.grad.numpy())
    c, r = CR.loss_value(rgb, tgt, t, inv, R, exact=True)
    assert r == 0 and abs(c - float(val)) <= 1e-12 * max(1.0, abs(float(val)))


@pytest.mark.parametrize("wd,step", [(0.0, 1), (1e-2, 2), (0.0, 10000), (1e-2, 7)])
def test_exact_adam_is_torch(wd, step):
    rng = np.random.default_rng(step)
    n = 257
    p = rng.standard_normal(n)
    m, v = rng.standard_normal(n) * 1e-2, rng.random(n) * 1e-4
    g = rng.standard_normal(n) * 0.1
    lr, b1, b2, eps = 1e-3, 0.9, 0.99, 1e-8
    pt = torch.tensor(p, requires_grad=True)
    opt = torch.optim.Adam([pt], lr=lr, betas=(b1, b2), eps=eps, weight_decay=wd)
    pt.grad = torch.tensor(g)
    opt.step()                                              # builds the state at step 1 ...
    st = opt.state[pt]
    with torch.no_grad():                                   # ... then step `step` from (p, m, v)
        pt.copy_(torch.tensor(p)); st["exp_avg"].copy_(torch.tensor(m)); st["exp_avg_sq"].copy_(torch.tensor(v))
        st["step"].fill_(step - 1)
    opt.step()
    (pc, pr), (mc, mr), (vc, vr) = CR.adam(p, g, m, v, lr, wd, b1, b2, eps, step, exact=True)
    assert pr.max() == 0 and _close(pc, pt.detach().numpy()) and _close(mc, st["exp_avg"].numpy()) and _close(vc, st["exp_avg_sq"].numpy())


# ---- fp32 restatements land inside --------------------------------------------------------------------------------------------
def _perturbed_exp(x, rng):
    """expf(x) off by up to 2 ulp."""
    e = np.exp(np.asarray(x, np.float64)).astype(f32)
    k = rng.integers(-2, 3, e.shape)
    for s in (1, 2):
        e = np.where(k >= s, np.nextafter(e, f32(np.inf)), np.where(k <= -s, np.nextafter(e, f32(0)), e))
    return np.maximum(e, f32(0))


def _rsum(x, rng):
    """fp32 sum in a random order."""
    x = np.asarray(x, f32)[rng.permutation(len(x))]
    s = f32(0)
    for v in x:
        s = f32(s + v)
    return s


def _emulate(case, bg, gr, gd, ga, rng, loss=None):
    """fp32 restatement of wb_composite_fwd / _bwd (/ _bwd_loss: loss = (target, type, inv)) with the kernels' prefixes, expf off
    by up to 2 ulp and every sum in a random order -> rgb, depth, alpha, g_shaded, loss value."""
    off, sh, dl, t = case["offsets"], case["shaded"], case["deltas"], case["depth"]
    pk = CR.packed(off)
    tau = sh[:, 3] * dl
    xe, xi = CR.prefixes(pk, tau)
    T, Tn = _perturbed_exp(-xe, rng), _perturbed_exp(-xi, rng)
    w = np.where(tau == 0, f32(0), T * (f32(1) - _perturbed_exp(-tau.astype(np.float64), rng)))
    bgv = np.asarray(bg, f32)
    R = pk.R
    rgb = np.tile(bgv, (R, 1)); depth = np.zeros(R, f32); alpha = np.zeros(R, f32)
    g = np.zeros((pk.S, 4), f32)
    lsum = []
    for r in range(R):
        b, e = off[r], off[r + 1]
        if e > b:
            ws = w[b:e]
            A = _rsum(ws, rng)
            C = [_rsum(ws * sh[b:e, c], rng) for c in range(3)]
            rgb[r] = [f32(bgv[c] * f32(f32(1) - A) + C[c]) for c in range(3)]
            depth[r], alpha[r] = _rsum(ws * t[b:e], rng), A
    if loss is not None:                                    # dL/drgb from the rgb buffer the caller passes (the forward's output)
        rgb_in, tgt, ty, inv = loss
        d = np.asarray(rgb_in, f32) - np.asarray(tgt, f32)
        gr = CR.loss_grad(rgb_in, tgt, ty, inv).astype(f32)
        gd, ga = np.zeros(R, f32), np.zeros(R, f32)
        ad = np.abs(d).astype(np.float64)
        terms = (d * d if ty == 0 else np.abs(d) if ty == 1 else np.where(ad < 1, f32(0.5) * d * d, np.abs(d) - f32(0.5))).astype(f32)
        lsum = f32(_rsum(terms.reshape(-1), rng) * f32(inv))
    for r in range(R):
        b, e = off[r], off[r + 1]
        if e == b:
            continue
        gaa = f32(ga[r] - f32(f32(gr[r, 0] * bgv[0] + gr[r, 1] * bgv[1]) + gr[r, 2] * bgv[2]))
        gk = (f32(gr[r, 0]) * sh[b:e, 0] + f32(gr[r, 1]) * sh[b:e, 1] + f32(gr[r, 2]) * sh[b:e, 2] + f32(gd[r]) * t[b:e] + gaa).astype(f32)
        gw = (gk * w[b:e]).astype(f32)
        G = _rsum(gw, rng)
        P = np.cumsum(gw, dtype=f32)
        suffix = (G - P).astype(f32)
        gtau = (gk * Tn[b:e] - suffix).astype(f32)
        g[b:e, :3] = (gr[r][None, :].astype(f32) * w[b:e, None]).astype(f32)
        g[b:e, 3] = gtau * dl[b:e]
    return rgb, depth, alpha, g, lsum


@pytest.mark.parametrize("regime", CR.REGIMES)
@pytest.mark.parametrize("bg", [(0.0, 0.0, 0.0), (1.0, 1.0, 1.0), (0.3, 0.6, 0.1)])
def test_fp32_restatement_is_inside(regime, bg):
    case = _case(R=140, regime=regime, seed=7)
    gr, gd, ga = _grads(140, seed=8)
    rng = np.random.default_rng(9)
    for rep in range(2):
        rgb, depth, alpha, g, _ = _emulate(case, bg, gr, gd, ga, rng)
        fw = CR.forward(case["offsets"], case["shaded"], case["depth"], case["deltas"], bg)
        assert _inside(rgb, fw.rgb, fw.rgb_r).all() and _inside(depth, fw.depth, fw.depth_r).all() and _inside(alpha, fw.alpha, fw.alpha_r).all()
        assert CR.hit_ok(fw.alpha, fw.alpha_r, alpha > 0, alpha).all()
        bw = CR.backward(case["offsets"], case["shaded"], case["depth"], case["deltas"], bg, gr, gd, ga)
        assert _inside(g, bw.g, bw.r).all(), np.argwhere(~_inside(g, bw.g, bw.r))[:5]


@pytest.mark.parametrize("loss_type", [0, 1, 2])
def test_fp32_loss_restatement_is_inside(loss_type):
    case = _case(R=140, seed=11)
    bg = (0.3, 0.6, 0.1)
    fw = CR.forward(case["offsets"], case["shaded"], case["depth"], case["deltas"], bg)
    rgb32 = fw.rgb.astype(f32)
    rng = np.random.default_rng(12)
    tgt = (rgb32 + rng.choice([0.0, 1.0, -1.0, 0.25, -3.0], rgb32.shape)).astype(f32)
    inv = float(f32(1.0 / (3 * 140)))
    _, _, _, g, lv = _emulate(case, bg, None, None, None, rng, loss=(rgb32, tgt, loss_type, inv))
    gl = CR.loss_grad(rgb32, tgt, loss_type, inv)
    bw = CR.backward(case["offsets"], case["shaded"], case["depth"], case["deltas"], bg, gl)
    assert _inside(g, bw.g, bw.r).all()
    c, r = CR.loss_value(rgb32, tgt, loss_type, inv, 140)
    assert abs(float(lv) - c) <= r


@pytest.mark.parametrize("wd,eps,gscale,step", [(0.0, 1e-8, 1.0, 1), (1e-2, 1e-15, 1e-12, 2), (1e-2, 1e-8, 0.25, 10000), (0.0, 1e-15, 1e-14, 3)])
def test_adam_fp32_emulation_is_inside(wd, eps, gscale, step):
    rng = np.random.default_rng(2)
    n = 4099
    p = rng.standard_normal(n).astype(f32)
    g = (rng.standard_normal(n) * gscale).astype(f32)
    g[:7] = 0.0
    m = (rng.standard_normal(n) * gscale * 0.1).astype(f32)
    v = (rng.random(n) * gscale * gscale * 0.01).astype(f32)
    p_sep, p_fma, m1, v1 = CR.adam_fp32(p, g, m, v, 1e-3, wd, 0.9, 0.999, eps, step)
    (pc, pr), (mc, mr), (vc, vr) = CR.adam(p, g, m, v, 1e-3, wd, 0.9, 0.999, eps, step)
    assert _inside(p_sep, pc, pr).all() and _inside(p_fma, pc, pr).all()
    assert _inside(m1, mc, mr).all() and _inside(v1, vc, vr).all()


# ---- mutations land outside ---------------------------------------------------------------------------------------------------
def _naive(case, bg, gr, gd, ga, *, inclusive=False, no_carry=False, tk_in_gtau=False, no_bg=False):
    """float64 restatement of the kernels on their fp32 prefixes, with one defect switched on -> rgb, g_shaded."""
    pk = CR.packed(case["offsets"])
    sh = case["shaded"].astype(np.float64)
    tau32 = case["shaded"][:, 3] * case["deltas"]
    tau = tau32.astype(np.float64)
    xe, xi = CR.prefixes(pk, tau32)
    if no_carry:                                            # the prefix restarts at every 32-sample chunk
        incl = CR.warp_scan(pk, tau32)
        xe, xi = (incl - tau32).astype(np.float64), incl.astype(np.float64)
    T = np.exp(-(xi if inclusive else xe))
    Tn = np.exp(-xi)
    w = T * (1 - np.exp(-tau))
    A = CR.seg_sum(pk, w)
    bgv = np.asarray(bg, f32).astype(np.float64)
    rgb = np.stack([bgv[c] * (1 - A) + CR.seg_sum(pk, w * sh[:, c]) for c in range(3)], 1)
    s = pk.ray
    gaa = ga - (0.0 if no_bg else gr.astype(np.float64) @ bgv)
    gk = (gr[s] * sh[:, :3]).sum(1) + gd[s] * case["depth"] + gaa[s]
    prod = gk * w
    suffix = CR.seg_sum(pk, prod)[s] - CR.seg_cumsum(pk, prod)
    gtau = gk * (T if tk_in_gtau else Tn) - suffix
    g = np.concatenate([gr[s] * w[:, None], (gtau * case["deltas"])[:, None]], 1)
    return rgb, g


GPU_SHAPES = [dict(R=205, seed=0), dict(R=1, seed=1, n=[2048]), dict(R=17, seed=2)]


def _gpu_case(sh):
    if "n" in sh:
        return CR.make_case(sh["n"], "mixed", sh["seed"])
    return _case(R=sh["R"], seed=sh["seed"])


@pytest.mark.parametrize("defect", ["inclusive", "no_carry", "tk_in_gtau", "no_bg"])
def test_composite_defects_land_outside(defect):
    """Over the GPU shapes together (a single opaque ray cannot show the bg term: it enters through the ray's final transmittance)."""
    bg = (0.3, 0.6, 0.1)
    caught = []
    for sh in GPU_SHAPES:
        case = _gpu_case(sh)
        R = case["n"].shape[0]
        gr, gd, ga = _grads(R)
        if defect == "no_carry" and case["n"].max() <= 32:
            continue
        fw = CR.forward(case["offsets"], case["shaded"], case["depth"], case["deltas"], bg)
        bw = CR.backward(case["offsets"], case["shaded"], case["depth"], case["deltas"], bg, gr, gd, ga)
        ok_rgb, ok_g = _naive(case, bg, gr, gd, ga)
        assert _inside(ok_rgb, fw.rgb, fw.rgb_r).all() and _inside(ok_g, bw.g, bw.r).all()
        bad_rgb, bad_g = _naive(case, bg, gr, gd, ga, **{defect: True})
        caught.append(not (_inside(bad_rgb, fw.rgb, fw.rgb_r).all() and _inside(bad_g, bw.g, bw.r).all()))
    assert any(caught), defect


@pytest.mark.parametrize("defect", ["no_inv_count", "huber_l1_grad"])
def test_loss_defects_land_outside(defect):
    case = _case(R=205, seed=0)
    bg = (0.3, 0.6, 0.1)
    fw = CR.forward(case["offsets"], case["shaded"], case["depth"], case["deltas"], bg)
    rgb32 = fw.rgb.astype(f32)
    rng = np.random.default_rng(4)
    tgt = (rgb32 + rng.uniform(-0.5, 0.5, rgb32.shape)).astype(f32)
    inv = float(f32(1.0 / (3 * 205)))
    gl = CR.loss_grad(rgb32, tgt, 2, inv)
    bw = CR.backward(case["offsets"], case["shaded"], case["depth"], case["deltas"], bg, gl)
    d = (rgb32 - tgt).astype(np.float64)
    bad = d if defect == "no_inv_count" else np.sign(d) * inv
    bad_g = CR.backward(case["offsets"], case["shaded"], case["depth"], case["deltas"], bg, bad, exact=True).g
    assert not _inside(bad_g, bw.g, bw.r).all()


@pytest.mark.parametrize("defect", ["no_v_bias", "adamw"])
def test_adam_defects_land_outside(defect):
    rng = np.random.default_rng(3)
    n, lr, wd, b1, b2, eps = 1000003, 1e-3, 1e-2, 0.9, 0.999, 1e-8
    p = rng.standard_normal(n).astype(f32)
    g = rng.standard_normal(n).astype(f32)
    m = (rng.standard_normal(n) * 0.1).astype(f32)
    v = (rng.random(n) * 0.01).astype(f32)
    for step in (1, 2, 10000):
        (pc, pr), _, _ = CR.adam(p, g, m, v, lr, wd, b1, b2, eps, step)
        bc1, bc2s = CR.bias_corrections(b1, b2, step, exact=True)
        if defect == "no_v_bias":
            (bad, _), _, _ = CR.adam(p, g, m, v, lr, wd, b1, b2, eps, step, exact=True, bc=(bc1, 1.0))
        else:                                               # p *= 1 - lr wd, then Adam on the raw gradient
            (bad, _), _, _ = CR.adam(p.astype(np.float64) * (1 - lr * wd), g, m, v, lr, 0.0, b1, b2, eps, step, exact=True)
        if step == 10000 and defect == "no_v_bias":
            continue                                        # 1 - b2^t = 1 - 4.5e-5: the defect moves p by less than a rounding
        assert not _inside(bad, pc, pr).all(), step


# ---- tightness ------------------------------------------------------------------------------------------------------------------
def _med_rel(c, r):
    """median of r / |c| over the entries above 1e-6 of the largest (the opaque tails' weights are below every rounding)."""
    big = np.abs(c) > 1e-6 * np.abs(c).max()
    return float(np.median(r[big] / np.abs(c[big])))


def test_radii_are_tight():
    """Median radius per output relative to the output's scale; thresholds at about twice what this prints."""
    case = _case(R=205, seed=0)
    bg = (0.3, 0.6, 0.1)
    gr, gd, ga = _grads(205)
    fw = CR.forward(case["offsets"], case["shaded"], case["depth"], case["deltas"], bg)
    bw = CR.backward(case["offsets"], case["shaded"], case["depth"], case["deltas"], bg, gr, gd, ga)
    hit = case["n"] > 0
    rel = {"rgb": np.median(fw.rgb_r[hit] / np.abs(fw.rgb[hit]).max()),
           "depth": np.median(fw.depth_r[hit] / np.abs(fw.depth[hit]).max()),
           "alpha": np.median(fw.alpha_r[hit]),
           "g_rgb": _med_rel(bw.g[:, :3], bw.r[:, :3]),
           "g_sigma": _med_rel(bw.g[:, 3], bw.r[:, 3])}
    p = np.random.default_rng(0).standard_normal(4099).astype(f32)
    (pc, pr), (mc, mr), (vc, vr) = CR.adam(p, p * 0.1, p * 0.01, np.abs(p) * 1e-3, 1e-3, 1e-2, 0.9, 0.999, 1e-8, 3)
    rel["adam_p"] = np.median(pr / np.abs(pc))
    rel["adam_m"] = np.median(mr / np.abs(mc))
    print("CRTIGHT " + " ".join(f"{k}={v:.3g}" for k, v in rel.items()))
    limits = {"rgb": 5e-6, "depth": 5e-6, "alpha": 5e-6, "g_rgb": 2.2e-5, "g_sigma": 5.2e-4, "adam_p": 1.2e-7, "adam_m": 3.8e-7}
    for k, v in rel.items():
        assert v <= limits[k], (k, v)
