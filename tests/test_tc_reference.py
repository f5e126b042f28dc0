"""CPU checks of oracle/tc_decoders.py, the fp16-faithful interval reference of the tensor-core decoders (no GPU needed).

  - with every rounding and gamma off the radius is 0 and the reference is the float64 MLP and its autograd (pins the backward
    algebra: the colour-input split, relu' from the retained activation, the density relu', the loss scale);
  - soundness: emulations of other valid kernels (fp32 accumulation in random orders, fp16 roundings at the same points) land
    inside the intervals;
  - tightness: on typical inputs the radius is far below the end-to-end tolerances of tests/test_gpu_parity.py (TOL[1]).
"""
import numpy as np
import pytest
import torch

from oracle import tc_decoders as T

TOL1_RGB, TOL1_GRAD = 2e-3, 3e-2          # tests/test_gpu_parity.py TOL[1]


def make_case(seed, dens_dims, col_hidden, view_mode=3, view_freq=2, bias=True, S=96, x_scale=0.5):
    rng = np.random.default_rng(seed)
    dout = dens_dims[-1]
    vd = 0 if view_mode == 0 else 3 if view_mode == 1 else 3 + 6 * view_freq
    col_dims = [dout - 1 + vd] + list(col_hidden) + [3]

    def mlp(dims):
        Ws = [rng.uniform(-1, 1, (o, i)).astype(np.float32) / np.sqrt(i) for i, o in zip(dims[:-1], dims[1:])]
        bs = [rng.uniform(-1, 1, o).astype(np.float32) / np.sqrt(i) for i, o in zip(dims[:-1], dims[1:])] if bias else None
        return Ws, bs
    dW, db = mlp(dens_dims)
    cW, cb = mlp(col_dims)
    if bias:
        db[-1][0] = 0.2
    dec = T.Decoders(dW, db, cW, cb)
    X0 = T.f16(rng.standard_normal((S, dens_dims[0])) * x_scale)
    X0[:5] = 0.0                                                   # exact zeros
    dirs = rng.standard_normal((S, 3)).astype(np.float32)
    dirs /= np.linalg.norm(dirs, axis=1, keepdims=True)
    go = (rng.standard_normal((S, 4)) * 1e-3).astype(np.float32)
    return dec, X0, dirs, go, view_mode, view_freq


def torch_mlp(dec, X0, view, go, planes, width):
    """float64 forward + autograd of the same decoders."""
    t = lambda a: torch.tensor(np.asarray(a, np.float64), requires_grad=True)
    dW, cW = [t(w) for w in dec.dens_W], [t(w) for w in dec.col_W]
    db = [t(b) for b in dec.dens_b] if dec.dens_b is not None else None
    cb = [t(b) for b in dec.col_b] if dec.col_b is not None else None
    x = t(X0)
    h = x
    for l in range(len(dW)):
        h = h @ dW[l].T + (db[l] if db else 0)
        if l < len(dW) - 1:
            h = torch.relu(h)
    df = h
    h = torch.cat([df[:, 1:dec.dout], torch.tensor(view)], 1)
    for l in range(len(cW)):
        h = h @ cW[l].T + (cb[l] if cb else 0)
        if l < len(cW) - 1:
            h = torch.relu(h)
    rgb, sigma = torch.sigmoid(h), torch.relu(df[:, 0])
    g = torch.tensor(go, dtype=torch.float64)
    ((rgb * g[:, :3]).sum() + (sigma * g[:, 3]).sum()).backward()

    def flat(Ws, bs):
        parts = []
        for i, w in enumerate(Ws):
            parts.append(w.grad.reshape(-1))
            if bs:
                parts.append(bs[i].grad.reshape(-1))
        return torch.cat(parts).numpy()
    dfeat = x.grad[:, :planes * width].numpy().reshape(-1, planes, width).transpose(1, 0, 2)
    return rgb.detach().numpy(), sigma.detach().numpy(), flat(dW, db), flat(cW, cb), dfeat


@pytest.mark.parametrize("dens_dims,col_hidden,view_mode,bias", [([32, 64, 16], [64, 64], 3, True), ([20, 24, 9], [40], 1, False),
                                                                   ([12, 2], [16, 24, 8], 0, True), ([36, 16], [128, 24], 3, True)])
def test_exact_mode_is_the_float64_mlp(dens_dims, col_hidden, view_mode, bias):
    dec, X0, dirs, go, vm, vf = make_case(1, dens_dims, col_hidden, view_mode=view_mode, bias=bias)
    view = T.view_embedding(dirs, vm, vf, exact=True)
    ref = T.Reference(dec, X0, view, rounding=False, accumulation=False)
    planes, width = dens_dims[0] // 4, 4
    scale = 8.0
    bw = ref.backward(go, scale, planes, width)
    rgb, sigma, gd, gc, dfeat = torch_mlp(dec, X0, view[0], go, planes, width)
    c, r = ref.shaded()
    assert np.all(r == 0) and all(np.all(bw[k][1] == 0) for k in ("dens", "col", "dfeat"))
    np.testing.assert_allclose(c[:, :3], rgb, rtol=0, atol=1e-12)
    np.testing.assert_allclose(c[:, 3], sigma, rtol=0, atol=1e-12)
    for got, want in ((bw["dens"][0], gd), (bw["col"][0], gc), (bw["dfeat"][0], dfeat * scale)):
        assert got.shape == want.shape
        assert np.abs(got - want).max() <= 1e-12 * max(1.0, np.abs(want).max())


# ---- emulation of another valid kernel: same fp16 rounding points, fp32 sums in random orders ----------------------------
def _fp32_sum(terms, rng):
    """terms [..., K] (each exactly representable in fp32) -> fp32 sequential sum in a random order per output element."""
    perm = np.argsort(rng.random(terms.shape), axis=-1)
    t = np.take_along_axis(terms, perm, axis=-1).astype(np.float32)
    acc = np.zeros(terms.shape[:-1], np.float32)
    for k in range(terms.shape[-1]):
        acc = (acc + t[..., k]).astype(np.float32)
    return acc.astype(np.float64)


def _lin32(x, W, b, rng):
    terms = x[:, None, :] * W[None, :, :]
    if b is not None:
        terms = np.concatenate([terms, np.broadcast_to(b[None, :, None], terms.shape[:2] + (1,))], axis=-1)
    return _fp32_sum(terms, rng)


def emulate(dec, X0, view16, go, scale, planes, width, rng):
    q = T.f16
    dW, cW = [q(w) for w in dec.dens_W], [q(w) for w in dec.col_W]
    db = [q(b) for b in dec.dens_b] if dec.dens_b is not None else [None] * len(dW)
    cb = [q(b) for b in dec.col_b] if dec.col_b is not None else [None] * len(cW)
    xs_d, xs_c = [], []
    h = X0
    for l in range(len(dW)):
        xs_d.append(h)
        h = _lin32(h, dW[l], db[l], rng)
        if l < len(dW) - 1:
            h = q(np.maximum(h, 0))
    df = h
    h = np.concatenate([q(df[:, 1:dec.dout]), view16], 1)
    for l in range(len(cW)):
        xs_c.append(h)
        h = _lin32(h, cW[l], cb[l], rng)
        if l < len(cW) - 1:
            h = q(np.maximum(h, 0))
    c3 = h.astype(np.float32)
    s = (np.float32(1) / (np.float32(1) + np.exp(-c3))).astype(np.float32)
    g = go.astype(np.float32)
    dy = q((((g[:, :3] * s).astype(np.float32) * (np.float32(1) - s)).astype(np.float32) * np.float32(scale)).astype(np.float64))
    grads = {"c": [None] * len(cW), "d": [None] * len(dW)}
    for kind, Ws, bs, xs in (("c", cW, cb, xs_c), ("d", dW, db, xs_d)):
        for l in range(len(Ws) - 1, -1, -1):
            x = xs[l]
            gw = _fp32_sum((dy.T[:, None, :] * x.T[None, :, :]), rng) / scale
            gb = _fp32_sum(dy.T, rng) / scale if bs[l] is not None else None
            grads[kind][l] = (gw, gb)
            dx = _fp32_sum(dy[:, None, :] * Ws[l].T[None, :, :], rng)
            if kind == "c" and l == 0:
                g0 = np.where(df[:, 0] > 0, go[:, 3].astype(np.float64) * scale, 0.0)
                dy = q(np.concatenate([g0[:, None], dx[:, :dec.dout - 1]], 1))
            elif kind == "d" and l == 0:
                dfeat = q(dx[:, :planes * width]).reshape(-1, planes, width).transpose(1, 0, 2)
            else:
                dy = np.where(x > 0, q(dx), 0.0)

    def pack(gs):
        parts = []
        for gw, gb in gs:
            parts.append(gw.reshape(-1))
            if gb is not None:
                parts.append(gb)
        return np.concatenate(parts)
    sh = np.concatenate([s.astype(np.float64), np.maximum(df[:, :1], 0)], 1)
    return sh, pack(grads["d"]), pack(grads["c"]), dfeat


def _inside(got, c, r):
    return np.abs(got - c) <= r * (1 + 1e-9) + 1e-300


@pytest.mark.parametrize("seed,dens_dims,col_hidden,view_mode", [(2, [32, 64, 16], [64, 64], 3), (3, [20, 40, 9], [24], 1), (4, [8, 2], [16, 16], 0)])
def test_other_valid_kernels_are_inside(seed, dens_dims, col_hidden, view_mode):
    dec, X0, dirs, go, vm, vf = make_case(seed, dens_dims, col_hidden, view_mode=view_mode, S=64)
    view = T.view_embedding(dirs, vm, vf)
    ref = T.Reference(dec, X0, view)
    planes, width = dens_dims[0] // 4, 4
    scale = 2.0 ** 12
    bw = ref.backward(go, scale, planes, width)
    c, r = ref.shaded()
    rng = np.random.default_rng(seed)
    for _ in range(3):
        sh, gd, gc, dfeat = emulate(dec, X0, view[0], go, scale, planes, width, rng)
        assert _inside(sh, c, r).all()
        for got, (cc, rr) in ((gd, bw["dens"]), (gc, bw["col"]), (dfeat, bw["dfeat"])):
            assert _inside(got, cc, rr).all(), np.max((np.abs(got - cc) - rr) / np.maximum(rr, 1e-30))


def test_intervals_are_tight():
    """Median radius at least 10x below TOL[1] on the same quantity (rgb: absolute; gradients: relative to the largest entry)."""
    dec, X0, dirs, go, vm, vf = make_case(5, [32, 64, 16], [64, 64], S=4096)
    ref = T.Reference(dec, X0, T.view_embedding(dirs, vm, vf))
    c, r = ref.shaded()
    assert np.median(r[:, :3]) <= TOL1_RGB / 10
    bw = ref.backward(go, 2.0 ** 14, 8, 4, wgrad_n=T.wgrad_height(4096, ctas=132))
    for k in ("dens", "col"):
        cc, rr = bw[k]
        assert np.median(rr) <= TOL1_GRAD / 10 * np.abs(cc).max(), k
    print("median radius rgb", np.median(r[:, :3]), "dens", np.median(bw["dens"][1]) / np.abs(bw["dens"][0]).max(),
          "col", np.median(bw["col"][1]) / np.abs(bw["col"][0]).max())


def test_gamma_and_heights():
    assert T.gamma(1) == pytest.approx(2.0 ** -23)
    assert T.wgrad_height(64, ctas=132) == 64 + 1 + 2 + 1
    assert T.wgrad_height(200_000, ctas=132) < T.wgrad_height(200_000)
