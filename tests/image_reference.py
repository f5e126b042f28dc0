"""Exact and float64 references of the app/image kernels (TEST INFRASTRUCTURE, NOT PRODUCT CODE): the 2-D hash-grid kernels
(wb_hashgrid2d_fwd / _bwd) and ImageNeuralField evaluated and trained in one launch (wb_image_eval / wb_image_train, csrc/wb_image.cu).

2-D cell (grid_index_reference.py's conventions, one axis fewer)
  cell       per axis gi.cell_axis: x = fmaf(c, res/2, res/2) clamped to [0, fl(res - 1 - 1e-5)] (NaN lands on the bound), p = floor(x),
             w = x - p, 1 - w rounded.  Bit-exact.
  coefs      c00 = (1-wx)(1-wy), c01 = (1-wx)wy, c10 = wx(1-wy), c11 = wx wy, each rounded to fp32; corner j = (x + (j>>1&1), y + (j&1)).
  rows       level-local; dense levels (res < T and res^2 < T) x + y res with the +1 corner kept on the cell's own row on the level's last
             cell (`top_clamp=False`: the reference kernel's unclamped rows); hashed levels (x ^ y*2654435761) & (T - 1).  Exact.
  forward    emulated: fl(v_0 c_0), then fmaf over corners 1..3 -- bit-exact.  Interval: float64 sum, radius gamma(4) sum |v c|.
  backward   every entry is its initial value plus fl(g c_j) per (sample, LOD, corner) not skipped (an all-zero pair / quad / feature
             is skipped), added by fp32 atomics in any order: centre = the float64 sum, radius = gamma(k) (|initial| + sum |terms|).

ImageNeuralField (float64 centres with a-priori radii; `rounding=False` drops every rounding term, leaving the float64 chain that torch
float64 autograd computes)
  x          [features, x, y, sin(c_a 2^f), cos(c_a 2^f)] (frequency-major, coordinate-minor).  'cat' features are the bit-exact fp32
             emulation (exact); 'sum' adds L of them in fp32: radius gamma(L) sum |f_l|.  sin / cos: CUDA's sinf / cosf are within
             2 ulp; the radius is 2^-21 |v| (4 ulp).
  a, h       a_j = b_j + sum_k W_jk x_k: radius gamma(IN + 1)(|b| + sum |W||x|) + sum |W| r_x; h = relu(a) as an interval (an a whose
             interval straddles 0 makes h and the relu mask uncertain: the backward then takes the hull of both branches).
  z, y       z_c = bo_c + sum_j Wo_cj h_j likewise; y = sigmoid(z): radius r_z / 4 + 4u y (expf, the add and the division).
  loss       sum (y - gt)^2 * inv over 3N values, inv = fl32(1 / (3N)): radius from r_y, plus gamma(3N + 64) of the sum.
  dy         inv * 2 (y - gt) * y (1 - y): radius 8u |dy| + inv * 2 (|y(1-y)| + |y - gt|) r_y + second order.
  da, g      da_j = [a_j > 0] sum_c dy_c Wo_cj; g_k = sum_j da_j W0_jk (feature columns): gamma(count) sums plus propagated radii.
  grads      dW0 = sum_s da x, db0 = sum_s da, dWo = sum_s dy h, dbo = sum_s dy: summed over the samples of a CTA in order and over CTAs
             by atomics, radius gamma(N + 256) sum |terms| plus propagated radii; the table gradient as the backward above with the
             radius of g carried through |c|."""
from __future__ import annotations

import numpy as np

import grid_index_reference as GI
import octree_reference as OR

f32, f64 = np.float32, np.float64
P1 = 2654435761
U = 2.0 ** -24
gamma = GI.gamma
BANDS = (1.0, 2.0, 4.0)


# ---- 2-D hash grid ------------------------------------------------------------------------------------------------------------
def is_dense(res: int, bitwidth: int) -> bool:
    T = 2 ** bitwidth
    return res < T and res * res < T


def level_rows(res: int, bitwidth: int, coord_dim: int) -> int:
    """Rows of one level of MultiTable(coord_dim): min(res^coord_dim, 2^bitwidth)."""
    return min(res ** coord_dim, 2 ** bitwidth)


def table_layout(resolutions, bitwidth, coord_dim):
    begin = np.zeros(len(resolutions) + 1, np.int64)
    begin[1:] = np.cumsum([level_rows(int(r), bitwidth, coord_dim) for r in resolutions])
    return begin


def corners(coords, res: int, bitwidth: int, top_clamp: bool = True):
    """-> (rows int64 [N, 4] level-local, coefs fp32 [N, 4]) of one level."""
    c = np.asarray(coords, f32)
    (px, wx, ix), (py, wy, iy) = (GI.cell_axis(c[:, a], res) for a in range(2))
    cf = np.stack([(ix * iy).astype(f32), (ix * wy).astype(f32), (wx * iy).astype(f32), (wx * wy).astype(f32)], 1)
    T, dense = 2 ** bitwidth, is_dense(res, bitwidth)
    rows = np.zeros((c.shape[0], 4), np.int64)
    for j in range(4):
        x, y = px + ((j >> 1) & 1), py + (j & 1)
        if dense and top_clamp:
            x, y = np.where(px < res - 1, x, px), np.where(py < res - 1, y, py)
        rows[:, j] = x + y * res if dense else (x ^ ((y * P1) & 0xFFFFFFFF)) & (T - 1)
    return rows, cf


def hashgrid2d_fwd(coords, table, resolutions, bitwidth, begin):
    """-> (emulated fp32 [N, L*F], centre float64 [N, L*F], radius float64 [N, L*F])."""
    table = np.asarray(table, f32)
    N = np.asarray(coords).shape[0]
    emu, cen, rad = [], [], []
    for l, res in enumerate(resolutions):
        rows, cf = corners(coords, int(res), bitwidth)
        v = table[begin[l] + rows]                                   # [N, 4, F]
        with np.errstate(invalid="ignore", over="ignore"):
            a = (v[:, 0] * cf[:, :1]).astype(f32)
            for j in range(1, 4):
                a = OR.fma32(v[:, j], np.broadcast_to(cf[:, j:j + 1], a.shape), a)
            terms = v.astype(f64) * cf[:, :, None].astype(f64)
        emu.append(a); cen.append(terms.sum(1)); rad.append(gamma(4) * np.abs(terms).sum(1))
    return (np.concatenate(emu, 1).reshape(N, -1), np.concatenate(cen, 1).reshape(N, -1), np.concatenate(rad, 1).reshape(N, -1))


def _scatter(cen, mag, k, rg_acc, rows_abs, cf, g, rg, F):
    """Add fl(g_f c_j) of every sample into one level's rows (g [n, F] fp32, rg [n, F] radius of g)."""
    live = np.repeat((g != 0).any(1, keepdims=True), F, 1) if F == 2 else \
        np.repeat((g.reshape(len(g), -1, 4) != 0).any(2), 4, 1) if F % 4 == 0 else (g != 0)
    n_rows = cen.shape[0]
    for f in range(F):
        m = live[:, f]
        if not m.any():
            continue
        t = (g[m, f][:, None].astype(f32) * cf[m]).astype(f32).astype(f64)
        r = rows_abs[m].ravel()
        cen[:, f] += np.bincount(r, weights=t.ravel(), minlength=n_rows)
        mag[:, f] += np.bincount(r, weights=np.abs(t).ravel(), minlength=n_rows)
        k[:, f] += np.bincount(r, minlength=n_rows)
        rg_acc[:, f] += np.bincount(r, weights=(rg[m, f][:, None] * cf[m].astype(f64)).ravel(), minlength=n_rows)


def hashgrid2d_bwd(coords, grad_feats, grad_table0, resolutions, bitwidth, begin):
    """-> (centre float64 [rows, F], radius float64 [rows, F], k int64 [rows, F] atomic adds per entry)."""
    g0 = np.asarray(grad_table0, f32)
    n_rows, F = g0.shape
    L = len(resolutions)
    go = np.asarray(grad_feats, f32).reshape(-1, L, F)
    cen = g0.astype(f64).copy(); mag = np.abs(cen); k = np.zeros((n_rows, F), np.int64); rg = np.zeros((n_rows, F))
    for l, res in enumerate(resolutions):
        rows, cf = corners(coords, int(res), bitwidth)
        _scatter(cen, mag, k, rg, begin[l] + rows, cf, go[:, l], np.zeros_like(go[:, l], f64), F)
    return cen, gamma(k) * mag, k


# ---- ImageNeuralField ---------------------------------------------------------------------------------------------------------
def unpack(params, IN, H):
    p = np.asarray(params, f64)
    o = 0
    out = []
    for shape in ((H, IN), (H,), (3, H), (3,)):
        n = int(np.prod(shape)); out.append(p[o:o + n].reshape(shape)); o += n
    return out


def embed(coords):
    """[N, 14] float64 centre of [x, y, sin(c 2^f), cos(c 2^f)] at fp32 arguments (c * 2^f is exact)."""
    c = np.asarray(coords, f32).astype(f64)
    w = np.concatenate([c * b for b in BANDS], 1)                    # [x1, y1, x2, y2, x4, y4]
    return np.concatenate([c, np.sin(w), np.cos(w)], 1)


def features(coords, table, resolutions, bitwidth, begin, multiscale, lod, rounding=True):
    """Decoder-input features: centre and radius [N, FW]."""
    emu, cen, _ = hashgrid2d_fwd(coords, table, resolutions, bitwidth, begin)
    N, L = emu.shape[0], len(resolutions)
    F = emu.shape[1] // L
    base = emu.astype(f64) if rounding else cen
    if multiscale == "sum":
        per = base.reshape(N, L, F)
        return per.sum(1), (gamma(L) * np.abs(per).sum(1) if rounding else np.zeros((N, F)))
    x = base.copy()
    x[:, lod * F:] = 0.0
    return x, np.zeros_like(x)


def _relu_interval(a, ra):
    lo, hi = np.maximum(a - ra, 0.0), np.maximum(a + ra, 0.0)
    return (lo + hi) / 2, (hi - lo) / 2, (a - ra > 0), (a + ra > 0) & (a - ra <= 0)


def forward(coords, table, params, resolutions, bitwidth, begin, multiscale, lod, H, rounding=True):
    """-> dict of centres / radii of x, a, h, z, y."""
    fx, rfx = features(coords, table, resolutions, bitwidth, begin, multiscale, lod, rounding)
    e = embed(coords)
    re = (2.0 ** -21) * np.abs(e) if rounding else np.zeros_like(e)
    re[:, :2] = 0.0                                                  # x, y are copied
    x, rx = np.concatenate([fx, e], 1), np.concatenate([rfx, re], 1)
    IN = x.shape[1]
    W0, b0, Wo, bo = unpack(params, IN, H)
    a = x @ W0.T + b0
    ra = (gamma(IN + 1) * (np.abs(x) @ np.abs(W0).T + np.abs(b0)) + rx @ np.abs(W0).T) if rounding else np.zeros_like(a)
    h, rh, on, amb = _relu_interval(a, ra) if rounding else (np.maximum(a, 0.0), np.zeros_like(a), a > 0, np.zeros_like(a, bool))
    z = h @ Wo.T + bo
    rz = (gamma(H + 1) * (np.abs(h) @ np.abs(Wo).T + np.abs(bo)) + rh @ np.abs(Wo).T) if rounding else np.zeros_like(z)
    y = 1.0 / (1.0 + np.exp(-z))
    ry = (rz / 4 + 4 * U * y) if rounding else np.zeros_like(y)
    return dict(x=x, rx=rx, a=a, ra=ra, h=h, rh=rh, on=on, amb=amb, z=z, rz=rz, y=y, ry=ry, IN=IN, W0=W0, b0=b0, Wo=Wo, bo=bo)


def train(coords, gt, table, params, resolutions, bitwidth, begin, multiscale, lod, H, grad_table0=None, grad_params0=None, rounding=True):
    """One wb_image_train launch: -> dict(loss, rloss, gtable, rgtable, gparams, rgparams) (centres and radii, float64), accumulated onto
    grad_table0 / grad_params0 (zeros when None)."""
    fw = forward(coords, table, params, resolutions, bitwidth, begin, multiscale, lod, H, rounding)
    N = fw["y"].shape[0]
    inv = float(f32(1.0 / (3.0 * N))) if rounding else 1.0 / (3.0 * N)
    gt = np.asarray(gt, f32).astype(f64)
    y, ry = fw["y"], fw["ry"]
    d = y - gt
    loss = (d * d).sum() * inv
    rloss = ((2 * np.abs(d) * ry + ry * ry).sum() * inv + gamma(3 * N + 64) * (d * d).sum() * inv) if rounding else 0.0
    s = y * (1 - y)
    dy = inv * 2 * d * s
    rdy = (8 * U * np.abs(dy) + inv * 2 * (np.abs(s) + np.abs(d)) * ry + inv * 2 * ry * ry) if rounding else np.zeros_like(dy)
    W0, Wo, IN = fw["W0"], fw["Wo"], fw["IN"]
    t = dy @ Wo                                                      # [N, H]
    rt = (gamma(3) * (np.abs(dy) @ np.abs(Wo)) + rdy @ np.abs(Wo)) if rounding else np.zeros_like(t)
    on, amb = fw["on"], fw["amb"]
    da = np.where(on, t, 0.0)
    rda = np.where(on, rt, 0.0)
    if rounding:                                                     # uncertain relu mask: hull of 0 and t
        lo, hi = np.minimum(t - rt, 0.0), np.maximum(t + rt, 0.0)
        da = np.where(amb, (lo + hi) / 2, da); rda = np.where(amb, (hi - lo) / 2, rda)
    x, rx, h, rh = fw["x"], fw["rx"], fw["h"], fw["rh"]
    L = len(resolutions)
    F = np.asarray(table).shape[1]
    FW = F if multiscale == "sum" else L * F
    g = da @ W0[:, :FW]                                              # [N, FW]
    rg = (gamma(H) * (np.abs(da) @ np.abs(W0[:, :FW])) + rda @ np.abs(W0[:, :FW])) if rounding else np.zeros_like(g)
    # table gradient
    n_rows = np.asarray(table).shape[0]
    g0 = np.zeros((n_rows, F), f32) if grad_table0 is None else np.asarray(grad_table0, f32)
    cen = g0.astype(f64).copy(); mag = np.abs(cen); k = np.zeros((n_rows, F), np.int64); rgt = np.zeros((n_rows, F))
    act = L if multiscale == "sum" else lod
    for l in range(act):
        rows, cf = corners(coords, int(resolutions[l]), bitwidth)
        gl = g if multiscale == "sum" else g[:, l * F:(l + 1) * F]
        rgl = rg if multiscale == "sum" else rg[:, l * F:(l + 1) * F]
        if rounding:
            _scatter(cen, mag, k, rgt, begin[l] + rows, cf, gl.astype(f32), rgl, F)
        else:
            for j in range(4):
                np.add.at(cen, begin[l] + rows[:, j], gl * cf[:, j:j + 1].astype(f64))
    rgtable = (gamma(k + 1) * mag + rgt + 2 * U * np.abs(cen)) if rounding else np.zeros_like(cen)
    # decoder gradients, packed [W0, b0, Wo, bo]
    n = N + 256
    gW0, gb0, gWo, gbo = da.T @ x, da.sum(0), dy.T @ h, dy.sum(0)
    gp = np.concatenate([gW0.ravel(), gb0, gWo.ravel(), gbo])
    if rounding:
        rW0 = gamma(n) * (np.abs(da).T @ np.abs(x)) + rda.T @ np.abs(x) + np.abs(da).T @ rx + rda.T @ rx
        rb0 = gamma(n) * np.abs(da).sum(0) + rda.sum(0)
        rWo = gamma(n) * (np.abs(dy).T @ np.abs(h)) + rdy.T @ np.abs(h) + np.abs(dy).T @ rh + rdy.T @ rh
        rbo = gamma(n) * np.abs(dy).sum(0) + rdy.sum(0)
        rgp = np.concatenate([rW0.ravel(), rb0, rWo.ravel(), rbo])
    else:
        rgp = np.zeros_like(gp)
    if grad_params0 is not None:
        p0 = np.asarray(grad_params0, f32).astype(f64)
        gp = gp + p0
        rgp = rgp + (gamma(n) * np.abs(p0) if rounding else 0.0)
    return dict(loss=loss, rloss=rloss, gtable=cen, rgtable=rgtable, gparams=gp, rgparams=rgp, y=y, ry=ry)
