"""float64 interval reference of NeuralSDF(OctreeGrid).sdf, SDFTrainer's L2 loss and their gradients (TEST INFRASTRUCTURE,
NOT PRODUCT CODE).

For a field (SPC, trinkets, feature levels, decoder of any depth, position embedding, 'sum' / 'cat', half_features) it returns, for
every output, a centre and a radius: a kernel that rounds where wb_sdf.cuh / wb_sdf_train.cu / wb_octree_grid.cu round and sums
in fp32 in any order lands in centre +- radius.

Rounding points
  features   cell lookup by oracle.oracle.query (bit-exact with wb_query); trilinear coefficients as the kernels compute them
             (coeffs: coords_to_trilinear_coeffs' formula, z fastest, in the kernels' fp32 operation order, bit-exact).  Every kernel blends a LOD by the same fp32 fma chain
             over the corners j = 0..7 and adds the LODs of a 'sum' grid in LOD order, so the features are emulated bit-exactly
             (fma32): half_features rounds every feature value to fp16 on load and each LOD's blend to fp16, radius 0.
  embedding  [x?, sin(x 2^f), cos(x 2^f)] frequency-major, coordinate-minor; x 2^f is exact, sinf / cosf are within 2 ulp (CUDA
             Programming Guide, mathematical functions, without fast math).
  decoder    every kernel runs the same fp32 fma chains: per unit seeded with the bias over the inputs in order, the output over
             the units in order.  They are emulated bit-exactly on the centres (fma_step); inputs with a radius (sinf / cosf) carry it
             through the monotone rounding: fl(v) of a value within r of v lies in [fl(v - r), fl(v + r)].  Samples whose hidden
             pre-activation lies within its radius of 0 are flagged (`amb`): callers drop them.
  loss       d = fl(y - gt), lsum = fmaf(d, d, lsum), dy = fl(fl(1/N) * 2 d); wb_warp_sum's butterfly, the four warp partials in
             order, the product with fl(1/N), one atomic per CTA.
  gradients  pass 2 per hidden unit: da = fl(dy * wout_j) for active units, dL/db += da, dL/dwout = fmaf(dy, relu(a), .),
             dL/dW0 = fmaf(da, x, .) over the CTA's samples in order; dL/dfeat = fl(fl(dy * G) * cf) per sample and corner, added
             atomically, G = sum_j wout_j W0[j, :] over active units.  The fp16 rounding of the forward is passed straight through.
             When every CTA owns one 128-sample tile (N <= 128 * SMs) the partition is known and every chain above is emulated in
             order (_tile_partials); only the atomics of the per-CTA partials and the grid scatter remain in unknown order.

Accumulation error.  SIMT fp32 fma / add / mul and atomicAdd round to nearest, so each addition has relative error <= u = 2^-24.
A sum in unknown order whose terms each pass through at most n roundings is bounded by gamma(n) * sum|terms| (Higham, Accuracy
and Stability of Numerical Algorithms, 2nd ed., section 4.2), with n the height of the real summation tree (TrainHeights); batches of
more tiles than SMs use these bounds throughout (their CTA partition depends on the occupancy).
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import List, Optional, Sequence

import numpy as np

from . import oracle as O
from . import octree_grid as OG
from .tc_decoders import f16, gamma

U = 2.0 ** -24                       # round-to-nearest fp32 (SIMT fma / add / mul / atomicAdd)
SIN_ULPS = 2.0                       # sinf / cosf maximum ulp error
TILE = 128                           # WB_SDF_TRAIN_TILE
MAX_CTAS_PER_SM = 2048 // TILE       # thread limit of an SM: an upper bound of the training kernels' occupancy


def g32(n):
    return gamma(n, U)


def r32(x):
    """Round to fp32 (nearest-even).  For a sum, product or quotient of two fp32 values computed in float64 this is the correctly
    rounded fp32 result (53 >= 2 * 24 + 2)."""
    return np.asarray(x, np.float64).astype(np.float32).astype(np.float64)


def fma32(a, b, c):
    """fmaf(a, b, c) of fp32 values held in float64: a * b is exact; s = fl64(a * b + c) rounds to the same fp32 as the exact sum
    unless s lies exactly halfway between two fp32 values (its 29 low mantissa bits are 1 followed by zeros), where the TwoSum
    error e of s decides."""
    a, b, c = np.broadcast_arrays(np.asarray(a, np.float64), np.asarray(b, np.float64), np.asarray(c, np.float64))
    p = a * b
    s = np.ascontiguousarray(p + c)
    r = s.astype(np.float32).astype(np.float64)
    bits = s.view(np.int64) & 0x1FFFFFFF
    tie = (bits == 0x10000000) | ((np.abs(s) < 2.0 ** -125) & (s != 0))     # fp32 subnormal range: decide every case exactly
    if tie.any():
        pt, ct, st = p[tie], c[tie], s[tie]
        z = st - pt
        e = (pt - (st - z)) + (ct - z)
        r32_ = st.astype(np.float32)
        rt = r32_.astype(np.float64)
        nb = np.nextafter(r32_, np.where(st > rt, np.float32(np.inf), np.float32(-np.inf))).astype(np.float64)
        mid = (st != rt) & ((st - rt) == (nb - st))
        r[tie] = np.where(mid & (e != 0) & (np.sign(e) == np.sign(nb - st)), nb, rt)
    return r


def round_radius(c, v, r):
    """Radius of an fp32 result c = fl(v) (v: the exact value on the operands' centres, in float64) when the operands' true values
    move the exact value by at most r: fl is monotone, so the kernel's result lies in [fl(v - r), fl(v + r)]."""
    r2 = r * (1 + 2.0 ** -50) + 2.0 ** -52 * np.abs(v)                    # float64 rounding of v
    return np.where(r > 0, np.maximum(r32(v + r2) - c, c - r32(v - r2)), 0.0)


def fma_step(sc, sr, ac, ar, bc, br):
    """One kernel step s = fmaf(a, b, s) on intervals: the centre is the fp32 step on the centres (bit-exact), the radius bounds the
    same step on any operands within the radii (round_radius); a product that is exactly zero on both sides adds nothing."""
    s = fma32(ac, bc, sc)
    e = sr + np.abs(ac) * br + ar * np.abs(bc) + ar * br
    zero = ((np.asarray(ac) == 0) & (np.asarray(ar) == 0)) | ((np.asarray(bc) == 0) & (np.asarray(br) == 0))
    return s, np.where(zero, sr, round_radius(s, np.asarray(ac) * bc + sc, e))


@dataclass
class Field:
    """NeuralSDF(OctreeGrid): feature levels for LODs base_lod .. base_lod + num_lods - 1; decoder in nn.Linear layout."""
    spc: O.SPC
    trinkets: np.ndarray
    feats: List[np.ndarray]
    base_lod: int
    multiscale: str
    Ws: List[np.ndarray]
    bs: List[np.ndarray]
    pos_mode: int = 1
    pos_freq: int = 0
    half: bool = True

    @property
    def num_lods(self):
        return len(self.feats)

    @property
    def F(self):
        return self.feats[0].shape[1]

    @property
    def pos_dim(self):
        m, f = self.pos_mode, self.pos_freq
        return 0 if m == 0 else 3 if m == 1 else 6 * f if m == 2 else 3 + 6 * f

    def packed(self) -> np.ndarray:
        """[W0, b0, W1, b1, ..., Wout, bout] (the order of the fused training step's decoder buffer)."""
        return np.concatenate([a.reshape(-1) for W, b in zip(self.Ws, self.bs) for a in (W, b)]).astype(np.float32)


def field_from_case(case, half=True) -> Field:
    """oracle.octree_grid.make_sdf_case -> Field (identity position input, as the case's decoder expects)."""
    return Field(case["spc"], case["trinkets"], case["feats"], case["active_lods"][0], case["multiscale"], list(case["W"]), list(case["b"]),
                 1, 0, half)


def random_decoder(rng, in_dim, pos_mode, hidden, layers, scale=0.05):
    """Decoder whose output is ~ (|x|+|y|+|z|)/sqrt(3) - 0.3 when the raw position is an input (so that rays hit a surface), plus a
    small random perturbation; every unit also sees the whole input."""
    dims = [in_dim] + [hidden] * layers + [1]
    Ws = [(rng.uniform(-1, 1, (o, i)) / np.sqrt(i) * scale).astype(np.float32) for i, o in zip(dims[:-1], dims[1:])]
    bs = [(rng.uniform(-1, 1, o) * scale).astype(np.float32) for o in dims[1:]]
    if pos_mode in (1, 3) and hidden >= 6:
        Ws[0][:6, :3] = np.array([[1, 0, 0], [-1, 0, 0], [0, 1, 0], [0, -1, 0], [0, 0, 1], [0, 0, -1.0]], np.float32)
        bs[0][:6] = 0.0
        for W, b in zip(Ws[1:-1], bs[1:-1]):
            W[:6, :] = 0.0; W[:6, :6] = np.eye(6, dtype=np.float32); b[:6] = 0.0
        Ws[-1][0, :6] = 1.0 / np.sqrt(3.0)
        bs[-1][0] = -0.3
    return Ws, bs


@dataclass
class TrainHeights:
    """Heights of the summation trees of wb_sdf_train for N samples on a GPU with `sms` SMs: between min(tiles, sms) and
    min(tiles, MAX_CTAS_PER_SM * sms) CTAs (one launch per loss LOD), each over a grid-stride run of 128-sample tiles."""
    chain: int          # samples one thread's decoder-gradient chain covers (tiles per CTA * TILE)
    tiles: int          # tiles per CTA (the loss / dL/dbout per-thread chain)
    ctas: int           # atomics per launch into one address

    @staticmethod
    def of(N: int, sms: int = 132) -> "TrainHeights":
        ntiles = max(1, -(-N // TILE))
        cmin, cmax = min(ntiles, sms), min(ntiles, MAX_CTAS_PER_SM * sms)
        t = -(-ntiles // cmin)
        return TrainHeights(t * TILE, t, cmax)


def _embed(field: Field, x: np.ndarray, exact: bool):
    m, fq = field.pos_mode, field.pos_freq
    N = x.shape[0]
    if m == 0:
        return np.zeros((N, 0)), np.zeros((N, 0))
    if m == 1:
        return x.copy(), np.zeros_like(x)
    parts_c, parts_r = ([x], [np.zeros_like(x)]) if m == 3 else ([], [])
    wind = np.concatenate([x * 2.0 ** f for f in range(fq)], -1)           # frequency-major, coordinate-minor
    for fn in (np.sin, np.cos):
        v = fn(wind)
        if exact:
            parts_c.append(v); parts_r.append(np.zeros_like(v))
        else:                                       # centre: sin rounded to fp32; sinf is within 2 ulp of sin, so 2.5 ulp of it
            c = r32(v)
            parts_c.append(c)
            parts_r.append((SIN_ULPS + 0.5) * np.spacing(np.abs(c).astype(np.float32)).astype(np.float64) * (1 + 2.0 ** -20))
    return np.concatenate(parts_c, -1), np.concatenate(parts_r, -1)


@dataclass
class Cells:
    """Per LOD k: rows that reach level base_lod + k (ok), their corner rows tk [n,8] and fp32 coefficients cf [n,8]."""
    ok: List[np.ndarray]
    tk: List[np.ndarray]
    cf: List[np.ndarray]


def cells(field: Field, coords: np.ndarray, nl: int) -> Cells:
    L = field.base_lod + nl - 1
    pidx = O.query(field.spc, coords, L, with_parents=True)[:, field.base_lod:]
    oks, tks, cfs = [], [], []
    for k in range(nl):
        ok = pidx[:, k] >= 0
        p = pidx[ok, k].astype(np.int64)
        oks.append(ok)
        tks.append(field.trinkets[p].astype(np.int64))
        cfs.append(coeffs(coords[ok], field.spc.points[p], field.base_lod + k))
    return Cells(oks, tks, cfs)


def coeffs(coords: np.ndarray, points: np.ndarray, level: int) -> np.ndarray:
    """The kernels' trilinear coefficients, bit-exact: u = fmaf(c, 2^(l-1), 2^(l-1)) - point (the subtraction is exact), then
    [(1-ux)(1-uy)(1-uz), (1-ux)(1-uy)uz, ...] z fastest in fp32.  coords_to_trilinear_coeffs' u = 2^l (c*0.5+0.5) - point rounded
    once differs from this by up to one ulp of 2^l."""
    hl = 2.0 ** (level - 1)
    u = fma32(coords.astype(np.float64), hl, hl) - points.astype(np.float64)
    iu = r32(1.0 - u)
    out = np.zeros((coords.shape[0], 8))
    for j in range(8):
        cx = u[:, 0] if (j & 4) else iu[:, 0]; cy = u[:, 1] if (j & 2) else iu[:, 1]; cz = u[:, 2] if (j & 1) else iu[:, 2]
        out[:, j] = r32(r32(cx * cy) * cz)
    return out


def features(field: Field, coords: np.ndarray, nl: int, exact: bool = False, cl: Optional[Cells] = None):
    """OctreeGrid.interpolate for LODs 0..nl-1 -> (centre, radius, ambiguous[N], cells)."""
    N, F = coords.shape[0], field.F
    cl = cl or cells(field, coords, nl)
    rnd = field.half and not exact
    amb = np.zeros(N, bool)
    blends_c, blends_r = [], []
    for k in range(nl):
        ok, tk, cf = cl.ok[k], cl.tk[k], cl.cf[k]
        ft = field.feats[k].astype(np.float64)
        if rnd:
            ft = f16(ft)
        bc, br = np.zeros((N, F)), np.zeros((N, F))
        if ok.any():
            v = ft[tk]                                                       # [n, 8, F]
            if exact:
                c = (v * cf[:, :, None]).sum(1)
            else:                                                            # every kernel: acc = fmaf(v_j, cf_j, acc), j = 0..7
                c = np.zeros(v.shape[::2])
                for j in range(8):
                    c = fma32(v[:, j], cf[:, j:j + 1], c)
                if rnd:
                    c = f16(c)
            bc[ok] = c
        blends_c.append(bc); blends_r.append(br)
    if field.multiscale == "sum" and nl > 1:
        c = blends_c[0]
        for b in blends_c[1:]:                                               # feat += blend, LOD by LOD
            c = c + b if exact else r32(c + b)
        return c, np.zeros_like(c), amb, cl
    return np.concatenate(blends_c, -1), np.concatenate(blends_r, -1), amb, cl


def _chain(xc, xr, W, b):
    """x W^T + b as every kernel computes it: an fp32 fma chain per unit, seeded with the bias, over the inputs in order."""
    W = W.astype(np.float64)
    s = np.broadcast_to(b.astype(np.float64), (xc.shape[0], W.shape[0])).copy()
    d = np.zeros_like(s)
    for k in range(W.shape[1]):
        s, d = fma_step(s, d, W[None, :, k], 0.0, xc[:, k:k + 1], xr[:, k:k + 1])
    return s, d


def _linear(xc, xr, W, b, exact, in_order=True):
    """x W^T + b by fp32 fma chains seeded with the bias (exact: float64; in_order: the kernels' order, emulated, else any order)."""
    if not exact and in_order:
        return _chain(xc, xr, W, b)
    W = W.astype(np.float64); b = b.astype(np.float64)
    c = xc @ W.T + b
    r = xr @ np.abs(W).T
    if not exact:
        r = r + g32(W.shape[1] + 1) * ((np.abs(xc) + xr) @ np.abs(W).T + np.abs(b))
    return c, r


def _mul(ac, ar, bc, br, rnd):
    c = ac * bc
    r = np.abs(ac) * br + ar * np.abs(bc) + ar * br
    return c, (r + U * (np.abs(c) + r) if rnd else r)


@dataclass
class Forward:
    y: np.ndarray; y_r: np.ndarray; amb: np.ndarray
    x: np.ndarray; x_r: np.ndarray                      # decoder input [position embedding | features]
    hs: list; hs_r: list; act: list                     # hidden activations (interval) and relu masks per layer
    pre: list; pre_r: list                              # hidden pre-activations
    cells: Cells


def forward(field: Field, coords: np.ndarray, lod_idx: Optional[int] = None, exact: bool = False, in_order: bool = True) -> Forward:
    """NeuralSDF.sdf(coords, lod_idx) -> Forward (y [N]: centre, y_r: radius, amb: ambiguous samples)."""
    coords = np.asarray(coords, np.float32)
    nl = (field.num_lods - 1 if lod_idx is None else lod_idx) + 1
    pc, pr = _embed(field, coords.astype(np.float64), exact)
    fc, fr, amb, cl = features(field, coords, nl, exact)
    xc, xr = np.concatenate([pc, fc], -1), np.concatenate([pr, fr], -1)
    hc, hr = xc, xr
    hs, hs_r, acts, pre, pre_r = [], [], [], [], []
    for W, b in zip(field.Ws[:-1], field.bs[:-1]):
        ac, ar = _linear(hc, hr, W, b, exact, in_order)
        amb |= ((np.abs(ac) <= ar) & (ar > 0)).any(1)                       # an exact pre-activation decides its mask exactly
        act = ac > 0
        hc, hr = np.where(act, ac, 0.0), np.where(act, ar, 0.0)
        hs.append(hc); hs_r.append(hr); acts.append(act); pre.append(ac); pre_r.append(ar)
    yc, yr = _linear(hc, hr, field.Ws[-1], field.bs[-1], exact, in_order)
    return Forward(yc[:, 0], yr[:, 0], amb, xc, xr, hs, hs_r, acts, pre, pre_r, cl)


def _scatter(field: Field, gx_c, gx_r, cl: Cells, nl: int, sum_: bool, rnd: bool):
    """sum over samples and corners of fl(gx * cf) into each feature level, one atomic per sample and corner
    -> [(centre, radius before accumulation error, sum|terms|, contributions per row)] per LOD."""
    F = field.F
    out = []
    for k in range(nl):
        rows = field.feats[k].shape[0]
        ok, tk, cf = cl.ok[k], cl.tk[k], cl.cf[k]
        cols = slice(0, F) if sum_ else slice(k * F, (k + 1) * F)
        gc, gr = gx_c[ok][:, cols], gx_r[ok][:, cols]
        C, R, A = np.zeros((rows, F)), np.zeros((rows, F)), np.zeros((rows, F))
        n = np.zeros(rows)
        for j in range(8):
            tc, tr = _mul(gc, gr, cf[:, j:j + 1], 0.0, rnd)
            idx = tk[:, j]
            n += np.bincount(idx, minlength=rows)
            for f in range(F):
                C[:, f] += np.bincount(idx, tc[:, f], rows)
                R[:, f] += np.bincount(idx, tr[:, f], rows)
                A[:, f] += np.bincount(idx, np.abs(tc[:, f]) + tr[:, f], rows)
        out.append((C, R, A, n))
    return out


def interp_backward(field: Field, coords: np.ndarray, go: np.ndarray, lod_idx: int, exact: bool = False):
    """OctreeGrid.interpolate backward (wb_octree_interp_bwd): d sum(go * feats) / d feature level k -> [(centre, radius)]."""
    coords = np.asarray(coords, np.float32)
    nl = lod_idx + 1
    cl = cells(field, coords, nl)
    go = np.asarray(go, np.float64)
    sc = _scatter(field, go, np.zeros_like(go), cl, nl, field.multiscale == "sum" and nl > 1, not exact)
    return [(C, R if exact else R + g32(n)[:, None] * A) for C, R, A, n in sc]


def _tile_partials(field: Field, fw: Forward, gt: np.ndarray, inv: float, C: int):
    """wb_sdf_train with one 128-sample tile per CTA (C CTAs): the per-CTA partials of the loss and of the packed decoder gradient,
    each computed in the kernel's order (fp32 chains per thread over the tile, the warp butterfly, the four warp partials, the
    product with fl(1/N)) -> (loss [C], loss_r, dec [C, P], dec_r).  Only the atomics of the partials are left in unknown order."""
    N = gt.shape[0]
    pad = lambda a: np.concatenate([a, np.zeros((C * TILE - N,) + a.shape[1:])]).reshape((C, TILE) + a.shape[1:])
    dc = r32(fw.y - gt); dr = round_radius(dc, fw.y - gt, fw.y_r)                   # d = out - gt
    dyc = r32(inv * (2.0 * dc)); dyr = round_radius(dyc, inv * 2.0 * dc, inv * 2.0 * dr)   # dy = inv_count * (2 d)
    # loss and dL/dbout: per thread one sample, wb_warp_sum's butterfly, then warp partials added in order from 0
    def cta_sum(vc, vr):
        vc, vr = vc.reshape(C, TILE // 32, 32), vr.reshape(C, TILE // 32, 32)
        for o in (16, 8, 4, 2, 1):
            perm = np.arange(32) ^ o
            vc, vr = fma_step(vc, vr, 1.0, 0.0, vc[..., perm], vr[..., perm])
        lc, lr = np.zeros(C), np.zeros(C)
        for w in range(TILE // 32):
            lc, lr = fma_step(lc, lr, 1.0, 0.0, vc[:, w, 0], vr[:, w, 0])
        return lc, lr
    sq = fma_step(0.0, 0.0, dc, dr, dc, dr)                                          # lsum = fmaf(d, d, 0)
    lc, lr = cta_sum(pad(sq[0]), pad(sq[1]))
    loss_c = r32(lc * inv); loss_r = round_radius(loss_c, lc * inv, lr * inv)
    bo_c, bo_r = cta_sum(pad(dyc), pad(dyr))
    # pass 2, thread per hidden unit j, samples of the tile in order
    W0, wo = field.Ws[0].astype(np.float64), field.Ws[1][0].astype(np.float64)
    H, IN = W0.shape
    xc, xr = pad(fw.x), pad(fw.x_r)
    hc, hr, act = pad(fw.hs[0]), pad(fw.hs_r[0]), pad(fw.act[0].astype(np.float64)) > 0
    dsc, dsr = pad(dyc), pad(dyr)
    gw = (np.zeros((C, H, IN)), np.zeros((C, H, IN)))
    gb, gwo = (np.zeros((C, H)), np.zeros((C, H))), (np.zeros((C, H)), np.zeros((C, H)))
    for t in range(TILE):
        ds, dsr_ = dsc[:, t, None], dsr[:, t, None]
        dac = np.where(act[:, t], r32(ds * wo), 0.0)                                 # da = a > 0 ? ds * wout_j : 0
        dar = np.where(act[:, t], round_radius(dac, ds * wo, dsr_ * np.abs(wo)), 0.0)
        gb = fma_step(*gb, 1.0, 0.0, dac, dar)
        gwo = fma_step(*gwo, ds, dsr_, hc[:, t], hr[:, t])
        gw = fma_step(*gw, dac[:, :, None], dar[:, :, None], xc[:, t, None, :], xr[:, t, None, :])
    dec_c = np.concatenate([gw[0].reshape(C, -1), gb[0], gwo[0], bo_c[:, None]], 1)
    dec_r = np.concatenate([gw[1].reshape(C, -1), gb[1], gwo[1], bo_r[:, None]], 1)
    return loss_c, loss_r, dec_c, dec_r


@dataclass
class Train:
    loss: float; loss_r: float
    dec: np.ndarray; dec_r: np.ndarray                  # packed like Field.packed()
    grid: list                                          # [(centre, radius)] per feature level
    amb: np.ndarray
    grid_n: list                                        # contributions (atomics) per feature row and level
    atomics: int                                        # atomics per decoder / loss address (CTAs of all launches, upper bound)


def train(field: Field, coords: np.ndarray, gt: np.ndarray, lods: Sequence[int], exact: bool = False, sms: int = 132) -> Train:
    """Loss sum_lod sum_i (y_i - gt_i)^2 / N and its gradients (SDFTrainer.step before the optimiser)."""
    coords = np.asarray(coords, np.float32)
    gt = np.asarray(gt, np.float64).reshape(-1)
    N = coords.shape[0]
    h = TrainHeights.of(N, sms)
    nlaunch = len(lods)
    loss_h = h.tiles + 5 + 4 + 2 + nlaunch * h.ctas                        # thread chain, warp tree, warp partials, fl(1/N) and product, atomics
    dec_h = h.chain + 5 + 4 + nlaunch * h.ctas
    rnd = not exact
    nparams = field.packed().size
    loss_c = loss_r = 0.0
    dec_c, dec_r, dec_a = np.zeros(nparams), np.zeros(nparams), np.zeros(nparams)
    grid = [(np.zeros(f.shape), np.zeros(f.shape)) for f in field.feats]
    grid_a = [np.zeros(f.shape) for f in field.feats]
    grid_n = [np.zeros(f.shape[0]) for f in field.feats]
    amb = np.zeros(N, bool)
    ntiles = -(-N // TILE)
    tiles = rnd and len(field.Ws) == 2 and ntiles <= sms       # every CTA owns exactly one tile: the partition is known
    inv = float(np.float32(1.0 / N)) if N else 0.0
    parts = []
    for lod in lods:
        fw = forward(field, coords, lod, exact, in_order=ntiles <= sms)    # batches of many tiles: any-order bounds (cost)
        amb |= fw.amb
        if tiles:
            parts.append(_tile_partials(field, fw, gt, inv, ntiles))
        dc = fw.y - gt
        dr = fw.y_r + (U * (np.abs(dc) + fw.y_r) if rnd else 0.0)
        sq_c, sq_r = dc * dc, 2 * np.abs(dc) * dr + dr * dr
        loss_c += sq_c.sum() / N
        loss_r += sq_r.sum() / N + (g32(loss_h) * (sq_c + sq_r).sum() / N if rnd else 0.0)
        dyc, dyr = _mul(dc, dr, 2.0 / N, 0.0, False)
        if rnd:
            dyr = dyr + (2 * U + U * U) * (np.abs(dyc) + dyr)               # fl(fl(1/N) * 2d)
        # decoder: walk back through the layers; G = d y / d (layer input) without the dy factor, masks from the forward
        layers = list(zip(field.Ws, field.bs))
        ins = [(fw.x, fw.x_r)] + list(zip(fw.hs, fw.hs_r))
        offs, o = [], 0
        for W, b in layers:
            offs.append(o); o += W.size + b.size
        Gc = np.ones((N, 1)); Gr = np.zeros((N, 1))
        for li in range(len(layers) - 1, -1, -1):
            W, b = layers[li]
            xc, xr = ins[li]
            if li == len(layers) - 1:
                dac, dar = dyc[:, None] * Gc, dyr[:, None] * Gc             # dL/dy = dy (no rounding: fma(dy, relu(a), gwo))
            else:
                dac, dar = _mul(dyc[:, None], dyr[:, None], Gc, Gr, rnd)    # da = fl(dy * wout_j)
            gw_c = dac.T @ xc
            gw_r = np.abs(dac).T @ xr + dar.T @ np.abs(xc) + dar.T @ xr
            gw_a = (np.abs(dac) + dar).T @ (np.abs(xc) + xr)
            gb_c, gb_r, gb_a = dac.sum(0), dar.sum(0), (np.abs(dac) + dar).sum(0)
            s = offs[li]
            dec_c[s:s + W.size] += gw_c.reshape(-1); dec_r[s:s + W.size] += gw_r.reshape(-1); dec_a[s:s + W.size] += gw_a.reshape(-1)
            s += W.size
            dec_c[s:s + b.size] += gb_c; dec_r[s:s + b.size] += gb_r; dec_a[s:s + b.size] += gb_a
            # G of this layer's input: sum over units (fp32 fma chain), masked by the previous relu
            Wd = W.astype(np.float64)
            nGc = Gc @ Wd
            nGr = Gr @ np.abs(Wd) + (g32(W.shape[0]) * (np.abs(Gc) + Gr) @ np.abs(Wd) if rnd else 0.0)
            if li > 0:
                act = fw.act[li - 1]
                nGc, nGr = np.where(act, nGc, 0.0), np.where(act, nGr, 0.0)
            Gc, Gr = nGc, nGr
        # grid: dL/dfeat = fl(dy * G) over the feature columns of the decoder input
        pd = field.pos_dim
        gxc, gxr = _mul(dyc[:, None], dyr[:, None], Gc[:, pd:], Gr[:, pd:], rnd)
        nl = lod + 1
        sc = _scatter(field, gxc, gxr, fw.cells, nl, field.multiscale == "sum" and nl > 1, rnd)
        for k, (C, R, A, n) in enumerate(sc):
            grid[k][0][...] += C; grid[k][1][...] += R; grid_a[k] += A; grid_n[k] += n
    if rnd:
        dec_r = dec_r + g32(dec_h) * dec_a
        grid = [(C, R + g32(n)[:, None] * A) for (C, R), A, n in zip(grid, grid_a, grid_n)]     # one atomic per contribution
    if tiles:                  # the partials of all launches reach the zeroed buffers by atomics in any order: one rounding each after the first
        lc = np.concatenate([p[0] for p in parts]); lr = np.concatenate([p[1] for p in parts])
        loss_c, loss_r = lc.sum(), lr.sum() + g32(lc.size - 1) * (np.abs(lc) + lr).sum()
        pc = np.concatenate([p[2] for p in parts]); pr = np.concatenate([p[3] for p in parts])
        dec_c, dec_r = pc.sum(0), pr.sum(0) + g32(pc.shape[0] - 1) * (np.abs(pc) + pr).sum(0)
    return Train(loss_c, loss_r, dec_c, dec_r, grid, amb, grid_n, nlaunch * h.ctas)
