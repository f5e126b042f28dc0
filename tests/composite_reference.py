"""float64 interval reference of packed compositing (wb_composite_fwd / wb_composite_bwd), the image loss fused into the
compositing backward (wb_composite_bwd_loss) and the Adam step (wb_adam_step) (TEST INFRASTRUCTURE, NOT PRODUCT CODE).

Every function returns, per output, a centre and a radius: a kernel that rounds where wb_composite.cu and wb_optim.cu round lands
in centre +- radius.  It builds on oracle/sdf_reference.py (U, fma32, g32, round_radius) and oracle/tc_decoders.py (gamma).

Rounding points
  prefix      tau = fl(sigma * delta) and the exclusive prefix carry + (incl - tau) are emulated bit-exactly in fp32: incl is the
              5-level __shfl_up Kogge-Stone scan of wb_warp_incl_scan inside each 32-sample chunk (lane = sample index % 32), carry
              adds each full chunk's total (lane 31) in chunk order.  T_{k+1} = expf(-(carry + incl)) takes the same prefix.
  expf        within 2 ulp (CUDA Programming Guide, mathematical functions, no fast math): radius 2^-22 * value + 2 subnormal ulps.
              1 - expf(-tau) carries that error as an ABSOLUTE error 2^-23, so tau below ~2^-20 has a relative radius of 1 or more
              (tau < 2^-25: expf rounds to 1 and the kernel's weight is 0); tau == 0 gives exactly w = 0.
  sums        per lane an fma chain over the ray's chunks, then wb_warp_sum's 5-level butterfly: a term passes through at most
              nchunks + 5 roundings, bounded by gamma(nchunks + 5) * sum|terms| (Higham, Accuracy and Stability of Numerical
              Algorithms, 2nd ed., section 4.2).  The backward's prefix gw_carry + gw_incl: one product, 5 scan levels, the carry chain,
              one add: gamma(nchunks + 7).  suffix = G - prefix keeps both radii, so its cancellation at the opaque tail of a long ray
              shows as a radius of the size of sum|g w|, not of the (near zero) suffix.
  small ops   rgb = bg (1 - A) + C, ga = g_alpha - g_rgb . bg, g_k's five-term sum and gtau = g_k T_{k+1} - suffix may be contracted
              into fmas by nvcc: gamma(#ops) * sum|terms|.  g_shaded = fl(g_rgb * w), fl(gtau * delta).
  loss        d = fl(rgb - target) and dL/drgb = fl(loss'(d) * inv_count) are emulated bit-exactly from the kernel's own rgb; the
              loss value is per-warp partial sums added by atomics in any order: gamma(height) * sum|terms|.
  Adam        one step from the kernel's fp32 state before the step, bc1 and bc2_sqrt as the fp32 values the host passes: interval
              arithmetic with one rounding per operation (the final p - step_size * q as two, which covers an fma contraction), and
              adam_fp32, the bit-exact fp32 emulation with both contractions of that last line.

exact=True turns every rounding and every gamma off: the prefix is then the float64 segmented cumsum and the result is the float64
operation (what the CPU tests compare with torch).
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Optional

import numpy as np

from oracle.sdf_reference import U, fma32, g32, round_radius      # noqa: F401  (round_radius: re-exported for the tests)
from oracle.tc_decoders import gamma                              # noqa: F401

f32 = np.float32
TINY = 2.0 ** -149                  # smallest fp32 subnormal: absolute error of a rounding that underflows
EXP_REL = 3.0 * 2.0 ** -23          # expf: 2 ulp from the correctly rounded value (half an ulp away), in the binade above at worst
LOSS_TYPES = {"l2": 0, "l1": 1, "huber": 2}
COMP_THREADS = 256                  # WB_COMP_THREADS


# ---- cases shared by the CPU and GPU tests ------------------------------------------------------------------------------------
RAY_LENGTHS = (0, 1, 31, 32, 33, 63, 64, 65, 1024, 2048)
REGIMES = ("mixed", "zero", "tiny", "opaque", "huge", "delta0")


def ray_lengths(R: int, rng, per_warp=(1, 2, 3, 4, 5, 32), lengths=RAY_LENGTHS):
    """Samples per ray for R rays: every length of `lengths` once, then blocks of 32 rays (one warp's rays) with k sampled rays
    for k in `per_warp` in turn, the rest empty."""
    n = np.zeros(R, np.int64)
    head = min(R, len(lengths))
    n[:head] = lengths[:head]
    b, i = head, 0
    while b < R:
        k = per_warp[i % len(per_warp)]
        blk = min(32, R - b)
        sel = rng.choice(blk, min(k, blk), replace=False)
        n[b + sel] = rng.choice(np.asarray(lengths[1:]), sel.size, p=None) if k < 32 else rng.integers(1, 40, sel.size)
        b += blk; i += 1
    return n


def make_case(n, regime: str = "mixed", seed: int = 0):
    """shaded [S, 4] (r, g, b, sigma), depth [S], deltas [S] (fp32) and offsets [R + 1] for the ray lengths n."""
    rng = np.random.default_rng(seed)
    n = np.asarray(n, np.int64)
    off = np.concatenate([[0], np.cumsum(n)]).astype(np.int64)
    S = int(off[-1])
    pk = packed(off)
    sh = np.empty((S, 4), f32)
    sh[:, :3] = rng.random((S, 3))
    dl = rng.uniform(2e-3, 2e-2, S)
    tau = np.exp(rng.uniform(np.log(1e-4), np.log(2.0), S))
    if regime == "zero":
        tau = np.zeros(S)
    elif regime == "tiny":                                  # below 2^-25: expf(-tau) rounds to 1
        tau = rng.uniform(0.0, 2.0 ** -26, S)
    elif regime == "opaque":                                # total tau of long rays above 104: T underflows to 0
        tau = rng.uniform(0.2, 0.8, S) + np.where(pk.n[pk.ray] <= 64, 4.0, 0.0)
    elif regime == "huge":                                  # the first sample of every ray tau ~ 1e4
        tau = np.where(pk.pos == 0, 1e4, tau)
    elif regime == "delta0":
        dl = np.where(rng.random(S) < 0.5, 0.0, dl)
    sh[:, 3] = tau / np.where(dl > 0, dl, 1.0)
    depth = (1.0 + pk.pos * 0.01 + rng.uniform(0, 0.01, S)).astype(f32)
    return dict(offsets=off, shaded=sh, depth=depth, deltas=dl.astype(f32), n=n)


# ---- ray layout -----------------------------------------------------------------------------------------------------------
@dataclass
class Packed:
    offsets: np.ndarray             # int64 [R + 1]
    ray: np.ndarray                 # int64 [S] ray of every sample
    pos: np.ndarray                 # int64 [S] index of the sample in its ray
    n: np.ndarray                   # int64 [R] samples per ray
    nchunks: np.ndarray             # int64 [R] 32-sample chunks per ray

    @property
    def R(self):
        return self.n.shape[0]

    @property
    def S(self):
        return int(self.offsets[-1])


def packed(offsets) -> Packed:
    off = np.asarray(offsets, np.int64)
    n = np.diff(off)
    ray = np.repeat(np.arange(n.shape[0], dtype=np.int64), n)
    pos = np.arange(int(off[-1]), dtype=np.int64) - off[:-1][ray]
    return Packed(off, ray, pos, n, -(-n // 32))


def seg_sum(pk: Packed, x):
    """sum of x over each ray [R]."""
    return np.bincount(pk.ray, np.asarray(x, np.float64), pk.R) if pk.S else np.zeros(pk.R)


def seg_cumsum(pk: Packed, x):
    """inclusive prefix of x within each ray (float64)."""
    x = np.asarray(x, np.float64)
    if pk.S == 0:
        return x.copy()
    cs = np.cumsum(x)
    base = np.concatenate([[0.0], cs])[pk.offsets[:-1]]
    return cs - base[pk.ray]


def warp_scan(pk: Packed, x):
    """wb_warp_incl_scan inside each 32-sample chunk, in x's dtype (fp32: bit-exact)."""
    v = np.array(x, copy=True)
    lane = pk.pos % 32
    for o in (1, 2, 4, 8, 16):
        t = np.zeros_like(v)
        t[o:] = v[:-o]
        v = np.where(lane >= o, v + t, v)
    return v


def prefixes(pk: Packed, tau32, exact: bool = False):
    """(exclusive, inclusive) prefix of tau per sample as the kernels form them: fp32 values held in float64 (exact: float64)."""
    if exact:
        incl = seg_cumsum(pk, tau32)
        return incl - np.asarray(tau32, np.float64), incl
    tau = np.asarray(tau32, f32)
    incl = warp_scan(pk, tau)
    carry = np.zeros(pk.S, f32)
    long_ = np.nonzero(pk.nchunks > 1)[0]
    if long_.size:
        mc = int(pk.nchunks[long_].max())
        tot = np.zeros((long_.size, mc), f32)
        for c in range(mc - 1):                             # totals of full chunks: lane 31
            k = pk.offsets[long_] + 32 * c + 31
            ok = k < pk.offsets[long_ + 1]
            tot[ok, c] = incl[k[ok]]
        car = np.zeros((long_.size, mc), f32)
        for c in range(1, mc):                              # carry += shfl(incl, 31), in chunk order
            car[:, c] = car[:, c - 1] + tot[:, c - 1]
        sel = pk.nchunks[pk.ray] > 1
        row = np.searchsorted(long_, pk.ray[sel])
        carry[sel] = car[row, pk.pos[sel] // 32]
    xe = carry + (incl - tau)
    xi = carry + incl
    return xe.astype(np.float64), xi.astype(np.float64)


def _exp_r(x):
    """radius of expf(x) around exp(x)."""
    return EXP_REL * x + 2 * TINY


# ---- forward ----------------------------------------------------------------------------------------------------------------
@dataclass
class Weights:
    tau: np.ndarray                 # fp32 values (float64)
    T: np.ndarray
    rT: np.ndarray
    Tn: np.ndarray
    rTn: np.ndarray
    w: np.ndarray
    rw: np.ndarray


def weights(pk: Packed, sigma, delta, exact: bool = False) -> Weights:
    """Per-sample transmittance T_k, T_{k+1} and weight w_k = T_k (1 - exp(-tau_k)) with radii."""
    tau = (np.asarray(sigma, f32) * np.asarray(delta, f32)).astype(np.float64)
    if exact:
        tau = np.asarray(sigma, np.float64) * np.asarray(delta, np.float64)
    xe, xi = prefixes(pk, tau, exact)
    T, Tn, e = np.exp(-xe), np.exp(-xi), np.exp(-tau)
    a = 1.0 - e
    w = T * a
    if exact:
        z = np.zeros_like(w)
        return Weights(tau, T, z, Tn, z, w, z)
    rT, rTn, re = _exp_r(T), _exp_r(Tn), _exp_r(e)
    ra = re + U * (a + re)
    rw = rT * a + T * ra + rT * ra + U * (T + rT) * (a + ra) + TINY
    zero = tau == 0.0                                       # expf(-0) = 1: w = T * 0 = 0 exactly
    return Weights(tau, T, rT, Tn, rTn, np.where(zero, 0.0, w), np.where(zero, 0.0, rw))


def _acc(pk: Packed, wt: Weights, c, exact):
    """sum_k w_k c_k per ray (c: exact fp32 values) -> (centre, radius)."""
    c = np.asarray(c, np.float64)
    cen = seg_sum(pk, wt.w * c)
    if exact:
        return cen, np.zeros_like(cen)
    prop = seg_sum(pk, wt.rw * np.abs(c))
    mag = seg_sum(pk, (np.abs(wt.w) + wt.rw) * np.abs(c))
    h = pk.nchunks + 5
    return cen, prop + g32(h) * mag + (pk.n + h) * TINY


@dataclass
class Fwd:
    rgb: np.ndarray                 # [R, 3]
    rgb_r: np.ndarray
    depth: np.ndarray               # [R]
    depth_r: np.ndarray
    alpha: np.ndarray
    alpha_r: np.ndarray
    wt: Weights


def forward(offsets, shaded, depth, deltas, bg, exact: bool = False) -> Fwd:
    """wb_composite_fwd: shaded [S, 4] (r, g, b, sigma), depth [S], deltas [S], bg (3,) -> per-ray rgb, depth, alpha."""
    pk = packed(offsets)
    sh = np.asarray(shaded, f32).reshape(-1, 4)
    wt = weights(pk, sh[:, 3], np.asarray(deltas, f32).reshape(-1), exact)
    A, rA = _acc(pk, wt, np.ones(pk.S), exact)
    D, rD = _acc(pk, wt, np.asarray(depth, f32).reshape(-1), exact)
    bgv = np.asarray(bg, f32).astype(np.float64)
    rgb, rr = np.zeros((pk.R, 3)), np.zeros((pk.R, 3))
    for ch in range(3):
        Cc, rC = _acc(pk, wt, sh[:, ch], exact)
        rgb[:, ch] = bgv[ch] * (1.0 - A) + Cc
        if not exact:
            rr[:, ch] = abs(bgv[ch]) * rA + rC + g32(3) * (abs(bgv[ch]) * (np.abs(1.0 - A) + rA) + np.abs(Cc) + rC)
    empty = pk.n == 0                                       # rays without samples: rgb = bg, depth = alpha = 0, exactly
    rgb[empty], rr[empty] = bgv, 0.0
    return Fwd(rgb, rr, D, np.where(empty, 0.0, rD), A, np.where(empty, 0.0, rA), wt)


def hit_ok(alpha_c, alpha_r, hit, alpha_k):
    """The kernel's hit equals its own alpha > 0, is True where the alpha interval is above 0 and False where it is {0}."""
    hit, ak = np.asarray(hit).astype(bool), np.asarray(alpha_k)
    return (hit == (ak > 0)) & np.where(alpha_c - alpha_r > 0, hit, True) & np.where(alpha_c + alpha_r == 0, ~hit, True)


# ---- backward ---------------------------------------------------------------------------------------------------------------
@dataclass
class Bwd:
    g: np.ndarray                   # [S, 4] dL/d(r, g, b, sigma)
    r: np.ndarray


def loss_grad(rgb_k, target, loss_type: int, inv_count, exact: bool = False):
    """dL/drgb [R, 3] as wb_composite_bwd_loss forms it from the kernel's rgb (fp32 bit-exact unless exact)."""
    t = np.float64 if exact else f32
    d = np.asarray(rgb_k, t) - np.asarray(target, t)
    if loss_type == 0:
        g = t(2) * d
    elif loss_type == 1:
        g = np.sign(d).astype(t)
    else:
        g = np.where(np.abs(d) < 1, d, np.sign(d)).astype(t)
    return (g * t(inv_count)).astype(np.float64)


def backward(offsets, shaded, depth, deltas, bg, g_rgb, g_depth=None, g_alpha=None, exact: bool = False) -> Bwd:
    """wb_composite_bwd (and the compositing part of wb_composite_bwd_loss with g_rgb = loss_grad(...), g_depth = g_alpha = None)."""
    pk = packed(offsets)
    sh = np.asarray(shaded, f32).reshape(-1, 4).astype(np.float64)
    dl = np.asarray(deltas, f32).reshape(-1).astype(np.float64)
    t = np.asarray(depth, f32).reshape(-1).astype(np.float64)
    wt = weights(pk, sh[:, 3], dl, exact)
    bgv = np.asarray(bg, f32).astype(np.float64)
    gr = np.asarray(g_rgb, np.float64).reshape(-1, 3)
    gd = np.zeros(pk.R) if g_depth is None else np.asarray(g_depth, np.float64).reshape(-1)
    gain = np.zeros(pk.R) if g_alpha is None else np.asarray(g_alpha, np.float64).reshape(-1)
    gb = gr @ bgv
    ga = gain - gb
    rga = np.zeros(pk.R) if exact else g32(4) * (np.abs(gain) + np.abs(gr) @ np.abs(bgv))
    s = pk.ray
    terms = np.concatenate([gr[s] * sh[:, :3], (gd[s] * t)[:, None]], 1)
    gk = terms.sum(1) + ga[s]
    rgk = rga[s] if exact else rga[s] + g32(5) * (np.abs(terms).sum(1) + np.abs(ga[s]) + rga[s])
    prod = gk * wt.w
    incl = seg_cumsum(pk, prod)
    suffix = seg_sum(pk, prod)[s] - incl
    w = wt.w
    g = np.concatenate([gr[s] * w[:, None], np.zeros((pk.S, 1))], 1)
    if exact:
        gtau = gk * wt.Tn - suffix
        g[:, 3] = gtau * dl
        return Bwd(g, np.zeros_like(g))
    M = (np.abs(gk) + rgk) * (np.abs(w) + wt.rw)
    prop = np.abs(gk) * wt.rw + rgk * np.abs(w) + rgk * wt.rw
    prop_suffix = seg_sum(pk, prop)[s] - seg_cumsum(pk, prop)
    nc = pk.nchunks[s]
    rs0 = g32(nc + 5) * seg_sum(pk, M)[s] + g32(nc + 7) * seg_cumsum(pk, M) + np.maximum(prop_suffix, 0.0) * (1 + 1e-12)
    rs = rs0 + U * (np.abs(suffix) + rs0) + 8 * TINY
    gtau = gk * wt.Tn - suffix
    rg0 = np.abs(gk) * wt.rTn + rgk * wt.Tn + rgk * wt.rTn + rs
    rgt = rg0 + g32(2) * ((np.abs(gk) + rgk) * (wt.Tn + wt.rTn) + np.abs(suffix) + rs)
    g[:, 3] = gtau * dl
    r = np.zeros_like(g)
    r[:, :3] = np.abs(gr[s]) * wt.rw[:, None] + U * np.abs(gr[s]) * (np.abs(w) + wt.rw)[:, None] + TINY
    r[:, 3] = (rgt + U * (np.abs(gtau) + rgt)) * np.abs(dl) + TINY
    return Bwd(g, r)


def loss_value(rgb_k, target, loss_type: int, inv_count, R: int, sms: int = 132, exact: bool = False):
    """wb_composite_bwd_loss's *loss_out: sum over rays and channels of loss(d) * inv_count -> (centre, radius)."""
    t = np.float64 if exact else f32
    d = (np.asarray(rgb_k, t) - np.asarray(target, t)).astype(np.float64)
    ad = np.abs(d)
    terms = d * d if loss_type == 0 else ad if loss_type == 1 else np.where(ad < 1, 0.5 * d * d, ad - 0.5)
    inv = float(t(inv_count))
    cen = terms.sum() * inv
    if exact:
        return cen, 0.0
    ctas = min(-(-R // COMP_THREADS), sms * 32)
    nwarps = ctas * COMP_THREADS // 32
    iters = -(-R // (nwarps * 32))
    h = 2 + 2 + iters + 5 + 1 + min(nwarps, -(-R // 32))
    return cen, float(g32(h) * np.abs(terms).sum() * inv + h * 3 * R * TINY)


# ---- Adam ---------------------------------------------------------------------------------------------------------------------
def bias_corrections(b1, b2, step: int, exact: bool = False):
    """(bc1, bc2_sqrt) as wb_adam_step computes them on the host: double, then rounded to fp32 (exact: kept in float64)."""
    b1d, b2d = (float(b1), float(b2)) if exact else (float(f32(b1)), float(f32(b2)))
    bc1, bc2s = 1.0 - b1d ** step, np.sqrt(1.0 - b2d ** step)
    return (bc1, float(bc2s)) if exact else (float(f32(bc1)), float(f32(bc2s)))


class _I:
    """Interval (centre, radius) with one fp32 rounding per operation (none when exact)."""

    def __init__(self, c, r, exact):
        self.c, self.r, self.x = np.asarray(c, np.float64), np.asarray(r, np.float64), exact

    def _rnd(self, c, r):
        return _I(c, r if self.x else r + U * (np.abs(c) + r) + TINY, self.x)

    def __add__(self, o):
        return self._rnd(self.c + o.c, self.r + o.r)

    def __sub__(self, o):
        return self._rnd(self.c - o.c, self.r + o.r)

    def __mul__(self, o):
        return self._rnd(self.c * o.c, np.abs(self.c) * o.r + self.r * np.abs(o.c) + self.r * o.r)

    def __truediv__(self, o):
        lo = np.abs(o.c) - o.r
        assert np.all(lo > 0), "divisor interval contains 0"
        c = self.c / o.c
        return self._rnd(c, (self.r + np.abs(c) * o.r) / lo)

    def sqrt(self):
        c = np.sqrt(self.c)
        return self._rnd(c, np.maximum(np.sqrt(self.c + self.r) - c, c - np.sqrt(np.maximum(self.c - self.r, 0.0))))

    def fma(self, b, d):            # self * b + d, one rounding
        return self._rnd(self.c * b.c + d.c, np.abs(self.c) * b.r + self.r * np.abs(b.c) + self.r * b.r + d.r)


def adam(p, g, m, v, lr, wd, b1, b2, eps, step: int, grad_scale: float = 1.0, exact: bool = False, bc=None):
    """One wb_adam_step over one segment from its fp32 state -> (p, m, v) each (centre, radius).  bc: (bc1, bc2_sqrt) override."""
    bc1, bc2s = bias_corrections(b1, b2, step, exact) if bc is None else bc
    k = lambda x: _I(x, np.zeros_like(np.asarray(x, np.float64)), exact)
    if exact:
        P, G, M, V = (k(np.asarray(a, np.float64)) for a in (p, g, m, v))
        cst = lambda x: k(float(x))
    else:
        P, G, M, V = (k(np.asarray(a, f32).astype(np.float64)) for a in (p, g, m, v))
        cst = lambda x: k(float(f32(x)))
    B1, B2, one = cst(b1), cst(b2), k(1.0)
    gg = G * cst(grad_scale)
    if wd != 0.0:
        gg = cst(wd).fma(P, gg)
    M1 = B1.fma(M, (one - B1) * gg)
    V1 = B2.fma(V, ((one - B2) * gg) * gg)
    ss = cst(lr) / k(bc1)
    den = V1.sqrt() / k(bc2s) + cst(eps)
    P1 = P - ss * (M1 / den)
    return (P1.c, P1.r), (M1.c, M1.r), (V1.c, V1.r)


def adam_fp32(p, g, m, v, lr, wd, b1, b2, eps, step: int, grad_scale: float = 1.0):
    """wb_adam_kernel's fp32 chain bit-exactly -> (p with `p - fl(ss * q)`, p with `fmaf(-ss, q, p)`, m, v) as float32 arrays."""
    bc1, bc2s = (f32(x) for x in bias_corrections(b1, b2, step))
    p, g, m, v = (np.asarray(a, f32) for a in (p, g, m, v))
    b1, b2, eps, lr, wd, gs = (f32(x) for x in (b1, b2, eps, lr, wd, grad_scale))
    gg = g * gs
    if wd != 0:
        gg = fma32(wd, p, gg).astype(f32)
    m1 = fma32(b1, m, (f32(1) - b1) * gg).astype(f32)
    v1 = fma32(b2, v, ((f32(1) - b2) * gg) * gg).astype(f32)
    ss = lr / bc1
    q = m1 / (np.sqrt(v1) / bc2s + eps)
    return p - ss * q, fma32(-ss, q, p).astype(f32), m1, v1
