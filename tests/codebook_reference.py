"""float64 interval reference of the VQAD codebook selection (wb_codebook_rows_fwd / wb_codebook_rows_bwd, csrc/wb_codebook.cu)
(TEST INFRASTRUCTURE, NOT PRODUCT CODE).

For a block of logit rows [R, K] and a dictionary [K, F] it returns the argmax as an exact integer and, for every other output, a
centre and a radius: a kernel that rounds where wb_codebook.cu rounds, with expf within 2 ulp and its sums in any order, lands in
centre +- radius.  It builds on oracle/sdf_reference.py (U, fma32, g32, round_radius, fma_step) and, for the per-sample blend of
CodebookOctreeGrid, on its cells / features / interp_backward.

Rounding points (one warp per row, logit k held by lane k % 32 in slot i = k // 32, KPL = 8 slots for K <= 256, else 32)
  argmax     the first maximiser of the logits (torch.max's rule), exact.  The reference class takes the argmax of the fp32
             SOFTMAX in training mode (codebook_grid.py:119-120); see DESIGN.md for where the two can differ.
  y          t = fl(l - max) exactly; expf(t) within 2 ulp (the library is built without fast math); s = per-lane chains of KPL
             adds and wb_warp_sum's 5-level butterfly: gamma(KPL + 5) * sum|e|; fl(1 / s); y = fl(e * fl(1 / s)).
  keys       (hard - y) + y in fp32: exactly 0 off the argmax, and exactly 1 on it for every y in [0, 1] (1 - y is exact for
             y >= 1/2; otherwise it is within 2^-25 of 1 - y and adding y rounds back to 1).  So the training forward
             E = sum_k key_k dictionary[k] is dictionary[argmax] bit for bit, as the eval forward.
  c_k        the fp32 fma chain over f of dictionary[k, f] * dE[f], emulated on the centres (fma_step), dE's radius carried.
  dot        sum_k y_k c_k: per-lane fma chain and the butterfly, gamma(KPL + 5) * sum|y c|.
  g_logits   fl(y * fl(c - dot)): dot's radius is absolute, so it survives the cancellation in c - dot.
  g_dict     dictionary[argmax] += 1 * dE per row through shared atomics, one global atomic per CTA: a row's term passes through at
             most (#rows with that argmax) + 1 roundings counting the buffer's initial value: gamma(n + 1) * sum|terms|.
  skip       rows whose dE is exactly zero in every feature are skipped: their g_logits keep the caller's zeros.

exact=True turns every rounding off: the result is then the float64 operation (softmax, straight-through keys, products).
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Optional

import numpy as np

from oracle.sdf_reference import U, fma32, fma_step, g32, r32, round_radius     # noqa: F401

TINY = 2.0 ** -149                  # smallest fp32 subnormal
EXP_REL = 3.0 * 2.0 ** -23          # expf: 2 ulp from the correctly rounded value (half an ulp away), in the binade above at worst
FWD_CTAS_PER_SM, BWD_CTAS_PER_SM, WARPS = 16, 2, 8      # grid caps of wb_codebook_rows_fwd / _bwd, 8 warps (rows) per CTA
SMEM_DEFAULT = 48 * 1024


def kpl(K: int) -> int:
    return 8 if K <= 256 else 32


def bwd_smem(K: int, F: int) -> int:
    """Dynamic shared memory of wb_codebook_rows_bwd: the CTA's [K, F] dictionary gradient and one dE row per warp."""
    return (K * F + WARPS * 32) * 4


def first_max(logits) -> np.ndarray:
    """Index of the first maximum of every row (np.argmax returns the first occurrence), exact."""
    return np.argmax(np.asarray(logits, np.float64), axis=1).astype(np.int64)


def softmax(logits, exact: bool = False):
    """y of every logit -> (centre, radius) [R, K]."""
    L = np.asarray(logits, np.float64)
    m = L.max(1, keepdims=True)
    K = L.shape[1]
    with np.errstate(over="ignore", under="ignore", invalid="ignore"):
        if exact:
            e = np.exp(L - m)
            return e / e.sum(1, keepdims=True), np.zeros_like(L)
        t = r32(L - m)                                                     # fl(l - gmx); -inf when it overflows
        ec = r32(np.exp(t))
        er = EXP_REL * ec + 2 * TINY
        sc = ec.sum(1, keepdims=True)
        sr = er.sum(1, keepdims=True) + g32(kpl(K) + 5) * (ec + er).sum(1, keepdims=True)
        ic = r32(1.0 / sc)                                                 # s >= expf(0) - its radius > 0.99
        ir = round_radius(ic, 1.0 / sc, sr / (sc * (sc - sr)))
        v = ec * ic
        yc = r32(v)
        yr = round_radius(yc, v, ec * ir + er * ic + er * ir)
    return yc, yr


def _key_am(y_am, exact):
    if exact:
        return (1.0 - y_am) + y_am
    k = r32(r32(1.0 - y_am) + y_am)
    assert np.all(k == 1.0), "fl(fl(1 - y) + y) is 1 for every y in [0, 1]"
    return k


@dataclass
class Rows:
    am: np.ndarray                  # int64 [R] argmax
    E: np.ndarray                   # [R, F] centre
    E_r: np.ndarray                 # [R, F] radius
    y: Optional[np.ndarray]         # [R, K] softmax (training only)
    y_r: Optional[np.ndarray]


def rows_fwd(logits, dictionary, training: bool, exact: bool = False) -> Rows:
    """wb_codebook_rows_fwd: eval E = dictionary[argmax]; training E = sum_k key_k dictionary[k] (only the argmax's key is non-zero)."""
    D = np.asarray(dictionary, np.float64)
    am = first_max(logits)
    if not training:
        return Rows(am, D[am], np.zeros((am.shape[0], D.shape[1])), None, None)
    yc, yr = softmax(logits, exact)
    key = _key_am(yc[np.arange(am.shape[0]), am], exact)
    E = key[:, None] * D[am]
    return Rows(am, E if exact else r32(E), np.zeros_like(E), yc, yr)


@dataclass
class Bwd:
    g_logits: np.ndarray; g_logits_r: np.ndarray        # [R, K]
    g_dict: np.ndarray; g_dict_r: np.ndarray            # [K, F]
    skipped: np.ndarray                                 # bool [R]: dE exactly zero, g_logits untouched (0)
    n: np.ndarray                                       # int [K]: rows that add into each dictionary row


def rows_bwd(logits, dictionary, dE_c, dE_r=None, g_dict0=None, exact: bool = False, chunk: int = 2048, with_logits: bool = True) -> Bwd:
    """wb_codebook_rows_bwd from dE (centre, radius) [R, F]; g_dict0: the buffer's value before the call (default zeros).
    with_logits=False leaves g_logits at zero (eval mode: only the dictionary gets a gradient)."""
    L = np.asarray(logits, np.float64)
    D = np.asarray(dictionary, np.float64)
    R, K = L.shape
    F = D.shape[1]
    dc = np.asarray(dE_c, np.float64)
    dr = np.zeros_like(dc) if dE_r is None else np.asarray(dE_r, np.float64)
    g0 = np.zeros((K, F)) if g_dict0 is None else np.asarray(g_dict0, np.float64)
    skipped = ((dc == 0) & (dr == 0)).all(1)
    am = first_max(L)
    gl, glr = np.zeros((R, K)), np.zeros((R, K))
    for s in range(0, R if with_logits else 0, chunk):
        sl = slice(s, min(R, s + chunk))
        yc, yr = softmax(L[sl], exact)
        if exact:
            cc, cr = dc[sl] @ D.T, np.zeros((yc.shape[0], K))
            dot = (yc * cc).sum(1, keepdims=True)
            gl[sl] = yc * (cc - dot)
            continue
        cc, cr = np.zeros_like(yc), np.zeros_like(yc)
        for f in range(F):                                             # c = fmaf(dict[k, f], dE[f], c), f in order
            cc, cr = fma_step(cc, cr, D[None, :, f], 0.0, dc[sl, f:f + 1], dr[sl, f:f + 1])
        dot_c = (yc * cc).sum(1, keepdims=True)
        mag = (yc + yr) * (np.abs(cc) + cr)
        dot_r = (yc * cr + yr * np.abs(cc) + yr * cr).sum(1, keepdims=True) + g32(kpl(K) + 5) * mag.sum(1, keepdims=True)
        v = cc - dot_c
        d_c = r32(v)
        d_r = round_radius(d_c, v, cr + dot_r)
        w = yc * d_c
        gl[sl] = r32(w)
        glr[sl] = round_radius(gl[sl], w, yc * d_r + yr * np.abs(d_c) + yr * d_r)
    gl[skipped] = 0.0; glr[skipped] = 0.0
    live = ~skipped
    n = np.bincount(am[live], minlength=K)
    gd = g0.copy()
    gd_a, gd_r = np.abs(g0), np.zeros((K, F))
    for f in range(F):
        gd[:, f] += np.bincount(am[live], dc[live, f], K)
        gd_r[:, f] += np.bincount(am[live], dr[live, f], K)
        gd_a[:, f] += np.bincount(am[live], np.abs(dc[live, f]) + dr[live, f], K)
    if not exact:
        gd_r = gd_r + np.where(n[:, None] > 0, g32(n + 1)[:, None] * gd_a, 0.0)
    return Bwd(gl, glr, gd, gd_r, skipped, n)


# ---- cases shared by the CPU and GPU tests ------------------------------------------------------------------------------------
REGIMES = ("init", "unit", "wide", "ties", "equal", "extreme")


def make_logits(R: int, K: int, regime: str, rng, shared: bool = True) -> np.ndarray:
    """fp32 logits [R, K].  init: N(0, 0.01) (nerf_codebook's feature_std); unit: N(0, 1); wide: N(0, 30) (y underflows for all
    but the maximum); ties: N(0, 1) with the maximum duplicated in the same lane, in another lane or in another slot; equal:
    every logit of a row equal; extreme: rows at or below -3e38 (all equal, or spread down to -FLT_MAX).  shared: the first third
    of the rows of init / unit / wide share one argmax."""
    std = {"init": 0.01, "unit": 1.0, "wide": 30.0, "ties": 1.0}.get(regime, 1.0)
    if regime == "equal":
        return np.repeat(rng.standard_normal((R, 1)), K, 1).astype(np.float32)
    if regime == "extreme":
        L = np.full((R, K), -3.0e38, np.float32)
        spread = rng.random(R) < 0.5
        L[spread] = rng.uniform(-3.4e38, -3.0e38, (int(spread.sum()), K)).astype(np.float32)
        return L
    L = (rng.standard_normal((R, K)) * std).astype(np.float32)
    if regime == "ties" and K > 1:
        m = np.argmax(L, 1)
        mode = np.arange(R) % 3
        off = np.where(mode == 0, 32, np.where(mode == 1, 1, 32 * rng.integers(1, 4, R) + rng.integers(1, 32, R)))
        k2 = np.where(m + off < K, m + off, (m + off) % K)                        # same lane / another lane / another slot
        L[np.arange(R), k2] = L[np.arange(R), m]
    elif shared and K > 1:
        L[:R // 3, K // 2] += np.float32(8 * std)
    return L


def make_dE(R: int, F: int, rng, scale: float = 1.0) -> np.ndarray:
    """fp32 dE [R, F]: rows of N(0, 1); every 7th row exactly zero (skipped), every 5th non-zero only in feature F - 1, every
    3rd zero in feature 0 only."""
    d = (rng.standard_normal((R, F)) * scale).astype(np.float32)
    i = np.arange(R)
    d[i % 3 == 1, 0] = 0.0
    d[i % 5 == 2, :F - 1] = 0.0
    d[i % 7 == 3] = 0.0
    return d


# ---- fp32 emulation of the kernels (CPU tests: emulations land inside, mutated emulations outside) --------------------------
MUTATIONS = ("tie_high", "dot_no_warp_sum", "key_one", "dict_by_y", "skip_lane0")


def _ulp_jitter(x32, rng, ulps=2):
    """x (fp32) moved by a random number of ulps in [-ulps, ulps], never below 0 (expf within 2 ulp)."""
    out = x32.copy()
    steps = rng.integers(-ulps, ulps + 1, x32.shape)
    for s in range(1, ulps + 1):
        up, dn = steps >= s, steps <= -s
        out = np.where(up, np.nextafter(out, np.float32(np.inf)), out)
        out = np.where(dn & (out > 0), np.nextafter(out, np.float32(0)), out)
    return out


def _warp_sum(v, rng):
    """wb_warp_sum over the last axis (32 lanes) after a random lane permutation: xor butterfly, fp32 adds."""
    v = v[..., rng.permutation(32)].astype(np.float32)
    for o in (16, 8, 4, 2, 1):
        v = (v + v[..., np.arange(32) ^ o]).astype(np.float32)
    return v[..., 0]


def _lanes(logits):
    """[R, K] -> [R, KPL, 32] fp32 (slot i, lane), padded with -inf, and the index k of every element."""
    R, K = logits.shape
    P = kpl(K)
    Lg = np.full((R, P * 32), -np.inf, np.float32)
    Lg[:, :K] = logits
    return Lg.reshape(R, P, 32), np.arange(P * 32).reshape(P, 32)


def _emu_softmax(logits, rng, mutation):
    R, K = logits.shape
    Lg, kk = _lanes(np.asarray(logits, np.float32))
    if mutation == "tie_high":
        am = K - 1 - np.argmax(Lg.reshape(R, -1)[:, :K][:, ::-1], axis=1)
    else:
        am = np.argmax(Lg.reshape(R, -1)[:, :K], axis=1)
    gmx = Lg.max((1, 2), keepdims=True)
    with np.errstate(over="ignore", invalid="ignore"):
        t = (Lg - gmx).astype(np.float32)
        e = np.where(kk < K, _ulp_jitter(np.exp(t.astype(np.float64)).astype(np.float32), rng), np.float32(0))
    s = np.zeros((R, 32), np.float32)
    for i in rng.permutation(e.shape[1]):
        s = (s + e[:, i]).astype(np.float32)
    s = _warp_sum(s, rng)
    inv = (np.float32(1) / s).astype(np.float32)
    y = (e * inv[:, None, None]).astype(np.float32)
    return am, y, kk


def emulate_fwd(logits, dictionary, training, rng, mutation=None):
    """wb_codebook_rows_fwd in fp32 -> (argmax, E)."""
    D = np.asarray(dictionary, np.float32)
    am, y, kk = _emu_softmax(logits, rng, mutation)
    if not training:
        return am, D[am].astype(np.float64)
    K, F = D.shape
    hard = (kk[None] == am[:, None, None]).astype(np.float32)
    key = ((hard - y).astype(np.float32) + y).astype(np.float32)
    Dp = np.zeros((kk.size, F), np.float32); Dp[:K] = D
    Dp = Dp.reshape(kk.shape + (F,))
    E = np.zeros((am.shape[0], F))
    for f in range(F):
        acc = np.zeros((am.shape[0], 32))
        for i in range(kk.shape[0]):
            acc = np.where(kk[i] < K, fma32(key[:, i], Dp[None, i, :, f], acc), acc)
        E[:, f] = _warp_sum(acc.astype(np.float32), rng)
    return am, E


def emulate_bwd(logits, dictionary, dE, rng, g_dict0=None, mutation=None, ctas=4):
    """wb_codebook_rows_bwd in fp32 -> (g_logits [R, K], g_dict [K, F]); the rows go to `ctas` CTAs at random, each CTA adds its
    rows' terms in a random order, the CTA partials reach the buffer in a random order."""
    D = np.asarray(dictionary, np.float32).astype(np.float64)
    dE = np.asarray(dE, np.float32).astype(np.float64)
    R, K = np.asarray(logits).shape
    F = D.shape[1]
    skip = (dE[:, 0] == 0) if mutation == "skip_lane0" else (dE == 0).all(1)
    am, y, kk = _emu_softmax(logits, rng, mutation)
    y = y.astype(np.float64)
    Dp = np.zeros((kk.size, F)); Dp[:K] = D
    Dp = Dp.reshape(kk.shape + (F,))
    c = np.zeros(y.shape)
    for f in range(F):
        c = fma32(Dp[None, :, :, f], dE[:, None, None, f], c)
    c = np.where(kk[None] < K, c, 0.0)
    dot = np.zeros((R, 32))
    for i in range(kk.shape[0]):
        dot = np.where(kk[i] < K, fma32(y[:, i], c[:, i], dot), dot)
    if mutation == "dot_no_warp_sum":
        dot = dot.astype(np.float32)[:, None, :]
    else:
        dot = _warp_sum(dot.astype(np.float32), rng)[:, None, None]
    g = r32(y * r32(c - dot)).reshape(R, -1)[:, :K]
    if mutation == "key_one":
        g = np.zeros_like(g)
    g[skip] = 0.0
    hard = (kk[None] == am[:, None, None]).astype(np.float64)
    key = (y if mutation == "dict_by_y" else r32(r32(hard - y) + y)).reshape(R, -1)[:, :K]
    gd = np.zeros((K, F)) if g_dict0 is None else np.asarray(g_dict0, np.float64).copy()
    cta = rng.integers(0, ctas, R)
    for b in rng.permutation(ctas):
        rows = np.flatnonzero((cta == b) & ~skip)
        part = np.zeros((K, F), np.float32)
        for r in rng.permutation(rows):
            nz = np.flatnonzero(key[r] != 0)
            part[nz] = (part[nz] + r32(key[r, nz, None] * dE[r][None])).astype(np.float32)
        gd = np.where(part != 0, r32(gd + part), gd)
    return g, gd
