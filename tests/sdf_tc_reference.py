"""float64 fp16-faithful interval reference of the precision-1 SDF training step, wb_sdf_train_tc (TEST INFRASTRUCTURE, NOT
PRODUCT CODE).

It uses the gathers and scatters of oracle/sdf_reference.py (octree fields; hash fields through the hook that
tests/sdf_hash_reference.py installs on import) and the fp16 rounding and accumulation model of oracle/tc_decoders.py (f16,
gamma), and rounds exactly where csrc/wb_sdf_train_tc.cu rounds.  Every output is a centre and a radius: a kernel that rounds at
these points and accumulates in fp32, in whatever order, lands in centre +- radius.  Through an fp16 rounding an interval [c - r,
c + r] becomes [f16(c - r), f16(c + r)] (f16 is monotone); through a sum of n terms the radius grows by the radii of the terms and
gamma(n) sum|terms| (fp16 x fp16 products are exact in fp32).

Rounding points (the autocast nn.Linear contract):
  forward   x = fp16([position embedding | features]); W, b = fp16(W), fp16(b); a hidden layer h = fp16(relu(b + x W^T));
            y = fp16(bout + h wout^T); d = y - gt (fp32), loss = sum d^2 / N.
  backward  dY = fp16(fl(2 d inv_count) * scale) with scale = 2^-e, frexp(inv_count) = (m, e); dY_{nh-1} = fp16(dY wout_j) where
            h_j > 0; dW_l += dY_l^T [X_l | 1]; dY_{l-1} = fp16(dY_l W_l) where X_l > 0; the feature gradient dY_0 W_0 stays fp32
            (autocast rounds it to fp16: a stated deviation); weight and feature gradients are divided by scale.
Samples whose relu mask the intervals cannot settle are flagged in `amb`; the checks drop them.
With rounding=False nothing is rounded, scale = 1 and every radius is 0: the float64 gradient of the float64 decoder.
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import List, Sequence, Tuple

import numpy as np

from oracle import sdf_reference as S
from oracle.tc_decoders import f16, gamma

ROWS = 64                        # samples per tile of wb_sdf_train_tc
U = 2.0 ** -24                   # one fp32 rounding (round to nearest)


def loss_scale(inv_count: float) -> float:
    """The power of two wb_sdf_train_tc multiplies dY by: inv_count * scale in [0.5, 1)."""
    if inv_count <= 0:
        return 1.0
    _, e = math.frexp(inv_count)
    return 2.0 ** -e


@dataclass
class TcTrain:
    loss: float
    loss_r: float
    dec: np.ndarray               # packed [W0, b0, ..., Wout, bout] gradient: centre
    dec_r: np.ndarray             #   radius
    grid: List[Tuple[np.ndarray, np.ndarray]]     # per feature level (octree) or the one table (hash): (centre, radius)
    amb: np.ndarray               # [N] samples with an unsettled relu mask
    dfeat: List[Tuple[np.ndarray, np.ndarray]]    # per loss LOD: the feature gradient [N, feat_dim] before the scatter


def heights(N: int) -> Tuple[int, int]:
    """Summation heights over the samples of one launch, for any grid: (weight-gradient entry, loss / dL/dbout).  A 64-sample
    wgmma chain (or a 64-sample fmaf chain) per tile, one addition per tile of a CTA (one CTA may take every tile), the warp
    tree and the four warps of the CTA, one atomic per CTA."""
    T = max(1, -(-N // ROWS))
    return ROWS + 2 * T + 2, 2 * T + 5 + 4 + 3


def _round(c, r, on):
    if not on:
        return c, r
    lo, hi = f16(c - r), f16(c + r)
    return (lo + hi) / 2, (hi - lo) / 2


def _relu_round(c, r, on):
    lo, hi = np.maximum(c - r, 0.0), np.maximum(c + r, 0.0)
    if on:
        lo, hi = f16(lo), f16(hi)
    return (lo + hi) / 2, (hi - lo) / 2, (lo == 0) & (hi > 0)


def _linear(xc, xr, W, b, on):
    """b + x W^T with exact W, b and an interval x, fp32 sums of K + 1 terms in any order."""
    c = xc @ W.T + b
    r = xr @ np.abs(W).T
    if on:
        r = r + gamma(W.shape[1] + 1) * ((np.abs(xc) + xr) @ np.abs(W).T + np.abs(b))
    return c, r


def _gram(ac, ar, bc, br, n, on):
    """sum over samples of a_s^T b_s (a [N, M], b [N, K]) with interval operands and a summation height n -> [M, K] (c, r)."""
    c = ac.T @ bc
    r = np.abs(ac).T @ br + ar.T @ np.abs(bc) + ar.T @ br
    if on:
        r = r + gamma(n) * ((np.abs(ac) + ar).T @ (np.abs(bc) + br))
    return c, r


def train_tc(field: S.Field, coords: np.ndarray, gt: np.ndarray, lods: Sequence[int], rounding: bool = True) -> TcTrain:
    """Loss sum_lod sum_i (y_i - gt_i)^2 / N and its gradients as wb_sdf_train_tc rounds them, one launch per loss LOD."""
    on = rounding
    coords = np.asarray(coords, np.float32)
    gt = np.asarray(gt, np.float64).reshape(-1)
    N = coords.shape[0]
    inv = float(np.float32(1.0 / N)) if on else 1.0 / N      # the kernel's inv_count is a float32
    scale = loss_scale(inv) if on else 1.0
    hW, hL = heights(N)
    Ws = [f16(W) if on else W.astype(np.float64) for W in field.Ws]
    bs = [f16(b) if on else b.astype(np.float64) for b in field.bs]
    nh = len(Ws) - 1
    dec_c = [np.zeros(a.size) for W, b in zip(Ws, bs) for a in (W, b)]
    dec_r = [np.zeros(a.size) for a in dec_c]
    grid = [[np.zeros(f.shape), np.zeros(f.shape), np.zeros(f.shape), np.zeros(f.shape[0])] for f in field.feats]
    loss_c = loss_r = 0.0
    amb = np.zeros(N, bool)
    dfeats = []
    ones = np.ones((N, 1))

    def acc(i, gc, gr):
        dec_c[i] += gc.reshape(-1); dec_r[i] += gr.reshape(-1)

    for lod in lods:
        nl = lod + 1
        pc, pr = S._embed(field, coords.astype(np.float64), not on)
        fc, fr, famb, cl = S.features(field, coords, nl, exact=not on)
        amb |= famb
        xs = [_round(np.concatenate([pc, fc], -1), np.concatenate([pr, fr], -1), on)]
        for l in range(nh):
            hc, hr, a = _relu_round(*_linear(*xs[-1], Ws[l], bs[l], on), on)
            amb |= a.any(1)
            xs.append((hc, hr))
        yc, yr = _linear(*xs[-1], Ws[-1], bs[-1], on)
        yc, yr = _round(yc[:, 0], yr[:, 0], on)
        dc = yc - gt
        dr = yr + (U * (np.abs(dc) + yr) if on else 0.0)
        sq_c, sq_r = dc * dc, 2 * np.abs(dc) * dr + dr * dr
        loss_c += float(sq_c.sum() * inv)
        loss_r += float(sq_r.sum() * inv + (gamma(hL) * (sq_c + sq_r).sum() * inv if on else 0.0))
        vc, vr = 2.0 * dc * inv * scale, 2.0 * dr * inv * scale
        if on:
            vr = vr + U * (np.abs(vc) + vr)                    # fl(inv * 2d); the scale is exact
        dyc, dyr = _round(vc, vr, on)
        acc(2 * nh, *_gram(dyc[:, None], dyr[:, None], *xs[-1], hW, on))
        acc(2 * nh + 1, *_gram(dyc[:, None], dyr[:, None], ones, 0.0 * ones, hL, on))
        wo = Ws[-1][0][None]
        mask = xs[-1][0] > 0
        Dc, Dr = _round(dyc[:, None] * wo, dyr[:, None] * np.abs(wo), on)
        Dc, Dr = np.where(mask, Dc, 0.0), np.where(mask, Dr, 0.0)
        for l in range(nh - 1, -1, -1):
            acc(2 * l, *_gram(Dc, Dr, *xs[l], hW, on))
            acc(2 * l + 1, *_gram(Dc, Dr, ones, 0.0 * ones, hW, on))
            nc, nr = Dc @ Ws[l], Dr @ np.abs(Ws[l])
            if on:
                nr = nr + gamma(Ws[l].shape[0] + 1) * ((np.abs(Dc) + Dr) @ np.abs(Ws[l]))
            if l > 0:
                mask = xs[l][0] > 0
                nc, nr = _round(nc, nr, on)
                nc, nr = np.where(mask, nc, 0.0), np.where(mask, nr, 0.0)
            Dc, Dr = nc, nr
        gc, gr = Dc[:, field.pos_dim:] / scale, Dr[:, field.pos_dim:] / scale
        dfeats.append((gc, gr))
        sc = S._scatter(field, gc, gr, cl, nl, field.multiscale == "sum" and nl > 1, on)
        for k, (C, R, A, n) in enumerate(sc):
            grid[k][0] += C; grid[k][1] += R; grid[k][2] += A; grid[k][3] += n
    grid = [(C, R + (S.g32(n)[:, None] * A if on else 0.0)) for C, R, A, n in grid]
    return TcTrain(loss_c, loss_r, np.concatenate(dec_c) / scale, np.concatenate(dec_r) / scale, grid, amb, dfeats)


def footprint(in_dim: int, pos_dim: int, feat_dim: int, H: int, nh: int) -> int:
    """Dynamic shared memory of a wb_sdf_train_tc launch (bytes), or -1 above 227 KB: the same plan as sdf_tc_plan."""
    up = lambda v, m: (v + m - 1) // m * m
    Hp, K0p = up(H, 16), up(in_dim, 16)
    off = sum(Hp * (K0p if l == 0 else Hp) * 2 for l in range(nh))
    off += up(nh * Hp * 2, 16) + (Hp + 4) * 4
    off = up(off, 128)
    acc = sum(H * ((in_dim if l == 0 else H) + 1) for l in range(nh)) + H
    off = up(off + acc * 4, 128)
    off += sum(((K0p if l == 0 else Hp) // 8 + 1) * 1024 for l in range(nh + 1))
    off += up(Hp, 64) // 8 * 1024 + up(ROWS * (feat_dim + 1) * 4, 16) + ROWS * 4 + 2 * 4 * 4
    return off if off <= 227 * 1024 else -1
