"""float64 interval reference of wb_sdf_train for decoders with 2 to 4 hidden layers (TEST INFRASTRUCTURE, NOT PRODUCT CODE).

It builds on oracle/sdf_reference.py (same Field, same forward, same rounding model and accumulation bounds) and differs from
its `train` only where wb_sdf_train_deep_kernel computes differently from the one-hidden-layer kernel:

  backward   the kernel carries dy from the top: delta of the last hidden layer = fl(dy * wout_j) where a_j > 0, delta of layer
             k-1 = the fp32 chain over the units of W_k[j, :] delta_k[j] (any order: gamma(H)), masked by layer k-1's relu; the
             feature gradient is the same chain through W0, scattered without a further product with dy.  Weight and bias
             gradients are chains over the CTA's samples of delta_k h_{k-1} and delta_k.
  heights    a CTA of 256 threads (8 warp partials) works on tiles of T samples, T in DEEP_TILES (the largest that fits in shared
             memory); with `tile` unknown every T is allowed and the tallest tree is used.  Every sum over samples and CTAs is
             bounded order-free (the CTA partition of the per-CTA partials is not emulated).

With exact=True, or for a decoder with one hidden layer, it is oracle.sdf_reference.train."""
from __future__ import annotations

from typing import Optional, Sequence

import numpy as np

from oracle import sdf_reference as S

DEEP_TILES = (32, 64, 96, 128)       # sample tiles of wb_sdf_train_deep_kernel
DEEP_WARPS = 256 // 32               # its threads per CTA / 32


def heights(N: int, sms: int, tiles: Sequence[int]) -> S.TrainHeights:
    """The tallest summation trees of a launch over N samples that may use any tile in `tiles` (S.TrainHeights per tile)."""
    out = S.TrainHeights(0, 0, 0)
    for T in tiles:
        ntiles = max(1, -(-N // T))
        cmin, cmax = min(ntiles, sms), min(ntiles, S.MAX_CTAS_PER_SM * sms)
        t = -(-ntiles // cmin)
        out = S.TrainHeights(max(out.chain, t * T), max(out.tiles, t), max(out.ctas, cmax))
    return out


def train(field: S.Field, coords: np.ndarray, gt: np.ndarray, lods: Sequence[int], exact: bool = False, sms: int = 132,
          tile: Optional[int] = None) -> S.Train:
    """Loss sum_lod sum_i (y_i - gt_i)^2 / N and its gradients as wb_sdf_train_deep_kernel rounds them -> S.Train."""
    if exact or len(field.Ws) <= 2:
        return S.train(field, coords, gt, lods, exact=exact, sms=sms)
    coords = np.asarray(coords, np.float32)
    gt = np.asarray(gt, np.float64).reshape(-1)
    N = coords.shape[0]
    U, g32 = S.U, S.g32
    h = heights(N, sms, (tile,) if tile else DEEP_TILES)
    nlaunch = len(lods)
    loss_h = h.tiles + 5 + DEEP_WARPS + 2 + nlaunch * h.ctas           # thread chain, warp tree, warp partials, fl(1/N) and product, atomics
    dec_h = h.chain + 5 + DEEP_WARPS + nlaunch * h.ctas
    nparams = field.packed().size
    loss_c = loss_r = 0.0
    dec_c, dec_r, dec_a = np.zeros(nparams), np.zeros(nparams), np.zeros(nparams)
    grid = [(np.zeros(f.shape), np.zeros(f.shape)) for f in field.feats]
    grid_a = [np.zeros(f.shape) for f in field.feats]
    grid_n = [np.zeros(f.shape[0]) for f in field.feats]
    amb = np.zeros(N, bool)
    ntiles = -(-N // S.TILE)
    layers = list(zip(field.Ws, field.bs))
    offs, o = [], 0
    for W, b in layers:
        offs.append(o); o += W.size + b.size
    last = len(layers) - 1
    for lod in lods:
        fw = S.forward(field, coords, lod, False, in_order=ntiles <= sms)   # batches of many tiles: any-order bounds (cost)
        amb |= fw.amb
        dc = fw.y - gt
        dr = fw.y_r + U * (np.abs(dc) + fw.y_r)
        sq_c, sq_r = dc * dc, 2 * np.abs(dc) * dr + dr * dr
        loss_c += sq_c.sum() / N
        loss_r += sq_r.sum() / N + g32(loss_h) * (sq_c + sq_r).sum() / N
        dyc, dyr = S._mul(dc, dr, 2.0 / N, 0.0, False)
        dyr = dyr + (2 * U + U * U) * (np.abs(dyc) + dyr)                   # fl(fl(1/N) * 2d)
        ins = [(fw.x, fw.x_r)] + list(zip(fw.hs, fw.hs_r))

        def accumulate(li, dac, dar):
            W, b = layers[li]
            xc, xr = ins[li]
            s = offs[li]
            dec_c[s:s + W.size] += (dac.T @ xc).reshape(-1)
            dec_r[s:s + W.size] += (np.abs(dac).T @ xr + dar.T @ np.abs(xc) + dar.T @ xr).reshape(-1)
            dec_a[s:s + W.size] += ((np.abs(dac) + dar).T @ (np.abs(xc) + xr)).reshape(-1)
            s += W.size
            dec_c[s:s + b.size] += dac.sum(0); dec_r[s:s + b.size] += dar.sum(0); dec_a[s:s + b.size] += (np.abs(dac) + dar).sum(0)

        accumulate(last, dyc[:, None], dyr[:, None])                         # dL/dwout = sum dy relu(a), dL/dbout = sum dy
        wo = field.Ws[-1][0].astype(np.float64)[None]
        act = fw.act[last - 1]
        Dc, Dr = S._mul(dyc[:, None], dyr[:, None], wo, 0.0, True)          # delta = fl(dy * wout_j) where a_j > 0
        Dc, Dr = np.where(act, Dc, 0.0), np.where(act, Dr, 0.0)
        for li in range(last - 1, -1, -1):
            accumulate(li, Dc, Dr)
            Wd = np.abs(field.Ws[li].astype(np.float64))
            nDc = Dc @ field.Ws[li].astype(np.float64)                       # chain over the units of W_li[j, :] delta[j]
            nDr = Dr @ Wd + g32(field.Ws[li].shape[0]) * (np.abs(Dc) + Dr) @ Wd
            if li > 0:
                nDc, nDr = np.where(fw.act[li - 1], nDc, 0.0), np.where(fw.act[li - 1], nDr, 0.0)
            Dc, Dr = nDc, nDr
        pd = field.pos_dim
        nl = lod + 1
        sc = S._scatter(field, Dc[:, pd:], Dr[:, pd:], fw.cells, nl, field.multiscale == "sum" and nl > 1, True)
        for k, (C, R, A, n) in enumerate(sc):
            grid[k][0][...] += C; grid[k][1][...] += R; grid_a[k] += A; grid_n[k] += n
    dec_r = dec_r + g32(dec_h) * dec_a
    grid = [(C, R + g32(n)[:, None] * A) for (C, R), A, n in zip(grid, grid_a, grid_n)]     # one atomic per contribution
    return S.Train(loss_c, loss_r, dec_c, dec_r, grid, amb, grid_n, nlaunch * h.ctas)
