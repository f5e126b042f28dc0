"""Exact and float64 references of the kernels that decide which table rows and which cells a sample touches (TEST INFRASTRUCTURE,
NOT PRODUCT CODE): the stand-alone hash-grid kernels (wb_hashgrid_fwd / _bwd), the occupancy bitmasks (wb_octree_build_bits /
_coarse) and the two halves of NeuralRadianceField.prune (wb_prune_samples / wb_prune_update).

Hash grid (wb_common.cuh: wb_cell, wb_corner_setup, wb_corner_indices; wb_core.cu: wb_make_grid)
  cell       per axis x = fmaf(c, res/2, res/2), clamped by fmaxf(0, fminf(hi, x)) with hi = fl(res - 1 - 1e-5) (a NaN coordinate
             lands on hi: fminf drops the NaN), p = floor(x), w = x - p (exact), 1 - w rounded.  Bit-exact.
  coefs      ((i_x i_y) i_z ...) z fastest, each product rounded to fp32.  Bit-exact.
  rows       level-local; dense levels (res^3 < 2^bitwidth) x + y res + z res^2 with the +1 corner kept on the cell's own row where
             the cell is the level's last on that axis (weight 0 there; `top_clamp=False` gives the unclamped arithmetic of the
             reference kernel), hashed levels (x ^ y*2654435761 ^ z*805459861) & (2^bitwidth - 1).  Exact.
  forward    emulated: fl(v_0 c_0), then fmaf over corners 1..7 -- bit-exact.  Interval: the float64 sum of v_j c_j (fp32 c_j) as
             the centre, gamma(8) * sum |v_j c_j| as the radius.
  backward   every table entry is its initial value plus fl(g c_j) for each (sample, LOD, corner) whose gradient is not skipped
             (F == 2: both components zero skips the pair; otherwise per feature), added by fp32 atomics in any order: centre = the
             float64 sum, radius = gamma(k) * (|initial| + sum |terms|) for k atomic adds.  Untouched entries are exact.

Occupancy bitmasks (wb_spc.cu)
  bits       bit x<<2L | y<<L | z of uint32 word (index >> 5), bit (index & 31), for every point of the level.
  coarse     the same at coarse_level for every cell c = p >> (level - coarse_level) and its 26 neighbours inside the grid.

Prune (nerf.py:186-198 and wb_prune_samples)
  samples    ((p + u) / 2^L) * 2 - 1, four fp32 ops; u explicit or jitter_stream(seed, N, 5)[:, :3] keyed by (seed, cell, axis);
             directions from columns 3 and 4 of the same stream.
  update     occupancy = max(density, fl(occupancy * decay)) with torch.max's NaN propagation; keep = occupancy > min_density."""
from __future__ import annotations

import numpy as np

import octree_reference as OR

f32, f64 = np.float32, np.float64
P1, P2 = 2654435761, 805459861
U = 2.0 ** -24


def gamma(n):
    n = np.asarray(n, f64)
    return n * U / (1.0 - n * U)


# ---- hash grid --------------------------------------------------------------------------------------------------------------
def is_dense(res: int, bitwidth: int) -> bool:
    T = 2 ** bitwidth
    return res < T and res ** 2 < T and res ** 3 < T


def level_rows(res: int, bitwidth: int) -> int:
    """Rows of one level of MultiTable: min(res^3, 2^bitwidth)."""
    return min(res ** 3, 2 ** bitwidth)


def table_layout(resolutions, bitwidth):
    begin = np.zeros(len(resolutions) + 1, np.int64)
    begin[1:] = np.cumsum([level_rows(int(r), bitwidth) for r in resolutions])
    return begin


def clamp_hi(res: int) -> f32:
    return f32(f64(res - 1) - 1e-5)


def cell_axis(c, res: int):
    """wb_cell: -> (p int64, w fp32, 1 - w fp32)."""
    c = np.asarray(c, f32)
    h = f32(0.5 * res)
    with np.errstate(over="ignore", invalid="ignore"):
        x = OR.fma32(c, np.full_like(c, h), np.full_like(c, h))
    x = np.fmax(f32(0.0), np.fmin(clamp_hi(res), x)).astype(f32)
    p = np.floor(x)
    w = (x - p).astype(f32)
    return p.astype(np.int64), w, (f32(1.0) - w).astype(f32)


def corners(coords, res: int, bitwidth: int, top_clamp: bool = True):
    """-> (rows int64 [N, 8] level-local, coefs fp32 [N, 8]) of one level, corner j = (x + (j>>2&1), y + (j>>1&1), z + (j&1))."""
    c = np.asarray(coords, f32)
    (px, wx, ix), (py, wy, iy), (pz, wz, iz) = (cell_axis(c[:, a], res) for a in range(3))
    xy = [ix * iy, ix * wy, wx * iy, wx * wy]                       # fp32 products
    cf = np.stack([(xy[j >> 1] * (wz if j & 1 else iz)).astype(f32) for j in range(8)], 1)
    T, dense = 2 ** bitwidth, is_dense(res, bitwidth)
    rows = np.zeros((c.shape[0], 8), np.int64)
    for j in range(8):
        x, y, z = (p + ((j >> s) & 1) for p, s in ((px, 2), (py, 1), (pz, 0)))
        if dense and top_clamp:
            x, y, z = (np.where(p < res - 1, q, p) for p, q in ((px, x), (py, y), (pz, z)))
        if dense:
            rows[:, j] = x + y * res + z * res * res
        else:
            rows[:, j] = (x ^ ((y * P1) & 0xFFFFFFFF) ^ ((z * P2) & 0xFFFFFFFF)) & (T - 1)
    return rows, cf


def hashgrid_fwd(coords, table, resolutions, bitwidth, begin=None):
    """-> (emulated fp32 [N, L*F], centre float64 [N, L*F], radius float64 [N, L*F])."""
    table = np.asarray(table, f32)
    begin = table_layout(resolutions, bitwidth) if begin is None else begin
    N, F = np.asarray(coords).shape[0], table.shape[1]
    emu, cen, rad = [], [], []
    for l, res in enumerate(resolutions):
        rows, cf = corners(coords, int(res), bitwidth)
        v = table[begin[l] + rows]                                   # [N, 8, F]
        with np.errstate(invalid="ignore", over="ignore"):
            a = (v[:, 0] * cf[:, :1]).astype(f32)
            for j in range(1, 8):
                a = OR.fma32(v[:, j], np.broadcast_to(cf[:, j:j + 1], a.shape), a)
            terms = v.astype(f64) * cf[:, :, None].astype(f64)
        emu.append(a); cen.append(terms.sum(1)); rad.append(gamma(8) * np.abs(terms).sum(1))
    return (np.concatenate(emu, 1).reshape(N, -1), np.concatenate(cen, 1).reshape(N, -1), np.concatenate(rad, 1).reshape(N, -1))


def hashgrid_bwd(coords, grad_feats, grad_table0, resolutions, bitwidth, begin=None):
    """-> (centre float64 [rows, F], radius float64 [rows, F], k int64 [rows, F] atomic adds per entry)."""
    g0 = np.asarray(grad_table0, f32)
    n_rows, F = g0.shape
    begin = table_layout(resolutions, bitwidth) if begin is None else begin
    L = len(resolutions)
    go = np.asarray(grad_feats, f32).reshape(-1, L, F)
    cen = g0.astype(f64).copy(); mag = np.abs(cen); k = np.zeros((n_rows, F), np.int64)
    for l, res in enumerate(resolutions):
        rows, cf = corners(coords, int(res), bitwidth)
        gl = go[:, l]                                                 # [N, F]
        live = np.repeat((gl != 0).any(1, keepdims=True), F, 1) if F == 2 else (gl != 0)
        for f in range(F):
            m = live[:, f]
            if not m.any():
                continue
            t = (gl[m, f][:, None] * cf[m]).astype(f32).astype(f64)   # fl(g c_j) [n, 8]
            r = (begin[l] + rows[m]).ravel()
            cen[:, f] += np.bincount(r, weights=t.ravel(), minlength=n_rows)
            mag[:, f] += np.bincount(r, weights=np.abs(t).ravel(), minlength=n_rows)
            k[:, f] += np.bincount(r, minlength=n_rows)
    return cen, gamma(k) * mag, k


# ---- occupancy bitmasks -----------------------------------------------------------------------------------------------------
def _words(idx, nbits):
    words = np.zeros((nbits + 31) // 32, np.uint32)
    idx = np.unique(np.asarray(idx, np.int64))
    np.bitwise_or.at(words, idx >> 5, (np.uint32(1) << (idx & 31).astype(np.uint32)))
    return words


def build_bits(points, level: int):
    """Exact wb_octree_build_bits: uint32 [(8^level + 31) // 32]."""
    p = np.asarray(points, np.int64).reshape(-1, 3)
    return _words((p[:, 0] << (2 * level)) | (p[:, 1] << level) | p[:, 2], 8 ** level)


def build_coarse(points, level: int, coarse_level: int):
    """Exact wb_octree_build_coarse: occupied coarse cells dilated by one cell in each of the 26 directions, clipped at the border."""
    n = 1 << coarse_level
    occ = np.zeros((n + 2, n + 2, n + 2), bool)
    c = np.asarray(points, np.int64).reshape(-1, 3) >> (level - coarse_level)
    occ[c[:, 0] + 1, c[:, 1] + 1, c[:, 2] + 1] = True
    dil = np.zeros_like(occ)
    for dx in (-1, 0, 1):
        for dy in (-1, 0, 1):
            for dz in (-1, 0, 1):
                dil[1:-1, 1:-1, 1:-1] |= occ[1 + dx:n + 1 + dx, 1 + dy:n + 1 + dy, 1 + dz:n + 1 + dz]
    return _words(np.flatnonzero(dil[1:-1, 1:-1, 1:-1].ravel()), 8 ** coarse_level)


def bbox(points, level: int):
    """The occupied extent as exact dyadic cell faces: ([lo x, y, z], [hi x, y, z]) in [-1, 1]."""
    p = np.asarray(points, np.int64).reshape(-1, 3)
    res = 2.0 ** level
    return [2.0 * m / res - 1.0 for m in p.min(0)], [2.0 * (m + 1) / res - 1.0 for m in p.max(0)]


# ---- prune ------------------------------------------------------------------------------------------------------------------
def prune_stream(seed: int, N: int):
    """[N, 5] fp32: u (columns 0..2) and the two direction draws (3, 4) of wb_prune_samples, keyed by (seed, cell, draw)."""
    return OR.jitter_stream(seed, N, 5)


def prune_samples(points, level: int, u):
    """((p + u) / 2^level) * 2 - 1 op by op in fp32 (nerf.py:189-192)."""
    p = np.asarray(points, np.int16).astype(f32)
    v = (p + np.asarray(u, f32)).astype(f32)
    v = (v / f32(2.0 ** level)).astype(f32)
    return ((v * f32(2.0)).astype(f32) - f32(1.0)).astype(f32)


def prune_update(density, occupancy, decay, min_density):
    """-> (occupancy fp32, keep bool): torch.stack([density, occupancy * decay], -1).max(-1)[0] (NaN from either side
    propagates), keep = occupancy > min_density."""
    d = np.asarray(density, f32)
    od = (np.asarray(occupancy, f32) * f32(decay)).astype(f32)
    occ = np.maximum(d, od)                                            # np.maximum propagates NaN, like torch.max
    return occ, occ > f32(min_density)
