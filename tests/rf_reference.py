"""float64 interval reference of the NeRF shade stage over TriplanarGrid, OctreeGrid and HashGrid (TEST INFRASTRUCTURE, NOT
PRODUCT CODE).

Every function returns, per output, a centre and a radius: a kernel that rounds where wb_featx.cuh, wb_triplane.cu, wb_shade.cu
and wb_featx_scatter_kernel (wb_shade_tc.cu) round, and sums in fp32 in any order where they sum in an unspecified order, lands in
centre +- radius.  It builds on oracle/sdf_reference.py (fma32, fma_step, round_radius, g32, cells, features, _scatter, _linear,
_embed) and oracle/tc_decoders.py (f16, gamma, Reference).

Rounding points
  triplanar  wb_tp_coord / wb_reflect / wb_tp_setup are emulated bit-exactly in fp32: unnormalize ((c + 1) * 0.5) * (size - 1),
             |x|, fmodf (exact), floorf(|x| / span) of the IEEE quotient, span - extra on odd flips, the clip, floorf, the four
             weights (1 - tx) * (1 - ty), ... and the in-bounds flags bx1 / by1.  The four-term blend may be contracted into fmas by
             nvcc, so it is bounded, not emulated: gamma(4) * sum|terms|; a 'sum' grid adds its LODs in order on top, one rounding
             per LOD: gamma(3 + nl).  Plane pairing: x <- (y, z), y <- (x, z), z <- (x, y).
  octree     sdf_reference.cells / features on a Field built from the NeRF grid: the same descent (base_lod, LODs past an
             unoccupied cell and points outside the cube give zeros), the same fma chain over the corners and the same fp16
             roundings (half_round), bit-exact; 'sum' over a single LOD is that LOD.
  hash       oracle.hashgrid_fwd (an fp32 restatement) as the centre; the kernel and the restatement are each within
             gamma(8) * sum|terms| of the exact blend, a 'sum' grid adds one rounding per LOD.
  scatters   one fp32 product fl(g * w) per texel / corner (precision 1: g = fl(h * inv_scale) of the fp16 dL/dfeat plane, exact:
             the scale is a power of two), added by atomics in any order, after at most 5 levels of the segmented warp scan at
             precision 1: gamma(n_terms + levels) * sum|terms| per entry, plus the propagated radius of g.  dL/dfeat feature f lives
             in plane f / width at column f % width (tc_dfeat_shape).
  decoders   (precision 0, wb_shade.cu) wb_layer_fwd: per unit an fp32 fma chain seeded with the bias over the inputs in
             ascending order, emulated on the centres (sdf_reference._chain); sinf / cosf of the view embedding within 2 ulp;
             rgb = 1 / (1 + expf(-c)) within tc_decoders.SIGMOID_REL; sigma = max(df0, 0).  Backward: gout = (go * r) * (1 - r)
             (three roundings), wb_dgrad's chain over the outputs in ascending order, emulated; relu' from the retained
             activation (the hull of 0 and the value where the activation interval reaches 0); the density head
             gin[0] = df0 > 0 ? go.w : 0.  wb_wgrad sums NT samples per tile in one fma chain per thread and adds every tile's
             partial by one atomic: height NT + ntiles - 1 (all tiles of all CTAs reach the same address); its bias gradient sums
             NT / 32 samples per lane, the 5-level warp butterfly, then the atomics: height NT / 32 + 5 + ntiles - 1.  NT mirrors
             wb_shade_{fwd,bwd}_launch's shared-memory rule (shade0_plan).
             Precision 1 over triplanar / octree grids feeds the X0 rows into tc_decoders.Reference.

exact=True turns every rounding and every gamma off: the result is then the float64 operation (what the CPU tests compare with
torch).  Accumulation bounds follow Higham, Accuracy and Stability of Numerical Algorithms, 2nd ed., section 4.2.
"""
from __future__ import annotations

from dataclasses import dataclass
from types import SimpleNamespace
from typing import List, Optional, Sequence

import numpy as np

from oracle import oracle as O
from oracle import sdf_reference as S
from oracle import tc_decoders as T
from oracle.sdf_reference import U, fma32, g32

f32 = np.float32
SCAN_LEVELS = 5                     # segmented warp scan of the precision-1 merged scatter (tc_warp_runs: dist <= 31)
SMEM_MAX = 227 * 1024               # wb_shade_{fwd,bwd}_launch
SMEM_RESERVED = 1024


def positions(origins, dirs, rec_ray, rec_t):
    """Sample positions as the kernels form them: fmaf(dir, t, origin) in fp32."""
    o = np.asarray(origins, f32)[rec_ray].astype(np.float64)
    d = np.asarray(dirs, f32)[rec_ray].astype(np.float64)
    return fma32(d, np.asarray(rec_t, f32).astype(np.float64)[:, None], o).astype(f32)


# ---- triplanar ----------------------------------------------------------------------------------------------------------
def tp_coord(c, size: int, exact: bool = False):
    """wb_tp_coord: grid_sampler_unnormalize (align_corners=True), reflect_coordinates(in, 0, 2 span), clip_coordinates."""
    t = np.float64 if exact else f32
    c = np.asarray(c, t)
    span = t(size - 1)
    x = ((c + t(1)) * t(0.5)) * span
    a = np.abs(x)
    extra = np.fmod(a, span)
    flips = np.floor(a / span).astype(np.int64)
    x = np.where(flips & 1, span - extra, extra).astype(t)
    return np.minimum(span, np.maximum(x, t(0)))


@dataclass
class Bilinear:
    idx: np.ndarray                 # [N, 4] texel offsets y * size + x of nw, ne, sw, se (out-of-range neighbours: the nw texel)
    w: np.ndarray                   # [N, 4] weights (0 for out-of-range neighbours), float64 holding the kernel's fp32 values


def tp_setup(coords, p: int, size: int, exact: bool = False) -> Bilinear:
    """wb_tp_setup of plane p: x-plane <- (y, z), y-plane <- (x, z), z-plane <- (x, y); grid x -> W, grid y -> H."""
    t = np.float64 if exact else f32
    c = np.asarray(coords, t)
    gx = c[:, 1] if p == 0 else c[:, 0]
    gy = c[:, 1] if p == 2 else c[:, 2]
    ix, iy = tp_coord(gx, size, exact), tp_coord(gy, size, exact)
    fx, fy = np.floor(ix), np.floor(iy)
    x0, y0 = fx.astype(np.int64), fy.astype(np.int64)
    tx, ty = ix - fx, iy - fy
    one = t(1)
    w = np.stack([(one - tx) * (one - ty), tx * (one - ty), (one - tx) * ty, tx * ty], 1).astype(np.float64)
    bx1, by1 = x0 + 1 < size, y0 + 1 < size
    o00 = y0 * size + x0
    idx = np.stack([o00, o00 + 1, o00 + size, o00 + size + 1], 1)
    live = np.stack([np.ones_like(bx1), bx1, by1, bx1 & by1], 1)
    return Bilinear(np.where(live, idx, o00[:, None]), np.where(live, w, 0.0))


@dataclass
class Triplanar:
    """TriplanarGrid: planes[l][p] = [C, size_l, size_l] (fmx, fmy, fmz of LOD l); nl LODs used."""
    planes: List[List[np.ndarray]]
    multiscale: str
    nl: int

    @property
    def C(self):
        return self.planes[0][0].shape[0]

    def feat_dim(self):
        return 3 * self.C * (self.nl if self.multiscale == "cat" else 1)

    def col(self, l, p, c):
        return (p * self.C + c) if self.multiscale == "sum" else ((l * 3 + p) * self.C + c)


def triplanar_features(tp: Triplanar, coords, exact: bool = False):
    """TriplanarGrid.interpolate over LODs 0..nl-1 -> (centre, radius) [N, feat_dim]."""
    N, C = coords.shape[0], tp.C
    cen, mag = np.zeros((N, tp.feat_dim())), np.zeros((N, tp.feat_dim()))
    for l in range(tp.nl):
        size = tp.planes[l][0].shape[-1]
        for p in range(3):
            b = tp_setup(coords, p, size, exact)
            pl = tp.planes[l][p].reshape(C, -1).astype(np.float64)
            for c in range(C):
                terms = pl[c][b.idx] * b.w
                f = tp.col(l, p, c)
                cen[:, f] += terms.sum(1)
                mag[:, f] += np.abs(terms).sum(1)
    if exact:
        return cen, np.zeros_like(cen)
    return cen, g32(4 if tp.multiscale == "cat" else 3 + tp.nl) * mag


def triplanar_scatter(tp: Triplanar, coords, gc, gr, levels: int = 0, exact: bool = False):
    """d sum(g * feats) / d plane, one fp32 product per texel and an atomic each (levels: scan levels before the atomics)
    -> [[(centre, radius) [C, size, size] per plane] per LOD]."""
    C = tp.C
    gc, gr = np.asarray(gc, np.float64), np.asarray(gr, np.float64)
    out = []
    for l in range(tp.nl):
        size = tp.planes[l][0].shape[-1]
        hw = size * size
        row = []
        for p in range(3):
            b = tp_setup(coords, p, size, exact)
            cen, rad, mag = np.zeros((C, hw)), np.zeros((C, hw)), np.zeros((C, hw))
            n = np.bincount(b.idx[b.w > 0], minlength=hw).astype(np.float64)
            for c in range(C):
                f = tp.col(l, p, c)
                g, r = gc[:, f:f + 1], gr[:, f:f + 1]
                cen[c] = np.bincount(b.idx.reshape(-1), (g * b.w).reshape(-1), hw)
                rad[c] = np.bincount(b.idx.reshape(-1), (r * b.w).reshape(-1), hw)
                mag[c] = np.bincount(b.idx.reshape(-1), ((np.abs(g) + r) * b.w).reshape(-1), hw)
            if not exact:
                rad = rad + g32(n + levels)[None, :] * mag
            row.append((cen.reshape(C, size, size), rad.reshape(C, size, size)))
        out.append(row)
    return out


# ---- octree -------------------------------------------------------------------------------------------------------------
def octree_field(spc, trinkets, feats, base_lod: int, multiscale: str, half: bool) -> S.Field:
    """The NeRF OctreeGrid as a sdf_reference.Field (feature levels base_lod .., no decoder)."""
    return S.Field(spc, trinkets, list(feats), base_lod, multiscale, [], [], 0, 0, half)


def octree_features(field: S.Field, coords, nl: int, exact: bool = False):
    """OctreeGrid.interpolate over LODs 0..nl-1 -> (centre, radius [0: bit-exact], cells)."""
    c, r, _, cl = S.features(field, np.asarray(coords, f32), nl, exact)
    return c, r, cl


def octree_scatter(field: S.Field, cl: S.Cells, nl: int, gc, gr, levels: int = 0, exact: bool = False):
    """d sum(g * feats) / d feature level -> [(centre, radius) [rows, F]] per LOD."""
    sc = S._scatter(field, np.asarray(gc, np.float64), np.asarray(gr, np.float64), cl, nl, field.multiscale == "sum" and nl > 1, not exact)
    return [(C_, R if exact else R + g32(n + levels)[:, None] * A) for C_, R, A, n in sc]


# ---- hash grid (precision 0 features) -----------------------------------------------------------------------------------
def hash_features(coords, table, resolutions, bw: int, multiscale: str, lod_idx: int):
    """HashGrid.interpolate as wb_gather computes it -> (centre, radius) [N, feat_dim]."""
    L, F = len(resolutions), table.shape[1]
    raw = O.hashgrid_fwd(coords, table, resolutions, bw).reshape(-1, L, F).astype(np.float64)
    mag = O.hashgrid_fwd(coords, np.abs(table), resolutions, bw).reshape(-1, L, F).astype(np.float64) * (1 + 1e-6)
    if multiscale == "cat":
        raw[:, lod_idx:] = 0.0; mag[:, lod_idx:] = 0.0
        return raw.reshape(raw.shape[0], -1), 2 * g32(8) * mag.reshape(mag.shape[0], -1)
    return raw.sum(1), 2 * g32(8 + L) * mag.sum(1)


# ---- precision-0 decoders -------------------------------------------------------------------------------------------------
def _r8(v):
    return -(-v // 8) * 8


@dataclass
class Plan:
    nt_fwd: int
    nt_bwd: int
    per_sm: int                     # backward CTAs per SM

    def ctas(self, S_: int, sms: int) -> int:
        return max(1, min(sms * self.per_sm, -(-S_ // self.nt_bwd)))

    def tiles_per_cta(self, S_: int, sms: int) -> int:
        return -(-max(1, -(-S_ // self.nt_bwd)) // self.ctas(S_, sms))


def shade0_plan(dens_dims: Sequence[int], col_dims: Sequence[int]) -> Optional[Plan]:
    """Tile sizes of wb_shade_fwd_launch / wb_shade_bwd_launch and the backward's CTAs per SM (wb_make_mlp's layout); None: the
    decoder does not fit."""
    dims = [(i, o) for i, o in zip(dens_dims[:-1], dens_dims[1:])] + [(i, o) for i, o in zip(col_dims[:-1], col_dims[1:])]
    nd = len(dens_dims) - 1
    fwd = -(-sum(i * _r8(o) + _r8(o) for i, o in dims) // 4) * 4
    maxw = max(max(_r8(i), _r8(o)) for i, o in dims)
    cols = sum(_r8(o) for _, o in dims) + _r8(dims[0][0]) + _r8(dims[nd][0])
    nt_f = next((nt for nt in (128, 64, 32) if (fwd + 2 * maxw * (nt + 1)) * 4 <= SMEM_MAX), None)
    nt_b = next((nt for nt in (128, 64, 32) if (cols + 2 * maxw) * (nt + 1) * 4 <= SMEM_MAX), None)
    if nt_f is None or nt_b is None:
        return None
    smem = (cols + 2 * maxw) * (nt_b + 1) * 4
    return Plan(nt_f, nt_b, min(8, max(1, SMEM_MAX // (smem + SMEM_RESERVED))))


def _hull(c, r, on, maybe):
    """relu' applied to (c, r): kept where on, the hull of 0 and the interval where maybe, 0 elsewhere."""
    lo, hi = np.minimum(c - r, 0.0), np.maximum(c + r, 0.0)
    return np.where(on, c, np.where(maybe, (lo + hi) * 0.5, 0.0)), np.where(on, r, np.where(maybe, (hi - lo) * 0.5, 0.0))


def _relu(c, r):
    lo, hi = np.maximum(c - r, 0.0), np.maximum(c + r, 0.0)
    return np.where(c - r >= 0, c, (lo + hi) * 0.5), np.where(c - r >= 0, r, (hi - lo) * 0.5)


class Shade0:
    """wb_rf_shade_fwd / wb_rf_shade_bwd at precision 0 for S samples.  x0: (centre, radius) [S, I0] of the density-decoder input
    (grid features, then the position embedding); dirs: [S, 3] fp32 ray directions of the samples."""

    def __init__(self, dec: T.Decoders, x0c, x0r, dirs, view_mode: int, view_freq: int, exact: bool = False, in_order: bool = True):
        self.dec, self.exact, self.in_order = dec, exact, in_order
        z = lambda Ws, bs, l: np.zeros(Ws[l].shape[0]) if bs is None else bs[l]
        self.layers = [(W, z(dec.dens_W, dec.dens_b, l)) for l, W in enumerate(dec.dens_W)] + \
                      [(W, z(dec.col_W, dec.col_b, l)) for l, W in enumerate(dec.col_W)]
        self.nd = len(dec.dens_W)
        self.ins = []                                   # (centre, radius) input of every layer
        h = (np.asarray(x0c, np.float64), np.asarray(x0r, np.float64))
        ve = S._embed(SimpleNamespace(pos_mode=view_mode, pos_freq=view_freq), np.asarray(dirs, f32).astype(np.float64), exact)
        nl = len(self.layers)
        for l, (W, b) in enumerate(self.layers):
            if l == self.nd:
                self.df = h
                h = (np.concatenate([h[0][:, 1:], ve[0]], 1), np.concatenate([h[1][:, 1:], ve[1]], 1))
            self.ins.append(h)
            a = S._linear(h[0], h[1], W, b, exact, in_order)
            h = a if l in (self.nd - 1, nl - 1) else _relu(*a)
        c3c, c3r = h
        s_lo, s_hi = 1.0 / (1.0 + np.exp(-(c3c - c3r))), 1.0 / (1.0 + np.exp(-(c3c + c3r)))
        if not exact:
            s_lo, s_hi = s_lo * (1 - T.SIGMOID_REL), s_hi * (1 + T.SIGMOID_REL)
        self.rgb = (s_lo, s_hi)
        d0c, d0r = self.df[0][:, 0], self.df[1][:, 0]
        self.sig = _relu(d0c, d0r)

    def shaded(self):
        """(centre, radius) [S, 4] of (r, g, b, sigma)."""
        c = np.concatenate([(self.rgb[0] + self.rgb[1]) * 0.5, self.sig[0][:, None]], 1)
        r = np.concatenate([(self.rgb[1] - self.rgb[0]) * 0.5, self.sig[1][:, None]], 1)
        return c, r

    def _wgrad(self, gc, gr, xc, xr, h_w, h_b):
        C_ = gc.T @ xc
        R = np.abs(gc).T @ xr + gr.T @ np.abs(xc) + gr.T @ xr
        Cb, Rb = gc.sum(0), gr.sum(0)
        if not self.exact:
            R = R + g32(h_w) * ((np.abs(gc) + gr).T @ (np.abs(xc) + xr))
            Rb = Rb + g32(h_b) * (np.abs(gc) + gr).sum(0)
        return (C_, R), (Cb, Rb)

    def backward(self, g_shaded, nt: int = 128, ntiles: int = 1):
        """g_shaded [S, 4] -> dict of (centre, radius): 'dens', 'col' (packed like Decoders.flat) and 'dx0' [S, I0]."""
        go = np.asarray(g_shaded, f32).astype(np.float64)
        exact = self.exact
        s_lo, s_hi = self.rgb
        q_a, q_b = s_lo * (1 - s_lo), s_hi * (1 - s_hi)
        q_lo, q_hi = np.minimum(q_a, q_b), np.where((s_lo <= 0.5) & (s_hi >= 0.5), 0.25, np.maximum(q_a, q_b))
        a, b = go[:, :3] * q_lo, go[:, :3] * q_hi
        lo, hi = np.minimum(a, b), np.maximum(a, b)
        if not exact:                                   # (go * r) * (1 - r): three roundings
            lo, hi = lo - np.abs(lo) * 4 * U, hi + np.abs(hi) * 4 * U
        gc, gr = (lo + hi) * 0.5, (hi - lo) * 0.5
        h_w, h_b = nt + ntiles - 1, nt // 32 + 5 + ntiles - 1
        grads = [None] * len(self.layers)
        for l in range(len(self.layers) - 1, -1, -1):
            W, bias = self.layers[l]
            xc, xr = self.ins[l]
            grads[l] = self._wgrad(gc, gr, xc, xr, h_w, h_b)
            nc, nr = S._linear(gc, gr, W.T, np.zeros(W.shape[1]), exact, self.in_order)      # wb_dgrad: chain over o ascending
            if l == self.nd:                            # colour input -> density head
                d0c, d0r = self.df[0][:, 0], self.df[1][:, 0]
                on, maybe = d0c - d0r > 0, d0c + d0r > 0
                h0c, h0r = _hull(go[:, 3], np.zeros_like(d0c), on, maybe)
                dout = self.df[0].shape[1]
                nc = np.concatenate([h0c[:, None], nc[:, :dout - 1]], 1)
                nr = np.concatenate([h0r[:, None], nr[:, :dout - 1]], 1)
            elif l > 0:                                 # relu' of the retained hidden activation (this layer's input)
                on, maybe = xc - xr > 0, xc + xr > 0
                nc, nr = _hull(nc, nr, on, maybe)
            gc, gr = nc, nr
        out = {"dx0": (gc, gr)}
        for key, ls in (("dens", range(self.nd)), ("col", range(self.nd, len(self.layers)))):
            has_b = (self.dec.dens_b if key == "dens" else self.dec.col_b) is not None
            cs, rs = [], []
            for l in ls:
                (wc, wr), (bc, br) = grads[l]
                cs.append(wc.reshape(-1)); rs.append(wr.reshape(-1))
                if has_b:
                    cs.append(bc); rs.append(br)
            out[key] = (np.concatenate(cs), np.concatenate(rs))
        return out


def view_dirs(dirs, rec_ray):
    return np.asarray(dirs, f32)[rec_ray]
