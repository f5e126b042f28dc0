"""fp16-faithful interval reference of the precision-1 (tensor-core) decoders (TEST INFRASTRUCTURE, NOT PRODUCT CODE).

numpy float64.  For one decoder configuration it rounds to fp16 exactly where wb_shade_tc.cu rounds and returns, for every
output, a centre and a radius: any kernel that rounds at those points and accumulates in fp32, in whatever order, lands in
centre +- radius.  Intervals are carried as (lo, hi) through roundings / relu and as (centre, radius) through linear layers.

Rounding points (wb_shade_tc.cu):
  forward   weights and biases fp16 (wb_tc_pack_kernel); the bias seeds the fp32 accumulator; each layer is an fp32 sum of exact
            fp16 products; a hidden layer stores fp16_rn(relu(acc)); the density head df stays fp32, sigma = max(df[0], 0); the
            colour input is fp16(df[1:dout]) then the per-ray fp16 view embedding (wb_ray_embed_kernel), zero padded; the colour
            head c3 stays fp32 and rgb = 1 / (1 + expf(-c3)) in fp32.
  backward  dY_last = fp16(go * s * (1 - s) * scale); weight gradients sum dY^T [X | 1] in fp32 and are unscaled in fp32 (exact:
            the scale is a power of two); dX = dY . W16 in fp32; a hidden layer's dY_prev = fp16(dX) masked by the retained fp16
            activation > 0; the first colour layer gives gdf[0] = go.w * scale if df[0] > 0 else 0 and gdf[j] = dX[j - 1] for
            j < dout, stored fp16; dL/dfeat = fp16 of the first planes * F columns of dX_0, still loss-scaled.

Accumulation error.  The PTX ISA specifies wgmma.mma_async ... .f32.f16.f16 as D = A * B + D with fp32 accumulators but
leaves the order and the rounding of the internal fp32 additions unspecified; the fp16 x fp16 products are exact in fp32 (22
significant bits).  The reference therefore assumes only that each term enters through an fp32 addition whose relative error
is at most 2^-23 (one ulp: truncation as well as round-to-nearest), in any order, and bounds a sum of n terms by
gamma(n) * sum|terms| with gamma(n) = n u / (1 - n u), u = 2^-23 (Higham, Accuracy and Stability of Numerical Algorithms, 2nd
ed., section 4.2).  For the weight-gradient sums n is the height of the real summation tree: a 64-sample chain, then the
group's sequential sum over its tiles, then the groups of a CTA, then the atomics across CTAs (wgrad_height).
tests/test_gpu_parity.py::test_wgmma_operand_layouts measures max|err| / sum|terms| of wgmma on the H100 against GAMMA_U.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import List, Optional, Sequence

import numpy as np

GAMMA_U = 2.0 ** -23          # per-addition relative error of the fp32 accumulation (see above)
SIGMOID_REL = 6e-7            # relative error of 1 / (1 + expf(-x)) in fp32: expf <= 2 ulp, add and divide 0.5 ulp each
PRODUCT_REL = 4 * 2.0 ** -24  # go * s * (1 - s) * scale in fp32: three roundings (the scale is a power of two)


def gamma(n, u: float = GAMMA_U):
    n = np.asarray(n, dtype=np.float64)
    return n * u / (1.0 - n * u)


def f16(x):
    """Round to fp16, nearest-even (numpy converts float64 -> float16 with one correct rounding); monotone."""
    return np.asarray(x, dtype=np.float64).astype(np.float16).astype(np.float64)


def wgrad_height(S: int, ctas: Optional[int] = None, groups: int = 2) -> int:
    """Height of the summation tree of one weight-gradient entry over S samples: 64-sample wgmma chain + the group's tiles + the
    groups of a CTA + one atomic per CTA.  ctas = None: every tile could be its own CTA (a bound for any grid)."""
    ntiles = max(1, -(-S // 64))
    if ctas is None:
        return 64 + ntiles + groups + 1
    grid = max(1, min(ctas, -(-ntiles // groups)))
    per_group = -(-ntiles // (grid * groups))
    return 64 + per_group + groups + grid


@dataclass
class Decoders:
    """Parameters in nn.Linear layout (fp32): W [out, in], b [out] or None."""
    dens_W: List[np.ndarray]
    dens_b: Optional[List[np.ndarray]]
    col_W: List[np.ndarray]
    col_b: Optional[List[np.ndarray]]

    @property
    def dout(self) -> int:
        return self.dens_W[-1].shape[0]

    def flat(self):
        """Packed parameter vectors [W0, b0?, W1, b1?, ...] of the two decoders (include/wispb200.h order)."""
        def pack(Ws, bs):
            parts = []
            for i, w in enumerate(Ws):
                parts.append(np.asarray(w, np.float32).reshape(-1))
                if bs is not None:
                    parts.append(np.asarray(bs[i], np.float32).reshape(-1))
            return np.concatenate(parts).astype(np.float32)
        return pack(self.dens_W, self.dens_b), pack(self.col_W, self.col_b)


def view_embedding(dirs: np.ndarray, mode: int, freq: int, exact: bool = False):
    """Per-sample colour-input embedding of wb_ray_embed_kernel as an fp16 interval (lo, hi) [S, view_dim].  The direction itself is
    fp16_rn of an fp32 value (exact); sin / cos come from fp32 sinf / cosf (a few ulp of fp32, on an exact argument x * 2^f) and
    may round to either fp16 neighbour near a midpoint.  exact=True: float64 values, no rounding (algebra checks)."""
    d = np.asarray(dirs, np.float32).astype(np.float64)
    parts_lo, parts_hi = [], []
    if mode in (1, 3):
        v = d if exact else f16(d)
        parts_lo.append(v); parts_hi.append(v)
    if mode >= 2:
        w = np.concatenate([d * 2.0 ** f for f in range(freq)], axis=1)       # [S, 3 * freq]: band f, axis c at 3 f + c
        for fn in (np.sin, np.cos):
            v = fn(w)
            if exact:
                parts_lo.append(v); parts_hi.append(v)
            else:
                parts_lo.append(f16(v - 2e-7)); parts_hi.append(f16(v + 2e-7))
    if not parts_lo:
        z = np.zeros((d.shape[0], 0))
        return z, z
    return np.concatenate(parts_lo, axis=1), np.concatenate(parts_hi, axis=1)


def position_embedding(x: np.ndarray, mode: int, freq: int) -> np.ndarray:
    """float64 embedding of the sample positions (positional_embedder.py:51-66), [S, pos_dim]."""
    x = np.asarray(x, np.float64)
    parts = []
    if mode in (1, 3):
        parts.append(x)
    if mode >= 2:
        w = np.concatenate([x * 2.0 ** f for f in range(freq)], axis=1)
        parts += [np.sin(w), np.cos(w)]
    return np.concatenate(parts, axis=1) if parts else np.zeros((x.shape[0], 0))


class Reference:
    """Interval evaluation of both decoders for S samples.

    X0: [S, I0] density-decoder input rows (fp16 values); view: (lo, hi) [S, view_dim] from view_embedding.
    rounding=False and accumulation=False turn every fp16 rounding and every gamma off: the radius is then 0 and the result is
    the float64 MLP (what the CPU tests compare with torch autograd)."""

    def __init__(self, dec: Decoders, X0, view, rounding: bool = True, accumulation: bool = True):
        self.dec, self.rounding, self.acc = dec, rounding, accumulation
        q = f16 if rounding else (lambda a: np.asarray(a, np.float64))
        self.q = q
        self.dW = [q(w) for w in dec.dens_W]
        self.cW = [q(w) for w in dec.col_W]
        self.db = [q(b) for b in dec.dens_b] if dec.dens_b is not None else None
        self.cb = [q(b) for b in dec.col_b] if dec.col_b is not None else None
        X0 = np.asarray(X0, np.float64)
        self.S = X0.shape[0]
        self._forward(X0, view)

    # ---- interval helpers -----------------------------------------------------------------------------------------
    def _round(self, lo, hi):
        return (f16(lo), f16(hi)) if self.rounding else (lo, hi)

    def _linear(self, lo, hi, W, b):
        """fp32 accumulation of [x | 1] . [W | b]^T over Kp (+ bias) terms -> (lo, hi) of the accumulator."""
        c, r = (lo + hi) * 0.5, (hi - lo) * 0.5
        Wa = np.abs(W)
        cc = c @ W.T + (b if b is not None else 0.0)
        rr = r @ Wa.T
        if self.acc:
            n = -(-W.shape[1] // 16) * 16 + (1 if b is not None else 0)
            rr = rr + gamma(n) * ((np.abs(c) + r) @ Wa.T + (np.abs(b) if b is not None else 0.0))
        return cc - rr, cc + rr

    def _relu_round(self, lo, hi):
        return self._round(np.maximum(lo, 0.0), np.maximum(hi, 0.0))

    # ---- forward ----------------------------------------------------------------------------------------------------
    def _forward(self, X0, view):
        nd, nc = len(self.dW), len(self.cW)
        lo, hi = X0, X0
        self.xd = []                                   # input interval of every density layer
        for l in range(nd):
            self.xd.append((lo, hi))
            lo, hi = self._linear(lo, hi, self.dW[l], self.db[l] if self.db else None)
            if l < nd - 1:
                lo, hi = self._relu_round(lo, hi)
        self.df = (lo, hi)                             # density head, fp32
        dout = self.dec.dout
        flo, fhi = self._round(lo[:, 1:dout], hi[:, 1:dout])
        lo = np.concatenate([flo, view[0]], axis=1)
        hi = np.concatenate([fhi, view[1]], axis=1)
        self.xc = []
        for l in range(nc):
            self.xc.append((lo, hi))
            lo, hi = self._linear(lo, hi, self.cW[l], self.cb[l] if self.cb else None)
            if l < nc - 1:
                lo, hi = self._relu_round(lo, hi)
        self.c3 = (lo, hi)
        s_lo, s_hi = 1.0 / (1.0 + np.exp(-lo)), 1.0 / (1.0 + np.exp(-hi))
        if self.rounding:
            s_lo, s_hi = s_lo * (1.0 - SIGMOID_REL), s_hi * (1.0 + SIGMOID_REL)
        self.rgb = (s_lo, s_hi)
        self.sigma = (np.maximum(self.df[0][:, 0], 0.0), np.maximum(self.df[1][:, 0], 0.0))

    # ---- backward ---------------------------------------------------------------------------------------------------
    def backward(self, g_shaded, scale: float, planes: int, width: int, wgrad_n: Optional[int] = None):
        """g_shaded [S, 4] fp32, scale: the power-of-two loss scale.  -> dict of (centre, radius): 'dens', 'col' (packed gradient
        vectors, unscaled) and 'dfeat' [planes, S, width] (loss-scaled fp16 values).  wgrad_n: height of the weight-gradient sums
        (wgrad_height); default: a bound for any grid."""
        go = np.asarray(g_shaded, np.float32).astype(np.float64)
        S = self.S
        n_w = wgrad_height(S) if wgrad_n is None else wgrad_n
        dout = self.dec.dout
        # ---- last colour layer: dY = go * s (1 - s) * scale ----
        s_lo, s_hi = self.rgb
        q_a, q_b = s_lo * (1 - s_lo), s_hi * (1 - s_hi)
        q_lo, q_hi = np.minimum(q_a, q_b), np.maximum(q_a, q_b)
        q_hi = np.where((s_lo <= 0.5) & (s_hi >= 0.5), 0.25, q_hi)
        g3 = go[:, :3] * scale
        a, b = g3 * q_lo, g3 * q_hi
        lo, hi = np.minimum(a, b), np.maximum(a, b)
        if self.rounding:
            lo, hi = lo - np.abs(lo) * PRODUCT_REL, hi + np.abs(hi) * PRODUCT_REL
        dy = self._round(lo, hi)
        grads_c, grads_d = [None] * len(self.cW), [None] * len(self.dW)
        layers = [("c", l) for l in range(len(self.cW))][::-1] + [("d", l) for l in range(len(self.dW))][::-1]
        out = {}
        for kind, l in layers:
            W = self.cW[l] if kind == "c" else self.dW[l]
            x = self.xc[l] if kind == "c" else self.xd[l]
            has_b = (self.cb if kind == "c" else self.db) is not None
            g = self._wgrad(dy, x, has_b, n_w, scale)
            (grads_c if kind == "c" else grads_d)[l] = g
            # data gradient dX = dY . W16 over the Np outputs
            dxl, dxh = self._linear(dy[0], dy[1], W.T, None)
            if kind == "c" and l == 0:
                # first colour layer: gdf[0] from relu'(density), gdf[1:dout] = dX[:dout-1]
                gw = go[:, 3] * scale
                df_lo, df_hi = self.df[0][:, 0], self.df[1][:, 0]
                g0_lo = np.where(df_lo > 0, gw, np.where(df_hi > 0, np.minimum(gw, 0), 0.0))
                g0_hi = np.where(df_lo > 0, gw, np.where(df_hi > 0, np.maximum(gw, 0), 0.0))
                lo = np.concatenate([g0_lo[:, None], dxl[:, :dout - 1]], axis=1)
                hi = np.concatenate([g0_hi[:, None], dxh[:, :dout - 1]], axis=1)
                dy = self._round(lo, hi)
            elif kind == "d" and l == 0:
                lo, hi = self._round(dxl[:, :planes * width], dxh[:, :planes * width])
                c, r = (lo + hi) * 0.5, (hi - lo) * 0.5
                out["dfeat"] = (c.reshape(S, planes, width).transpose(1, 0, 2), r.reshape(S, planes, width).transpose(1, 0, 2))
            else:
                # hidden layer: relu' of the retained fp16 activation (= this layer's input); an activation interval that reaches 0
                # gives the hull of 0 and the value
                alo, ahi = x
                lo, hi = self._round(dxl, dxh)
                on, maybe = alo > 0, ahi > 0
                dy = (np.where(on, lo, np.where(maybe, np.minimum(lo, 0), 0.0)), np.where(on, hi, np.where(maybe, np.maximum(hi, 0), 0.0)))
        out["dens"] = self._pack(grads_d)
        out["col"] = self._pack(grads_c)
        return out

    def _wgrad(self, dy, x, has_b, n, scale):
        """sum over samples of dY^T [X | 1], unscaled: (centre, radius) of [O, I] and [O] (bias or None)."""
        (yl, yh), (xl, xh) = dy, x
        cy, ry, cx, rx = (yl + yh) * 0.5, (yh - yl) * 0.5, (xl + xh) * 0.5, (xh - xl) * 0.5
        ay, ax = np.abs(cy), np.abs(cx)
        C = cy.T @ cx
        R = ay.T @ rx + ry.T @ ax + ry.T @ rx
        if self.acc:
            R = R + gamma(n) * ((ay + ry).T @ (ax + rx))
        out = [(C / scale, R / scale)]
        if has_b:
            Cb, Rb = cy.sum(0), ry.sum(0)
            if self.acc:
                Rb = Rb + gamma(n) * (ay + ry).sum(0)
            out.append((Cb / scale, Rb / scale))
        return out

    @staticmethod
    def _pack(grads):
        cs, rs = [], []
        for g in grads:
            for c, r in g:
                cs.append(c.reshape(-1)); rs.append(r.reshape(-1))
        return np.concatenate(cs), np.concatenate(rs)

    # ---- outputs ----------------------------------------------------------------------------------------------------
    def shaded(self):
        """(centre, radius) [S, 4] of (r, g, b, sigma)."""
        lo = np.concatenate([self.rgb[0], self.sigma[0][:, None]], axis=1)
        hi = np.concatenate([self.rgb[1], self.sigma[1][:, None]], axis=1)
        return (lo + hi) * 0.5, (hi - lo) * 0.5


def table_scatter_bound(dfeat, scale: float, coords, n_rows: int, resolutions: Sequence[int], codebook_bitwidth: int, lod_idx: int,
                        multiscale: str = "cat"):
    """Reference of the table scatter of dL/dfeat planes (fp16, loss-scaled) [planes, S, F] -> (centre, radius) [rows, F].

    The kernels form corner products dfeat * w in fp16 and sum runs of lanes that share a cell with a warp scan of at most 5
    fp16 additions (wb_table_scatter_kernel / tc_scatter_level_f2), so every entry is off by at most one fp16 rounding per
    scan step plus the product rounding (6 * 2^-11 relative, 6 half-ulps of the smallest subnormal absolute, per term), then
    summed in fp32 by atomics.  The corner weights are non-negative: the scatter of |dfeat| is sum |terms| per entry."""
    from oracle import oracle as O
    P, S, F = dfeat.shape
    L = len(resolutions)
    g = np.zeros((S, L * F), np.float32)
    if multiscale == "cat":
        for p in range(P):
            g[:, p * F:(p + 1) * F] = dfeat[p] / scale
    else:
        for l in range(L):
            g[:, l * F:(l + 1) * F] = dfeat[0] / scale
    centre = O.hashgrid_bwd(coords, g, n_rows, resolutions, codebook_bitwidth).astype(np.float64)
    mag = O.hashgrid_bwd(coords, np.abs(g), n_rows, resolutions, codebook_bitwidth).astype(np.float64)
    # terms per entry (subnormal fp16 products / partial sums carry an absolute error instead of a relative one)
    _, corners = O.hashgrid_fwd(coords, np.zeros((n_rows, F), np.float32), resolutions, codebook_bitwidth, return_corners=True)
    begin = O.table_layout(resolutions, codebook_bitwidth)
    live = np.abs(g).reshape(S, L, F).max(axis=2) > 0                              # [S, L]
    rows = (corners.astype(np.int64) + begin[:L][None, :, None])[live]             # [n, 8]
    cnt = np.bincount(rows.reshape(-1), minlength=n_rows).astype(np.float64)[:, None]
    radius = mag * (6 * 2.0 ** -11 + 1e-5) + cnt * 6 * 2.0 ** -25 / scale
    return centre, radius
