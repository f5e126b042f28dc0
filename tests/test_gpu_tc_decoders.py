"""Tensor-core (precision 1) decoder kernels through the C ABI against the fp16-faithful interval reference
(oracle/tc_decoders.py): every output must lie inside centre +- radius, which any kernel that rounds at the same points lands
in whatever order it sums.  Covers what the end-to-end parity tests cannot resolve at their fp32-oracle tolerances: decoder
widths 16..128 and unequal widths, bias on / off, density-head widths 2..16, decoder depths, the view / position embeddings,
the saved X0 rows, the fused and the stand-alone table scatter, the chunked backward of wide decoders, the loss scale, and sample
counts around the 64-sample tile.

Case ids name the kernel instances: fwd64 / fwd128 = the forward kernel's widest padded layer (NMAX), gNpM = the decoder backward
runs N groups per CTA in M passes (bwd_plan mirrors tc_bwd_layout / tc_bwd_passes of wb_shade_tc.cu), +fused = the table
scatter runs in the decoder backward's last epilogue (wb_rf_shade_bwd), otherwise wb_rf_table_scatter runs separately."""
import ctypes as C
from dataclasses import dataclass
from fractions import Fraction
from typing import List

import numpy as np
import pytest
import torch

from oracle import oracle as O
from oracle import tc_decoders as T

pytestmark = pytest.mark.gpu

TOL1_RGB, TOL1_GRAD = 2e-3, 3e-2          # tests/test_gpu_parity.py TOL[1]: what the end-to-end tests resolve


@pytest.fixture(scope="module")
def W():
    import wisp_b200
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return wisp_b200


def embed_dim(mode, freq):
    return 0 if mode == 0 else 3 if mode == 1 else 6 * freq if mode == 2 else 3 + 6 * freq


@dataclass
class Case:
    name: str
    dens_hidden: List[int]
    col_hidden: List[int]
    dout: int = 16
    L: int = 8
    F: int = 2
    multiscale: str = "cat"
    lod_idx: int = -1                      # -1: all LODs live
    pos: tuple = (0, 0)
    view: tuple = (3, 4)
    bias: bool = True
    S: int = 700
    R: int = 40
    backward: bool = True
    seed: int = 0
    bw: int = 12

    def dims(self):
        feat = self.L * self.F if self.multiscale == "cat" else self.F
        dens = [feat + embed_dim(*self.pos)] + list(self.dens_hidden) + [self.dout]
        col = [self.dout - 1 + embed_dim(*self.view)] + list(self.col_hidden) + [3]
        return dens, col


def bwd_plan(case):
    """Groups per CTA of each pass of the decoder backward: mirrors tc_bwd_layout / tc_bwd_passes (wb_shade_tc.cu)."""
    dens, col = case.dims()
    I = dens[:-1] + col[:-1]; O_ = dens[1:] + col[1:]
    r16 = lambda v: -(-v // 16) * 16
    Kp, Np = [r16(i) for i in I], [r16(o) for o in O_]
    maxw = max(max(Kp), max(Np))
    blob = r16(sum(k * n * 2 + n * 32 for k, n in zip(Kp, Np)))
    scr = r16(64 * 33 * 4)

    def fits(mask, groups):
        off = sum((k // 8 + 1) * 1024 for k in Kp) + max(maxw, 64) // 8 * 1024 + scr
        off += r16(4 * sum(O_[l] * (I[l] + 1) for l in range(len(I)) if (mask >> l) & 1))
        return groups * off + blob <= 227 * 1024 - 1024
    masks, cur = [], 0
    for l in range(len(I)):
        if cur and not fits(cur | (1 << l), 1):
            masks.append(cur); cur = 0
        cur |= 1 << l
    masks.append(cur)
    return [2 if fits(m, 2) else 1 for m in masks]


def case_id(c):
    dens, col = c.dims()
    r16 = lambda v: -(-v // 16) * 16
    s = f"{c.name}-fwd{128 if max(r16(v) for v in dens + col) > 64 else 64}"
    if c.backward:
        groups = bwd_plan(c)
        s += f"-g{'/'.join(map(str, groups))}p{len(groups)}" + ("+fused" if fusable(c) else "")
    return s


def fusable(c):
    """wb_rf_shade_bwd fuses the scatter into the last pass of the decoder backward for F == 2 'cat' grids when that pass runs two groups."""
    return c.F == 2 and c.multiscale == "cat" and bwd_plan(c)[-1] == 2


CASES = [
    # widths (uniform), with the embeddings and head widths spread over them
    Case("w16", [16], [16, 16], view=(3, 1), pos=(1, 0), L=8),
    Case("w24_nobias_F4", [24], [24, 24], dout=9, bias=False, view=(1, 0), pos=(2, 2), L=5, F=4),
    Case("w40_sum", [40], [40, 40], dout=2, view=(0, 0), pos=(3, 3), L=6, multiscale="sum"),
    Case("w64_L16", [64], [64, 64], view=(3, 6), L=16, S=1000),
    Case("w80", [80], [80, 80], view=(3, 2), pos=(3, 1), L=12),
    Case("w96", [96], [96, 96], dout=9, view=(3, 5), L=16),
    Case("w112_nobias", [112], [112, 112], bias=False, view=(3, 3), pos=(1, 0), L=10, F=4),
    Case("w128", [128], [128, 128], view=(3, 4), L=16, S=900),
    Case("w128_F8sum", [128], [128, 128], dout=2, view=(1, 0), L=4, F=8, multiscale="sum"),
    # unequal widths, depths: dens_layers 1..2, col_layers 1..3
    Case("unequal", [48], [96, 32], dout=9, view=(3, 2), L=12),
    Case("dens1_col1", [], [], view=(3, 1), pos=(2, 1), L=8),
    Case("dens2_col3", [32, 24], [40, 16], dout=9, view=(3, 2), L=8),
    Case("dens2_col2_F4_lod", [40, 56], [24], view=(1, 0), L=6, F=4, lod_idx=4),
    Case("cat_lod_F2", [32], [32, 32], view=(3, 2), L=12, lod_idx=9),
    # F = 2 'cat' with L % 8 in {5, 6, 7} and a position embedding: the last partial slab shares its bytes with the embedding
    Case("race_L6_pos", [32], [32, 32], L=6, pos=(3, 2), view=(3, 4)),
    Case("race_L13_pos", [64], [64, 64], L=13, pos=(1, 0), view=(3, 4)),
    Case("race_L7_posonly", [32], [32, 32], L=7, pos=(2, 4), view=(0, 0), dout=2),
    # deeper than the tensor-core backward takes: forward only, precision_supported(backward=1) == 0
    Case("deep_fwd_only", [64, 64, 64], [64, 64, 64, 64], view=(3, 4), L=16, backward=False),
]


def _f16ulp(a):
    return np.spacing(np.abs(np.asarray(a, np.float64)).astype(np.float16)).astype(np.float64)


class Setup:
    """Device buffers and the C-ABI calls of one case."""

    def __init__(self, W, c: Case, S=None):
        self.W, self.A, self.c = W, W._cabi, c
        from wisp_b200 import ops
        rng = np.random.default_rng(1000 + c.seed)
        S = c.S if S is None else S
        self.S, self.R = S, c.R
        self.res = O.geometric_resolutions(c.L, 4, 64) if c.L > 1 else [16]
        self.begin = O.table_layout(self.res, c.bw)
        self.table = (rng.standard_normal((int(self.begin[-1]), c.F)) * 0.5).astype(np.float32)
        self.lod_idx = c.L if c.lod_idx < 0 else c.lod_idx
        dens, col = c.dims()

        def mlp(dims):
            Ws = [(rng.uniform(-1, 1, (o, i)) / np.sqrt(i)).astype(np.float32) for i, o in zip(dims[:-1], dims[1:])]
            bs = [(rng.uniform(-1, 1, o) / np.sqrt(i)).astype(np.float32) for i, o in zip(dims[:-1], dims[1:])] if c.bias else None
            return Ws, bs
        dW, db = mlp(dens); cW, cb = mlp(col)
        if c.bias:
            db[-1][0] = 0.1
        self.dec = T.Decoders(dW, db, cW, cb)
        self.dens_dims, self.col_dims = dens, col
        # rays and sample records: samples of a ray are consecutive and ordered by t; the last sample belongs to the last ray
        self.o = rng.uniform(-0.4, 0.4, (c.R, 3)).astype(np.float32)
        d = rng.standard_normal((c.R, 3)).astype(np.float32)
        self.d = (d / np.linalg.norm(d, axis=1, keepdims=True)).astype(np.float32)
        ray = np.sort(rng.integers(0, c.R, S)).astype(np.int32)
        if S:
            ray[-1] = c.R - 1
        t = rng.uniform(0.0, 0.5, S).astype(np.float32)
        order = np.lexsort((t, ray))
        self.rec_ray, self.rec_t = ray[order], t[order]
        # sample positions as the kernels form them: fma(dir, t, origin) in fp32
        self.pos = (self.o[self.rec_ray].astype(np.float64) + self.d[self.rec_ray].astype(np.float64) * self.rec_t[:, None].astype(np.float64)).astype(np.float32)
        spec = ops.NefSpec(resolutions=self.res, begin_idxes=[int(b) for b in self.begin], codebook_size=2 ** c.bw, feature_dim=c.F,
                           multiscale=c.multiscale, lod_idx=self.lod_idx, pos_mode=c.pos[0], pos_freq=c.pos[1], view_mode=c.view[0],
                           view_freq=c.view[1], has_bias=c.bias, dens_dims=dens, col_dims=col)
        fd, fc = self.dec.flat()
        self.t_table, self.t_fd, self.t_fc = [torch.from_numpy(a).cuda() for a in (self.table, fd, fc)]
        self.desc, self.keep = spec.desc([self.t_table], self.t_fd, self.t_fc)
        self.rays, self.rkeep = self.A.make_rays(torch.from_numpy(self.o).cuda(), torch.from_numpy(self.d).cuda(), 0.0, 1.0)
        self.t_rec_t, self.t_rec_ray = torch.from_numpy(self.rec_t).cuda(), torch.from_numpy(self.rec_ray).cuda()
        L = self.A.lib()
        self.L = L
        nblob = int(L.wb_rf_param_blob_floats(C.byref(self.desc), C.c_int32(1)))
        assert nblob > 0, L.wb_last_error()
        self.blob = torch.empty(nblob, dtype=torch.float32, device="cuda")
        self.A.check(L.wb_rf_pack_params(C.byref(self.desc), C.c_int32(1), self.A.ptr(self.blob), self.A.stream()))
        r16 = lambda v: -(-v // 16) * 16
        self.Kp0, self.Kc = r16(dens[0]), r16(col[0])
        self.planes = (min(self.lod_idx, c.L) if c.multiscale == "cat" else 1)
        wsb = int(L.wb_rf_workspace_bytes(C.byref(self.desc), C.c_int32(1), C.c_int64(c.R), C.c_int64(S), C.c_int32(1 if c.backward else 0)))
        assert wsb > 0
        self.ws = torch.zeros(wsb, dtype=torch.uint8, device="cuda")
        fb = int(L.wb_rf_feat_bytes(C.byref(self.desc), C.c_int32(1), C.c_int64(S))) if c.backward else self.Kp0 * 2 * S + 256
        assert fb > 0, L.wb_last_error()
        self.feat = torch.full((fb,), 0xFF, dtype=torch.uint8, device="cuda")
        self.view = T.view_embedding(self.d[self.rec_ray], *c.view)

    # ---- calls ----------------------------------------------------------------------------------------------------
    def forward(self):
        shaded = torch.full((max(self.S, 1), 4), 7.0, dtype=torch.float32, device="cuda")
        self.A.check(self.L.wb_rf_shade_fwd(C.byref(self.desc), self.A.ptr(self.blob), C.c_int32(1), C.byref(self.rays), self.A.ptr(self.t_rec_t),
                                            self.A.ptr(self.t_rec_ray), C.c_int64(self.S), self.A.ptr(shaded), self.A.ptr(self.feat),
                                            self.A.ptr(self.ws), self.A.stream()))
        torch.cuda.synchronize()
        return shaded.cpu().numpy().astype(np.float64)

    def x0_rows(self):
        n = self.Kp0 * self.S
        h = self.feat[:2 * n].view(torch.float16).reshape(self.Kp0 // 8, self.S, 8).permute(1, 0, 2).reshape(self.S, self.Kp0)
        return h.float().cpu().numpy().astype(np.float64)

    def set_x0_rows(self, X):
        Xp = np.zeros((self.S, self.Kp0), np.float16); Xp[:, :X.shape[1]] = X
        img = np.ascontiguousarray(Xp.reshape(self.S, self.Kp0 // 8, 8).transpose(1, 0, 2)).reshape(-1)
        self.feat[:2 * img.size].view(torch.float16).copy_(torch.from_numpy(img).cuda())

    def loss_scale(self, g):
        absmax = torch.tensor([float(np.abs(g).max()) if g.size else 0.0], dtype=torch.float32, device="cuda")
        scale = torch.empty(1, dtype=torch.float32, device="cuda")
        self.A.check(self.L.wb_rf_loss_scale(self.A.ptr(absmax), self.A.ptr(scale), self.A.stream()))
        return scale

    def zeros_grads(self):
        return (torch.zeros_like(self.t_fd), torch.zeros_like(self.t_fc), torch.zeros_like(self.t_table))

    def decoder_bwd(self, g, scale):
        gd, gc, _ = self.zeros_grads()
        tg = torch.from_numpy(np.ascontiguousarray(g, np.float32)).cuda()
        self.A.check(self.L.wb_rf_decoder_bwd(C.byref(self.desc), self.A.ptr(self.blob), C.byref(self.rays), self.A.ptr(self.t_rec_t),
                                              self.A.ptr(self.t_rec_ray), C.c_int64(self.S), self.A.ptr(tg), self.A.ptr(scale), self.A.ptr(self.feat),
                                              self.A.ptr(self.ws), self.A.ptr(gd), self.A.ptr(gc), self.A.stream()))
        torch.cuda.synchronize()
        off = (self.R * self.Kc * 2 + 255) // 256 * 256          # dL/dfeat planes behind the per-ray rows (include/wispb200.h)
        n = self.planes * self.S * self.c.F
        planes = self.ws[off:off + 2 * n].view(torch.float16).reshape(self.planes, self.S, self.c.F).float().cpu().numpy().astype(np.float64)
        return gd.cpu().numpy().astype(np.float64), gc.cpu().numpy().astype(np.float64), planes

    def table_scatter(self, scale):
        gt = torch.zeros_like(self.t_table)
        self.A.check(self.L.wb_rf_table_scatter(C.byref(self.desc), C.byref(self.rays), self.A.ptr(self.t_rec_t), self.A.ptr(self.t_rec_ray),
                                                C.c_int64(self.S), self.A.ptr(scale), self.A.ptr(self.ws), self.A.ptr(gt), self.A.stream()))
        torch.cuda.synchronize()
        return gt.cpu().numpy().astype(np.float64)

    def shade_bwd(self, g, scale):
        gd, gc, gt = self.zeros_grads()
        tg = torch.from_numpy(np.ascontiguousarray(g, np.float32)).cuda()
        self.A.check(self.L.wb_rf_shade_bwd(C.byref(self.desc), self.A.ptr(self.blob), C.c_int32(1), C.byref(self.rays), self.A.ptr(self.t_rec_t),
                                            self.A.ptr(self.t_rec_ray), C.c_int64(self.S), self.A.ptr(tg), self.A.ptr(scale), self.A.ptr(self.feat),
                                            self.A.ptr(self.ws), self.A.ptr(gt), self.A.ptr(gd), self.A.ptr(gc), self.A.stream()))
        torch.cuda.synchronize()
        return gd.cpu().numpy().astype(np.float64), gc.cpu().numpy().astype(np.float64), gt.cpu().numpy().astype(np.float64)

    # ---- references -----------------------------------------------------------------------------------------------
    def grid_features(self):
        """fp32 hash-grid features of the sample positions, 'cat' zeroing / 'sum' applied -> [S, feat_dim]."""
        c = self.c
        raw = O.hashgrid_fwd(self.pos, self.table, self.res, c.bw).reshape(self.S, c.L, c.F)
        if c.multiscale == "cat":
            raw[:, self.lod_idx:] = 0.0
            return raw.reshape(self.S, -1).astype(np.float64)
        acc = np.zeros((self.S, c.F), np.float32)
        for l in range(c.L):
            acc = (acc + raw[:, l]).astype(np.float32)
        return acc.astype(np.float64)

    def wgrad_n(self):
        sms = torch.cuda.get_device_properties(0).multi_processor_count
        return max(T.wgrad_height(self.S, ctas=sms, groups=g) for g in (1, 2))


def _check_inside(name, got, centre, radius, report):
    err = np.abs(got - centre)
    bad = err > radius
    ratio = float(np.max(err / np.maximum(radius, 1e-300))) if got.size else 0.0
    report.append(f"{name}: max|k-c|/r={ratio:.3f} median_r={float(np.median(radius)) if radius.size else 0:.3e}")
    assert not bad.any(), (name, int(bad.sum()), np.argwhere(bad)[:5].tolist(), got[bad][:5], centre[bad][:5], radius[bad][:5])


def _forward_checks(s: Setup, report):
    c = s.c
    shaded = s.forward()
    X = s.x0_rows()
    feat_dim = c.L * c.F if c.multiscale == "cat" else c.F
    pd = embed_dim(*c.pos)
    ref = s.grid_features()
    assert np.all(np.abs(X[:, :feat_dim] - T.f16(ref)) <= _f16ulp(ref)), "grid features of the saved X0 rows"
    if pd:
        pe = T.position_embedding(s.pos.astype(np.float64), *c.pos)
        err = np.abs(X[:, feat_dim:feat_dim + pd] - T.f16(pe))
        assert np.all(err <= _f16ulp(pe)), ("position embedding of the saved X0 rows", np.argwhere(err > _f16ulp(pe))[:5].tolist())
    assert np.all(X[:, feat_dim + pd:] == 0.0), "padding of the saved X0 rows"
    rf = T.Reference(s.dec, X[:, :feat_dim + pd], s.view)
    cen, rad = rf.shaded()
    _check_inside("shaded", shaded, cen, rad, report)
    report.append(f"shaded median radius rgb {np.median(rad[:, :3]):.2e} vs TOL[1] rgb {TOL1_RGB:.0e}")


def _backward_checks(s: Setup, report, rng):
    c = s.c
    I0 = s.dens_dims[0]
    # synthetic X0 rows with exact zeros and negatives
    X = T.f16(rng.standard_normal((s.S, I0)) * 0.7)
    X[rng.random((s.S, I0)) < 0.1] = 0.0
    s.set_x0_rows(X.astype(np.float16))
    g = (rng.standard_normal((s.S, 4)) * 1e-2).astype(np.float32)
    g[rng.random(s.S) < 0.05] = 0.0
    scale_t = s.loss_scale(g)
    scale = float(scale_t.item())
    gd, gc, planes = s.decoder_bwd(g, scale_t)
    rf = T.Reference(s.dec, X, s.view)
    bw = rf.backward(g, scale, s.planes, c.F, wgrad_n=s.wgrad_n())
    for nm, got in (("grad_dens", gd), ("grad_col", gc), ("dfeat", planes)):
        key = {"grad_dens": "dens", "grad_col": "col", "dfeat": "dfeat"}[nm]
        _check_inside(nm, got, *bw[key], report)
    for key in ("dens", "col"):
        cc, rr = bw[key]
        report.append(f"{key}: median radius / max|grad| {np.median(rr) / max(np.abs(cc).max(), 1e-30):.2e} vs TOL[1] grad {TOL1_GRAD:.0e}")
    # stand-alone table scatter of the planes this kernel produced
    gt = s.table_scatter(scale_t)
    cen, rad = T.table_scatter_bound(planes, scale, s.pos, s.table.shape[0], s.res, c.bw, s.lod_idx, c.multiscale)
    _check_inside("table_scatter", gt, cen, rad, report)
    if fusable(c):
        gd2, gc2, gt2 = s.shade_bwd(g, scale_t)
        _check_inside("fused grad_dens", gd2, *bw["dens"], report)
        _check_inside("fused grad_col", gc2, *bw["col"], report)
        # the fused epilogue scatters the fp32 dX: one rounding less than the planes, which are one fp16 rounding away
        _check_inside("fused table_scatter", gt2, cen, rad * (7.0 / 6.0), report)
    return g, X


@pytest.mark.parametrize("case", CASES, ids=case_id)
def test_tc_decoders_vs_interval_reference(W, case):
    s = Setup(W, case)
    report = [case_id(case)]
    supported = int(s.L.wb_rf_precision_supported(C.byref(s.desc), C.c_int32(1), C.c_int32(1)))
    assert supported == int(case.backward)
    assert int(s.L.wb_rf_precision_supported(C.byref(s.desc), C.c_int32(1), C.c_int32(0))) == 1
    _forward_checks(s, report)
    if case.backward:
        _backward_checks(s, report, np.random.default_rng(case.seed + 7))
    print("TCREPORT " + " | ".join(report))


SIZE_CASE = Case("sizes", [64], [64, 64], view=(3, 4), L=16, R=7)


@pytest.mark.parametrize("S", [1, 63, 64, 65, 129, 200_003])
def test_tc_decoders_sample_counts(W, S):
    """The tail tile, a single sample, whole tiles and a large launch (every CTA walks several tiles) on the bench-shaped decoder."""
    case = Case(**{**SIZE_CASE.__dict__, "S": S, "R": 7 if S < 1000 else 3000})
    s = Setup(W, case)
    report = [f"S={S} {case_id(case)}"]
    _forward_checks(s, report)
    _backward_checks(s, report, np.random.default_rng(S))
    print("TCREPORT " + " | ".join(report))


def test_tc_no_samples_touches_nothing(W):
    s = Setup(W, Case("empty", [32], [32, 32], L=8), S=0)
    sentinel = 3.25
    shaded = torch.full((4, 4), sentinel, device="cuda")
    gd, gc, gt = (torch.full_like(t, sentinel) for t in (s.t_fd, s.t_fc, s.t_table))
    g = torch.zeros((1, 4), device="cuda"); scale = torch.ones(1, device="cuda")
    A, L, p = s.A, s.L, s.A.ptr
    A.check(L.wb_rf_shade_fwd(C.byref(s.desc), p(s.blob), C.c_int32(1), C.byref(s.rays), p(s.t_rec_t), p(s.t_rec_ray), C.c_int64(0), p(shaded),
                              p(s.feat), p(s.ws), A.stream()))
    A.check(L.wb_rf_decoder_bwd(C.byref(s.desc), p(s.blob), C.byref(s.rays), p(s.t_rec_t), p(s.t_rec_ray), C.c_int64(0), p(g), p(scale), p(s.feat),
                                p(s.ws), p(gd), p(gc), A.stream()))
    A.check(L.wb_rf_table_scatter(C.byref(s.desc), C.byref(s.rays), p(s.t_rec_t), p(s.t_rec_ray), C.c_int64(0), p(scale), p(s.ws), p(gt), A.stream()))
    A.check(L.wb_rf_shade_bwd(C.byref(s.desc), p(s.blob), C.c_int32(1), C.byref(s.rays), p(s.t_rec_t), p(s.t_rec_ray), C.c_int64(0), p(g), p(scale),
                              p(s.feat), p(s.ws), p(gt), p(gd), p(gc), A.stream()))
    torch.cuda.synchronize()
    for t in (shaded, gd, gc, gt):
        assert bool((t == sentinel).all())


def test_chunked_backward_matches_two_stages(W):
    """From 2^20 samples on, wb_rf_shade_bwd of a decoder whose backward runs one group per CTA cuts the samples into four chunks and
    runs the table scatter of each chunk on a side stream beside the decoder backward of the next.  It must compute what
    wb_rf_decoder_bwd followed by wb_rf_table_scatter over all samples computes, up to the order of the atomic additions."""
    case = Case("chunked", [128], [128, 128], view=(3, 4), L=16, S=(1 << 20) + 4097, R=5000)
    plan = bwd_plan(case)
    assert plan[0] == 1
    s = Setup(W, case)
    s.forward()
    g = (np.random.default_rng(5).standard_normal((s.S, 4)) * 1e-2).astype(np.float32)
    scale = s.loss_scale(g)
    n0 = s.A.launch_count()
    gd1, gc1, gt1 = s.shade_bwd(g, scale)
    # the per-ray rows once, then per chunk every pass of the decoder backward and one scatter
    assert s.A.launch_count() - n0 == 1 + 4 * (len(plan) + 1)
    gd2, gc2, _ = s.decoder_bwd(g, scale)
    gt2 = s.table_scatter(scale)
    report = [case_id(case)]
    for nm, a, b in (("grad_table", gt1, gt2), ("grad_dens", gd1, gd2), ("grad_col", gc1, gc2)):
        top = float(np.abs(b).max())
        ratio = float(np.abs(a - b).max()) / top
        report.append(f"{nm}: max|chunked - two-stage| / max|two-stage| = {ratio:.2e}")
        assert top > 0.0 and ratio <= TOL1_GRAD, (nm, ratio)
    print("TCREPORT " + " | ".join(report))


def test_ray_rows_flag_applies_to_the_next_backward_only(W):
    """wb_rf_workspace_holds_ray_rows(1) covers the next backward call of the thread, also when that call has nothing to do (S == 0):
    a later backward into a workspace without the per-ray colour-input rows must write them itself."""
    s = Setup(W, Case("rows", [64], [64, 64], view=(3, 4), L=16))
    rng = np.random.default_rng(3)
    X = T.f16(rng.standard_normal((s.S, s.dens_dims[0])) * 0.7)
    s.set_x0_rows(X.astype(np.float16))
    g = (rng.standard_normal((s.S, 4)) * 1e-2).astype(np.float32)
    scale = s.loss_scale(g)
    want = s.decoder_bwd(g, scale)
    A, L, p = s.A, s.L, s.A.ptr
    gd, gc, _ = s.zeros_grads()
    A.check(L.wb_rf_workspace_holds_ray_rows(C.c_int32(1)))
    A.check(L.wb_rf_decoder_bwd(C.byref(s.desc), p(s.blob), C.byref(s.rays), p(s.t_rec_t), p(s.t_rec_ray), C.c_int64(0), p(gd), p(scale),
                                p(s.feat), p(s.ws), p(gd), p(gc), A.stream()))
    s.ws.fill_(0xFF)                          # a fresh workspace: 0xFFFF is an fp16 NaN
    got = s.decoder_bwd(g, scale)
    bw = T.Reference(s.dec, X, s.view).backward(g, float(scale.item()), s.planes, 2, wgrad_n=s.wgrad_n())
    for a, b, key in zip(got, want, ("dens", "col", "dfeat")):
        assert np.all(np.abs(a - b) <= 2 * bw[key][1]), key        # both inside the reference interval: atomic order only


def _scale_formula(a):
    """2^clamp(floor(log2(64 / max(absmax, 1e-30))), -20, 60) in exact arithmetic (include/wispb200.h)."""
    a = max(float(np.float32(a)), float(np.float32(1e-30)))
    x = Fraction(64) / Fraction(a)
    k = x.numerator.bit_length() - x.denominator.bit_length()
    while Fraction(2) ** k > x:
        k -= 1
    while Fraction(2) ** (k + 1) <= x:
        k += 1
    return 2.0 ** min(max(k, -20), 60)


def test_loss_scale_formula(W):
    vals = [0.0, 1e-30, 1e-35, 2.0 ** -54, 2.0 ** -55, 2.0 ** 26, 2.0 ** 27 * 1.5, 3e38]
    for e in range(-3, 10):                                          # around each power of two near 64
        p = np.float32(2.0 ** e)
        vals += [float(np.nextafter(p, np.float32(0))), float(p), float(np.nextafter(p, np.float32(np.inf))), float(p) * 1.5]
    A = W._cabi
    absmax = torch.tensor(vals, dtype=torch.float32, device="cuda")
    out = torch.empty_like(absmax)
    for i in range(len(vals)):
        A.check(A.lib().wb_rf_loss_scale(C.c_void_p(absmax.data_ptr() + 4 * i), C.c_void_p(out.data_ptr() + 4 * i), A.stream()))
    got = out.cpu().numpy()
    want = np.array([_scale_formula(np.float32(v)) for v in vals], np.float32)
    bad = got != want
    assert not bad.any(), [(vals[i], float(got[i]), float(want[i])) for i in np.flatnonzero(bad)]


@pytest.mark.parametrize("k", [3, -5])
def test_backward_is_invariant_to_the_loss_scale(W, k):
    """g_shaded * 2^k -> a loss scale 2^-k times smaller: the fp16 values are the same, the unscaled gradients are 2^k times the
    original up to atomic order (both lie in the reference interval, so they differ by at most 2^k * 2 radius)."""
    s = Setup(W, Case("scale", [64], [64, 64], view=(3, 4), L=16, S=777))
    rng = np.random.default_rng(11)
    X = T.f16(rng.standard_normal((s.S, s.dens_dims[0])) * 0.7)
    s.set_x0_rows(X.astype(np.float16))
    g = (rng.standard_normal((s.S, 4)) * 1e-2).astype(np.float32)
    s1, s2 = s.loss_scale(g), s.loss_scale(g * np.float32(2.0 ** k))
    assert float(s1.item()) == float(s2.item()) * 2.0 ** k
    gd1, gc1, p1 = s.decoder_bwd(g, s1)
    gd2, gc2, p2 = s.decoder_bwd(g * np.float32(2.0 ** k), s2)
    assert np.array_equal(p1, p2)
    bw = T.Reference(s.dec, X, s.view).backward(g, float(s1.item()), s.planes, 2, wgrad_n=s.wgrad_n())
    for a, b, key in ((gd1, gd2, "dens"), (gc1, gc2, "col")):
        assert np.all(np.abs(b - 2.0 ** k * a) <= 2.0 ** k * 2 * bw[key][1] + 1e-30), key
