"""The NeRF shade kernels over TriplanarGrid, OctreeGrid and HashGrid through the C ABI, against the float64 interval reference
tests/rf_reference.py: every output must lie in centre +- radius.

Covers what the end-to-end comparisons cannot resolve at their tolerances:
  - the fused gather (wb_featx_gather) and scatter (wb_featx_scatter, wb_featx_scatter_kernel) of triplanar grids with fdim 1..8,
    both plane layouts, 'cat' / 'sum', 1..12 LODs, plane sides 2, 3, odd and 513, fewer LODs than the grid has, samples outside
    the cube, at +-1 and on texel lines, runs of consecutive samples in one texel cell longer than a warp;
  - the same for octree grids with F 1..32, base_lod > 0 and 0, half_round on and off, lod_idx below the finest, 'sum' over a
    single LOD, points whose descent stops at a coarse level and points outside the cube;
  - both precisions where wb_rf_precision_supported allows them (precision 1: the saved X0 rows, wb_rf_decoder_bwd +
    wb_rf_table_scatter and wb_rf_shade_bwd);
  - the fp32 SIMT decoders (precision 0) of depth 1..3 / 1..4, widths up to 256 and not multiples of 8, with and without bias,
    every embedding mode, the NT = 128 / 64 / 32 tiles, 1 sample, NT +- 1 samples and three tiles per CTA;
  - the unfused wb_triplane_fwd / wb_triplane_bwd at fdim 1..8.
Each case prints one RFREPORT line: max|k - c| / r and the median radius of every checked output."""
import ctypes as C
from dataclasses import dataclass, field
from typing import List

import numpy as np
import pytest
import torch

from oracle import octree_grid as OG
from oracle import oracle as O
from oracle import sdf_reference as S
from oracle import tc_decoders as T

import rf_reference as RF

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def W():
    import wisp_b200
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return wisp_b200


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def embed_dim(mode, freq):
    return 0 if mode == 0 else 3 if mode == 1 else 6 * freq if mode == 2 else 3 + 6 * freq


@dataclass
class Case:
    name: str
    kind: str                               # 'triplanar' | 'octree' | 'hash'
    ms: str = "cat"
    C: int = 4                              # triplanar channels per plane / octree features per LOD / hash features per LOD
    sides: tuple = (5, 9)                   # triplanar plane sides of the grid's LODs
    nl: int = 0                             # LODs used (lod_idx + 1); 0: all
    layout: int = 0                         # triplanar plane layout (1: channel-last)
    level: int = 5                          # octree depth
    lods: int = 3                           # octree LODs of the grid
    half: bool = True
    dens: List[int] = field(default_factory=lambda: [32])
    col: List[int] = field(default_factory=lambda: [32, 32])
    dout: int = 16
    pos: tuple = (0, 0)
    view: tuple = (3, 2)
    bias: bool = True
    S: int = 1500
    R: int = 48
    seed: int = 0

    def grid_lods(self):
        return len(self.sides) if self.kind == "triplanar" else self.lods if self.kind == "octree" else 8

    def used(self):
        return self.nl or self.grid_lods()

    def feat_dim(self):
        w = 3 * self.C if self.kind == "triplanar" else self.C
        return w * (self.used() if self.ms == "cat" else 1)

    def dims(self):
        return ([self.feat_dim() + embed_dim(*self.pos)] + list(self.dens) + [self.dout],
                [self.dout - 1 + embed_dim(*self.view)] + list(self.col) + [3])


SIDES12 = (2, 3, 4, 5, 7, 9, 11, 13, 17, 33, 65, 129)
TRIPLANAR = [
    Case("tp_f1_cat_side2", "triplanar", C=1, sides=(2,), view=(3, 4)),
    Case("tp_f1_S20", "triplanar", C=1, sides=(3, 5), S=20, R=5),
    Case("tp_f2_sum_L4", "triplanar", ms="sum", C=2, sides=(3, 5, 9, 17), pos=(1, 0), view=(1, 0)),
    Case("tp_f2_cat_L12", "triplanar", C=2, sides=SIDES12, dens=[64], col=[64, 64]),
    Case("tp_f3_cat_lod2of4", "triplanar", C=3, sides=(3, 7, 13, 25), nl=2, pos=(3, 1)),
    Case("tp_f4_cat_layout0", "triplanar", C=4, sides=(5, 9, 17, 33)),
    Case("tp_f4_cat_layout1", "triplanar", C=4, sides=(65, 129, 257, 513), layout=1),
    Case("tp_f4_sum_layout1", "triplanar", ms="sum", C=4, sides=(3, 5, 9, 17), layout=1, view=(2, 2)),
    Case("tp_f5_sum_L12", "triplanar", ms="sum", C=5, sides=SIDES12, view=(0, 0)),
    Case("tp_f8_cat_L4", "triplanar", C=8, sides=(2, 3, 11, 513), dens=[64], col=[64, 64]),
    Case("tp_f8_sum_513", "triplanar", ms="sum", C=8, sides=(513,), pos=(2, 2)),
]
OCTREE = [
    Case("oct_F1_cat", "octree", C=1, lods=4, view=(3, 4)),
    Case("oct_F3_sum_half0", "octree", ms="sum", C=3, lods=4, half=False, pos=(1, 0)),
    Case("oct_F8_cat_lod1of4", "octree", C=8, lods=4, nl=2),
    Case("oct_F8_sum_base0", "octree", ms="sum", C=8, level=3, lods=4),
    Case("oct_F16_sum_lod0", "octree", ms="sum", C=16, lods=3, nl=1, half=False),
    Case("oct_F16_cat_half0", "octree", C=16, lods=3, half=False, view=(2, 1)),
    Case("oct_F32_cat", "octree", C=32, lods=3, dens=[64], col=[64, 64]),
]
# precision-0 decoders over a hash grid; the comments give the backward tile NT of rf_reference.shade0_plan
DECODERS = [
    Case("d1c1_w16", "hash", C=2, dens=[], col=[], view=(1, 0), pos=(2, 3)),                     # NT 128
    Case("d2c3_w48_nobias", "hash", C=2, dens=[48], col=[48, 48], bias=False, pos=(3, 2), view=(2, 3)),
    Case("d3c4_w100_nt64", "hash", C=2, dens=[100, 60], col=[100, 36, 20], pos=(1, 0), view=(3, 4)),  # NT 64
    Case("d2c2_w256_nt32", "hash", C=2, dens=[256], col=[256], view=(3, 4), S=700),            # NT 32
    Case("d2c3_w20_F4", "hash", C=4, dens=[20], col=[20, 44], dout=9, pos=(0, 0), view=(0, 0)),
]


def _rays(c: Case, rng):
    """Rays and ray-sorted sample records.  Triplanar: far rays (positions several periods outside [-1, 1]), axis-aligned rays whose
    two other coordinates are exactly +-1, 0 or texel lines, and dense rays whose samples stay in one texel cell for 40+ records."""
    R, S_ = c.R, c.S
    if c.kind == "triplanar":
        o = rng.uniform(-3.5, 3.5, (R, 3))
        d = rng.standard_normal((R, 3))
        special = np.array([-1.0, 1.0, 0.0, 0.5, -0.5, 0.75, 3.0, -2.0])
        for r in range(0, R, 3):                            # axis-aligned: coordinates k+1, k+2 stay exact
            k = r % 3
            d[r] = 0.0; d[r, k] = 1.0
            o[r] = special[rng.integers(0, special.size, 3)]; o[r, k] = -1.0
    elif c.kind == "octree":
        o = rng.uniform(-1.3, 1.3, (R, 3)); d = rng.standard_normal((R, 3))
    else:
        o = rng.uniform(-0.4, 0.4, (R, 3)); d = rng.standard_normal((R, 3))
    d = d / np.linalg.norm(d, axis=1, keepdims=True)
    ray = np.sort(rng.integers(0, R, S_)).astype(np.int32)
    t = rng.uniform(0.0, 2.0 if c.kind != "hash" else 0.5, S_)
    if c.kind == "triplanar" and S_ >= 400:                 # two dense rays of 70 records each
        for k, r in enumerate((1, 4)):
            ray[ray == r] = r + 1
            sl = slice(100 + 150 * k, 170 + 150 * k)
            ray[sl] = r
            t[sl] = 0.3 + rng.uniform(0, 1e-4, 70)
    if S_:
        ray[-1] = R - 1
    order = np.lexsort((t, ray))
    return o.astype(np.float32), d.astype(np.float32), ray[order].astype(np.int32), t[order].astype(np.float32)


class Setup:
    def __init__(self, W, c: Case, S_=None):
        from wisp_b200 import ops
        self.W, self.A, self.c = W, W._cabi, c
        if S_ is not None:
            c = Case(**{**c.__dict__, "S": S_})
            self.c = c
        rng = np.random.default_rng(100 + c.seed)
        self.o, self.d, self.rec_ray, self.rec_t = _rays(c, rng)
        self.S = c.S
        self.pos = RF.positions(self.o, self.d, self.rec_ray, self.rec_t)
        self.dirs = self.d[self.rec_ray]
        dens, col = c.dims()
        self.dens_dims, self.col_dims = dens, col

        def mlp(dims):
            Ws = [(rng.uniform(-1, 1, (o, i)) / np.sqrt(i)).astype(np.float32) for i, o in zip(dims[:-1], dims[1:])]
            bs = [(rng.uniform(-1, 1, o) / np.sqrt(i)).astype(np.float32) for i, o in zip(dims[:-1], dims[1:])] if c.bias else None
            return Ws, bs
        dW, db = mlp(dens); cW, cb = mlp(col)
        self.dec = T.Decoders(dW, db, cW, cb)
        fd, fc = self.dec.flat()
        self.t_fd, self.t_fc = dev(fd), dev(fc)
        nl = c.used()
        common = dict(multiscale=c.ms, pos_mode=c.pos[0], pos_freq=c.pos[1], view_mode=c.view[0], view_freq=c.view[1], has_bias=c.bias,
                      dens_dims=dens, col_dims=col)
        self.t_table = None
        if c.kind == "triplanar":
            planes = [[(rng.standard_normal((c.C, s, s)) * 0.5).astype(np.float32) for _ in range(3)] for s in c.sides]
            self.tp = RF.Triplanar(planes, c.ms, nl)
            host = [p if c.layout == 0 else np.ascontiguousarray(p.transpose(1, 2, 0)) for l in range(nl) for p in planes[l]]
            self.grid = [dev(p) for p in host]
            self.grads = [torch.zeros_like(g) for g in self.grid]
            spec = ops.NefSpec(resolutions=[s - 1 for s in c.sides[:nl]], begin_idxes=[], codebook_size=0, feature_dim=3 * c.C,
                               lod_idx=nl - 1, kind="triplanar", num_lods=nl, **common)
            self.desc, self.keep = spec.desc(self.grid, self.t_fd, self.t_fc, grads=self.grads, layout=c.layout)
            self.width = 3 * c.C
        elif c.kind == "octree":
            spc = O.octree_to_spc(O.points_to_octree(O.lego_like_points(c.level), c.level))
            _, pyr, trinkets, _ = OG.make_trilinear_spc(spc)
            base = c.level - c.lods + 1
            feats = [(rng.standard_normal((int(pyr[0, base + k]), c.C)) * 0.5).astype(np.float32) for k in range(c.lods)]
            self.field = RF.octree_field(spc, trinkets, feats, base, c.ms, c.half)
            self.blas = W.OctreeAS(dev(spc.octree))
            self.t_trinkets = dev(trinkets.astype(np.int32))
            self.grid = [dev(f) for f in feats[:nl]]
            self.grads = [torch.zeros_like(g) for g in self.grid]
            spec = ops.NefSpec(resolutions=[], begin_idxes=[], codebook_size=0, feature_dim=c.C, lod_idx=nl - 1, kind="octree", num_lods=nl,
                               base_lod=base, half_round=c.half, **common)
            self.desc, self.keep = spec.desc(self.grid, self.t_fd, self.t_fc, self.blas.tensors(), self.t_trinkets, grads=self.grads)
            self.width = c.C
        else:
            self.res = O.geometric_resolutions(8, 4, 64)
            self.begin = O.table_layout(self.res, 12)
            self.table = (rng.standard_normal((int(self.begin[-1]), c.C)) * 0.5).astype(np.float32)
            self.t_table = dev(self.table)
            spec = ops.NefSpec(resolutions=self.res, begin_idxes=[int(b) for b in self.begin], codebook_size=2 ** 12, feature_dim=c.C,
                               lod_idx=8, **common)
            self.desc, self.keep = spec.desc([self.t_table], self.t_fd, self.t_fc)
            self.grads = [torch.zeros_like(self.t_table)]
            self.width = c.C
        self.planes = nl if c.ms == "cat" else 1
        self.rays, self.rkeep = self.A.make_rays(dev(self.o), dev(self.d), 0.0, 1.0)
        self.t_rec_t, self.t_rec_ray = dev(self.rec_t), dev(self.rec_ray)
        self.L = self.A.lib()

    # ---- reference features -----------------------------------------------------------------------------------------------
    def x0(self):
        """(centre, radius) of the density-decoder input [S, I0] and the octree cells."""
        c = self.c
        self.cells = None
        if c.kind == "triplanar":
            fc, fr = RF.triplanar_features(self.tp, self.pos)
        elif c.kind == "octree":
            fc, fr, self.cells = RF.octree_features(self.field, self.pos, c.used())
        else:
            fc, fr = RF.hash_features(self.pos, self.table, self.res, 12, c.ms, 8)
        pc, pr = S._embed(S.Field(None, None, [], 0, "", [], [], c.pos[0], c.pos[1]), self.pos.astype(np.float64), False)
        return np.concatenate([fc, pc], 1), np.concatenate([fr, pr], 1)

    def grid_reference(self, gc, gr, levels):
        c = self.c
        if c.kind == "triplanar":
            out = RF.triplanar_scatter(self.tp, self.pos, gc, gr, levels)
            res = []
            for l in range(c.used()):
                for p in range(3):
                    cc, rr = out[l][p]
                    if c.layout == 1:
                        cc, rr = cc.transpose(1, 2, 0), rr.transpose(1, 2, 0)
                    res.append((cc, rr))
            return res
        return RF.octree_scatter(self.field, self.cells, c.used(), gc, gr, levels)

    # ---- calls ----------------------------------------------------------------------------------------------------------------
    def blob(self, precision):
        n = int(self.L.wb_rf_param_blob_floats(self.desc, precision))
        assert n > 0, self.L.wb_last_error()
        b = torch.empty(n, dtype=torch.float32, device="cuda")
        self.L.wb_rf_pack_params(self.desc, precision, self.A.ptr(b), self.A.stream())
        return b

    def zero(self):
        for g in self.grads:
            g.zero_()
        return torch.zeros_like(self.t_fd), torch.zeros_like(self.t_fc)

    def grid_grads(self):
        return [g.cpu().numpy().astype(np.float64) for g in self.grads]

    def fwd(self, precision, blob, feat=None, ws=None):
        shaded = torch.full((max(self.S, 1), 4), 7.0, dtype=torch.float32, device="cuda")
        p = self.A.ptr
        self.L.wb_rf_shade_fwd(self.desc, p(blob), precision, self.rays, p(self.t_rec_t), p(self.t_rec_ray),
                               self.S, p(shaded), p(feat), p(ws), self.A.stream())
        torch.cuda.synchronize()
        return shaded.cpu().numpy().astype(np.float64)[:self.S]

    def shade_bwd(self, precision, blob, g, scale=None, feat=None, ws=None):
        gd, gc = self.zero()
        tg = dev(np.asarray(g, np.float32))
        p = self.A.ptr
        gt = self.grads[0] if self.c.kind == "hash" else None      # triplanar / octree: the gradients named in the description
        self.L.wb_rf_shade_bwd(self.desc, p(blob), precision, self.rays, p(self.t_rec_t), p(self.t_rec_ray),
                               self.S, p(tg), p(scale), p(feat), p(ws), p(gt), p(gd), p(gc), self.A.stream())
        torch.cuda.synchronize()
        return gd.cpu().numpy().astype(np.float64), gc.cpu().numpy().astype(np.float64), self.grid_grads()


def _inside(name, got, centre, radius, report):
    got, centre, radius = (np.asarray(a, np.float64) for a in (got, centre, radius))
    err = np.abs(got - centre)
    bad = ~(err <= radius)
    ratio = float(np.max(err / np.maximum(radius, 1e-300))) if got.size else 0.0
    report.append(f"{name}: {ratio:.3f} r~{float(np.median(radius)) if radius.size else 0:.1e}")
    assert not bad.any(), (name, int(bad.sum()), np.argwhere(bad)[:5].tolist(), got[bad][:5], centre[bad][:5], radius[bad][:5])


def _grid_checks(name, s, got, ref, report):
    for i, (g, (cc, rr)) in enumerate(zip(got, ref)):
        _inside(f"{name}[{i}]", g.reshape(cc.shape), cc, rr, report)


def _g_shaded(s, rng):
    g = (rng.standard_normal((s.S, 4)) * 1e-2).astype(np.float32)
    g[rng.random(s.S) < 0.05] = 0.0
    return g


def run_precision0(s: Setup, report, rng, in_order=True):
    c = s.c
    blob = s.blob(0)
    shaded = s.fwd(0, blob)
    x0c, x0r = s.x0()
    ref = RF.Shade0(s.dec, x0c, x0r, s.dirs, *c.view, in_order=in_order)
    _inside("p0 shaded", shaded, *ref.shaded(), report)
    g = _g_shaded(s, rng)
    gd, gc, grid = s.shade_bwd(0, blob, g)
    plan = RF.shade0_plan(s.dens_dims, s.col_dims)
    bw = ref.backward(g, plan.nt_bwd, max(1, -(-s.S // plan.nt_bwd)))
    _inside("p0 grad_dens", gd, *bw["dens"], report)
    _inside("p0 grad_col", gc, *bw["col"], report)
    if c.kind != "hash":
        fdim = c.feat_dim()
        _grid_checks("p0 grid", s, grid, s.grid_reference(bw["dx0"][0][:, :fdim], bw["dx0"][1][:, :fdim], 0), report)
    return plan


def run_precision1(s: Setup, report, rng):
    c, A, L, p = s.c, s.A, s.L, s.A.ptr
    bwd = int(L.wb_rf_precision_supported(s.desc, 1, 1))
    if not int(L.wb_rf_precision_supported(s.desc, 1, 0)):
        report.append("p1 refused")
        return
    blob = s.blob(1)
    I0 = s.dens_dims[0]
    Kp0, Kc = -(-I0 // 16) * 16, -(-s.col_dims[0] // 16) * 16
    wsb = int(L.wb_rf_workspace_bytes(s.desc, 1, c.R, s.S, bwd))
    ws = torch.zeros(wsb, dtype=torch.uint8, device="cuda")
    fb = int(L.wb_rf_feat_bytes(s.desc, 1, s.S)) if bwd else Kp0 * 2 * s.S + 256
    feat = torch.full((fb,), 0xFF, dtype=torch.uint8, device="cuda")
    shaded = s.fwd(1, blob, feat, ws)
    X = feat[:2 * Kp0 * s.S].view(torch.float16).reshape(Kp0 // 8, s.S, 8).permute(1, 0, 2).reshape(s.S, Kp0).float().cpu().numpy().astype(np.float64)
    x0c, x0r = s.x0()
    fdim = c.feat_dim()
    lo, hi = T.f16(x0c[:, :fdim] - x0r[:, :fdim]), T.f16(x0c[:, :fdim] + x0r[:, :fdim])
    _inside("p1 X0 feats", X[:, :fdim], (lo + hi) * 0.5, (hi - lo) * 0.5, report)
    assert np.all(X[:, I0:] == 0.0), "padding of the saved X0 rows"
    view = T.view_embedding(s.dirs, *c.view)
    rf = T.Reference(s.dec, X[:, :I0], view)
    _inside("p1 shaded", shaded, *rf.shaded(), report)
    if not bwd:
        report.append("p1 backward refused")
        return
    g = _g_shaded(s, rng)
    absmax = torch.tensor([float(np.abs(g).max())], dtype=torch.float32, device="cuda")
    scale_t = torch.empty(1, dtype=torch.float32, device="cuda")
    L.wb_rf_loss_scale(p(absmax), p(scale_t), A.stream())
    scale = float(scale_t.item())
    tg = dev(g)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    bw = rf.backward(g, scale, s.planes, s.width, wgrad_n=max(T.wgrad_height(s.S, ctas=sms, groups=k) for k in (1, 2)))
    off = (c.R * Kc * 2 + 255) // 256 * 256                   # dL/dfeat planes behind the per-ray rows (include/wispb200.h)

    def planes():
        n = s.planes * s.S * s.width
        return ws[off:off + 2 * n].view(torch.float16).reshape(s.planes, s.S, s.width).float().cpu().numpy().astype(np.float64)

    def scatter_ref(pl):
        gx = pl.transpose(1, 0, 2).reshape(s.S, -1) / scale          # feature f: plane f / width, column f % width
        return s.grid_reference(gx, np.zeros_like(gx), RF.SCAN_LEVELS)
    # two stages
    gd, gc = s.zero()
    L.wb_rf_decoder_bwd(s.desc, p(blob), s.rays, p(s.t_rec_t), p(s.t_rec_ray), s.S, p(tg), p(scale_t),
                        p(feat), p(ws), p(gd), p(gc), A.stream())
    L.wb_rf_table_scatter(s.desc, s.rays, p(s.t_rec_t), p(s.t_rec_ray), s.S, p(scale_t), p(ws), None,
                          A.stream())
    torch.cuda.synchronize()
    pl = planes()
    _inside("p1 grad_dens", gd.cpu().numpy(), *bw["dens"], report)
    _inside("p1 grad_col", gc.cpu().numpy(), *bw["col"], report)
    _inside("p1 dfeat", pl, *bw["dfeat"], report)
    _grid_checks("p1 scatter", s, s.grid_grads(), scatter_ref(pl), report)
    # one call
    gd, gc, grid = s.shade_bwd(1, blob, g, scale_t, feat, ws)
    pl2 = planes()
    _inside("p1 shade_bwd grad_dens", gd, *bw["dens"], report)
    _inside("p1 shade_bwd grad_col", gc, *bw["col"], report)
    _inside("p1 shade_bwd dfeat", pl2, *bw["dfeat"], report)
    _grid_checks("p1 shade_bwd grid", s, grid, scatter_ref(pl2), report)


@pytest.mark.parametrize("case", TRIPLANAR + OCTREE, ids=lambda c: c.name)
def test_featx_grids_vs_interval_reference(W, case):
    s = Setup(W, case)
    report = [case.name]
    rng = np.random.default_rng(case.seed + 7)
    run_precision0(s, report, rng)
    run_precision1(s, report, rng)
    print("RFREPORT " + " | ".join(report))


@pytest.mark.parametrize("case", DECODERS, ids=lambda c: c.name)
def test_precision0_decoders_vs_interval_reference(W, case):
    s = Setup(W, case)
    report = [case.name]
    plan = run_precision0(s, report, np.random.default_rng(case.seed + 7))
    report.insert(1, f"NT {plan.nt_fwd}/{plan.nt_bwd}")
    print("RFREPORT " + " | ".join(report))


def _nt_case(nt):
    return {128: DECODERS[1], 64: DECODERS[2], 32: DECODERS[3]}[nt]


@pytest.mark.parametrize("nt,extra", [(128, 1), (128, -1), (128, 1 - 128), (64, 1), (64, -1), (32, 1), (32, -1), (32, "tiles")])
def test_precision0_sample_counts(W, nt, extra):
    """One sample, NT - 1 and NT + 1 samples (the partial tile), and three tiles per CTA (grid-stride over tiles)."""
    case = _nt_case(nt)
    plan = RF.shade0_plan(*case.dims())
    assert plan.nt_bwd == nt
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    S_ = 2 * sms * plan.per_sm * nt + 1 if extra == "tiles" else nt + extra
    s = Setup(W, case, S_=S_)
    if extra == "tiles":
        assert plan.tiles_per_cta(S_, sms) == 3
    report = [f"{case.name} S={S_} NT {plan.nt_bwd}"]
    run_precision0(s, report, np.random.default_rng(S_), in_order=extra != "tiles")
    print("RFREPORT " + " | ".join(report))


def test_precision0_no_samples_touches_nothing(W):
    s = Setup(W, TRIPLANAR[0], S_=0)
    sentinel = 3.25
    shaded = torch.full((4, 4), sentinel, device="cuda")
    for gg in s.grads:
        gg.fill_(sentinel)
    gd, gc = (torch.full_like(t, sentinel) for t in (s.t_fd, s.t_fc))
    g = torch.zeros((1, 4), device="cuda")
    A, L, p = s.A, s.L, s.A.ptr
    blob = s.blob(0)
    L.wb_rf_shade_fwd(s.desc, p(blob), 0, s.rays, p(s.t_rec_t), p(s.t_rec_ray), 0, p(shaded),
                      None, None, A.stream())
    L.wb_rf_shade_bwd(s.desc, p(blob), 0, s.rays, p(s.t_rec_t), p(s.t_rec_ray), 0, p(g), None,
                      None, None, None, p(gd), p(gc), A.stream())
    torch.cuda.synchronize()
    for t in [shaded, gd, gc] + s.grads:
        assert bool((t == sentinel).all())


@pytest.mark.parametrize("fdim", range(1, 9))
def test_unfused_triplane_vs_interval_reference(W, fdim):
    """wb_triplane_fwd / wb_triplane_bwd (the unfused TriplanarGrid.interpolate) against the same feature and scatter reference."""
    case = Case(f"unfused_f{fdim}", "triplanar", C=fdim, sides=(2, 3, 9, 65)[: 1 + fdim % 4], S=1200)
    s = Setup(W, case)
    A, L, p = s.A, s.L, s.A.ptr
    nl = case.used()
    planes = [dev(pl) for l in range(nl) for pl in s.tp.planes[l]]
    gplanes = [torch.zeros_like(t) for t in planes]
    res = (C.c_int32 * nl)(*[sd - 1 for sd in case.sides])
    pp = (C.c_void_p * (3 * nl))(*[t.data_ptr() for t in planes])
    gp = (C.c_void_p * (3 * nl))(*[t.data_ptr() for t in gplanes])
    coords = dev(s.pos)
    feats = torch.empty((s.S, 3 * nl * fdim), dtype=torch.float32, device="cuda")
    L.wb_triplane_fwd(p(coords), s.S, nl, fdim, res, pp, p(feats), A.stream())
    rng = np.random.default_rng(fdim)
    go = rng.standard_normal((s.S, 3 * nl * fdim)).astype(np.float32)
    go[rng.random(go.shape) < 0.1] = 0.0
    L.wb_triplane_bwd(p(coords), s.S, nl, fdim, res, pp, p(dev(go)), gp, A.stream())
    torch.cuda.synchronize()
    report = [case.name]
    _inside("feats", feats.cpu().numpy(), *RF.triplanar_features(s.tp, s.pos), report)
    ref = RF.triplanar_scatter(s.tp, s.pos, go, np.zeros(go.shape), 0)
    for i, t in enumerate(gplanes):
        _inside(f"gplane[{i}]", t.cpu().numpy()[0] if t.dim() == 4 else t.cpu().numpy(), *ref[i // 3][i % 3], report)
    print("RFREPORT " + " | ".join(report))
