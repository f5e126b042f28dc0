"""The app/nerf-shaped tensor-core instances (TcShapeNerf64 in wb_shade_tc.cu) over every decoder they accept, and at coordinate, run
and tile edges.

TcShapeNerf64::matches compares the padded geometry only (Kp = 32, 64, 48, 64, 64 and Np = 64, 16, 64, 64, 16), so the shaped forward
(wb_shade_fwd_tc_kernel<3, false, 64, TcShapeNerf64>) serves every hash-grid decoder of that geometry, and the shaped backward with the
fused table scatter (wb_mlp_bwd_tc_kernel<2, true, TcShapeNerf64>) every such F == 2 'cat' decoder with at most 16 live LODs.  What the
members differ in (real widths, dout, bias, live LODs, embeddings) is read at run time inside the shaped code.  This file

  1. mirrors the selection (nerf64_expected) and sweeps seeded descriptors against wb_rf_tc_shaped, so the family neither shrinks nor
     grows unnoticed (tests/test_tc_shape_family_cpu.py pins the mirror's geometry to the source);
  2. runs members of the family, and controls just outside it, inside the interval reference of test_gpu_tc_decoders.py at S = 700 and
     at three tiles per group; _backward_checks puts the run-time route (wb_rf_decoder_bwd + wb_rf_table_scatter) and the fused one
     (wb_rf_shade_bwd) inside the same intervals;
  3. runs the bench-shaped decoder on explicit sample layouts: coordinates at +-1, on cell faces and outside the cube; long runs of
     lanes in one cell (the scatter's warp run merging) and tail tiles whose clamped lanes share the last sample's cell; sample counts
     where the backward's next-tile prefetch lands on, before or past the last tile of a group; the ray-rows hint before
     wb_rf_shade_bwd.
Every case prints a TCREPORT line with max|k - c|/r and the median radius of each checked output."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import oracle as O
from oracle import tc_decoders as T
from test_gpu_tc_decoders import SIZE_CASE, Case, Setup, _backward_checks, _check_inside, _forward_checks, bwd_plan, fusable

pytestmark = pytest.mark.gpu

# ---- mirror of the instance selection (wb_shade_tc.cu) -------------------------------------------------------------------------
NERF64_ND, NERF64_NC = 2, 3                          # TcShapeNerf64 = TcShape<ND, NC, TcList<KP...>, TcList<NP...>>
NERF64_KP = (32, 64, 48, 64, 64)
NERF64_NP = (64, 16, 64, 64, 16)
TC_SMEM_MAX = 227 * 1024 - 1024
TC_SLAB = 64 * 16
TC_SCR_BYTES = -(-(64 * 33 * 4) // 16) * 16


def _r16(v):
    return -(-v // 16) * 16


def padded_dims(case):
    """(nl_d, nl_c, Kp, Np) as wb_tc_make pads them."""
    dens, col = case.dims()
    I = dens[:-1] + col[:-1]
    O_ = dens[1:] + col[1:]
    return len(dens) - 1, len(col) - 1, tuple(_r16(v) for v in I), tuple(_r16(v) for v in O_)


def tc_refuses(case):
    """wb_tc_make's descriptor checks on the decoders this file builds: a head of 2..16, widths <= 128."""
    dens, col = case.dims()
    return not 2 <= dens[-1] <= 16 or max(dens + col) > 128 or min(dens + col) < 1


def fwd_per_sm(Kp, Np):
    """The CTAs per SM that tc_fwd_kernel picks for a hash grid: from the forward's shared memory, which only the padded widths set."""
    maxw = max(Kp + Np)
    blob = _r16(sum(k * n * 2 + n * 32 for k, n in zip(Kp, Np)))
    smem = 2 * (maxw // 8 * TC_SLAB + TC_SCR_BYTES) + blob
    per_sm = max(1, min(3, TC_SMEM_MAX // (smem + 1024)))
    return min(per_sm, 2) if maxw > 64 else max(per_sm, 2)


def live_planes(case):
    """tc_dfeat's planes: one plane per live LOD ('cat'), one plane ('sum')."""
    if case.multiscale != "cat":
        return 1
    return case.L if case.lod_idx < 0 else max(0, min(case.lod_idx, case.L))


def nerf64_expected(case, backward):
    """What wb_rf_tc_shaped(desc, backward) reports: TcShapeNerf64::matches, plus tc_fwd_nerf64 (forward) or tc_bwd_fuses (backward,
    the last pass as bwd_plan / tc_bwd_passes plan it).  A descriptor the library refuses is not shaped."""
    if tc_refuses(case):
        return 0
    nd, nc, Kp, Np = padded_dims(case)
    if (nd, nc, Kp, Np) != (NERF64_ND, NERF64_NC, NERF64_KP, NERF64_NP):
        return 0
    if not backward:
        return int(max(Kp + Np) <= 64 and fwd_per_sm(Kp, Np) == 3)
    return int(case.F == 2 and case.multiscale == "cat" and live_planes(case) <= 16 and bwd_plan(case)[-1] == 2)


@pytest.fixture(scope="module")
def W():
    import wisp_b200
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return wisp_b200


def tc_shaped(W, desc, backward):
    v = C.c_int32(-1)
    W._cabi.lib().wb_rf_tc_shaped(desc, backward, C.addressof(v))
    return v.value


def shaped_or_refused(W, desc, backward):
    """wb_rf_tc_shaped, with a refused descriptor (WispB200Error) counted as not shaped: -> (shaped, error message or None)."""
    try:
        return tc_shaped(W, desc, backward), None
    except W._cabi.WispB200Error as e:
        return 0, str(e)


def host_desc(W, case, buf):
    """The descriptor of `case` for host-side calls only: every pointer is the small device buffer `buf` (nothing is launched)."""
    from wisp_b200 import ops
    res = O.geometric_resolutions(case.L, case.res_min, case.res_max) if case.L > 1 else [16]
    begin = O.table_layout(res, case.bw)
    dens, col = case.dims()
    lod = case.L if case.lod_idx < 0 else case.lod_idx
    spec = ops.NefSpec(resolutions=res, begin_idxes=[int(b) for b in begin], codebook_size=2 ** case.bw, feature_dim=case.F,
                       multiscale=case.multiscale, lod_idx=lod, pos_mode=case.pos[0], pos_freq=case.pos[1], view_mode=case.view[0],
                       view_freq=case.view[1], has_bias=case.bias, dens_dims=dens, col_dims=col)
    return spec.desc([buf[:case.F].view(1, case.F)], buf, buf)


# ---- 1. the sweep -------------------------------------------------------------------------------------------------------------
# classes of family members the sweep must find (section 2 below runs one or more of each); `fused`: the shaped backward runs
FAMILY_CLASSES = {
    "fused: hidden width below 64": (True, lambda c: min(c.dens_hidden + c.col_hidden) < 64),
    "fused: bias off": (True, lambda c: not c.bias),
    "fused: unequal colour hidden widths": (True, lambda c: len(set(c.col_hidden)) > 1),
    "fused: dout below 16": (True, lambda c: c.dout < 16),
    "fused: view embedding without the raw direction": (True, lambda c: c.view[0] == 2),
    "fused: lod_idx below L": (True, lambda c: live_planes(c) < c.L),
    "fused: L below 16 with a position embedding": (True, lambda c: c.L < 16 and c.pos[0] != 0),
    "fused: no position embedding, L below 16": (True, lambda c: c.L < 16 and c.pos[0] == 0),
    "forward only: F = 4 'cat'": (False, lambda c: c.F == 4 and c.multiscale == "cat"),
    "forward only: F = 8 'sum'": (False, lambda c: c.F == 8 and c.multiscale == "sum"),
    "forward only: F = 1 'cat'": (False, lambda c: c.F == 1 and c.multiscale == "cat"),
}


SWEEP_N, SWEEP_SEED = 3000, 20261018


def _sweep_case(rng, i):
    """A seeded descriptor: half of them drawn near the family (so every class gets members), half over the whole sweep range."""
    near = i % 2 == 0
    F = int(rng.choice([1, 2, 4, 8], p=[0.15, 0.55, 0.15, 0.15] if near else None))
    ms = "sum" if rng.random() < (0.15 if near else 0.5) else "cat"
    if near and ms == "cat":
        L = int(rng.integers(max(1, 17 // F - 2), max(2, 32 // F + 2)))
    else:
        L = int(rng.integers(1, 33))
    L = min(max(L, 1), 32)
    lod_idx = -1 if rng.random() < 0.6 else int(rng.integers(0, L + 1))
    pos = (0, 0) if rng.random() < (0.5 if near else 0.3) else (int(rng.integers(1, 4)), int(rng.integers(0, 5)))
    if near:
        view = [(3, 4), (3, 5), (2, 4), (3, 3), (2, 5), (1, 0), (0, 0)][int(rng.integers(0, 7))]
    else:
        view = (int(rng.integers(0, 4)), int(rng.integers(0, 7)))
    dout = int(rng.integers(1, 18))
    width = lambda: int(rng.integers(47, 67)) if not near else int(rng.choice([int(rng.integers(47, 67)), 64]))
    dens_hidden = [width() for _ in range(1 if rng.random() < 0.9 else 2)]
    col_hidden = [width() for _ in range(2 if rng.random() < 0.85 else int(rng.choice([0, 1])))]
    if near and col_hidden and rng.random() < 0.5:
        col_hidden = [col_hidden[0]] * len(col_hidden)
    return Case(f"sweep{i}", dens_hidden, col_hidden, dout=dout, L=L, F=F, multiscale=ms, lod_idx=lod_idx, pos=pos, view=view,
                bias=bool(rng.random() < 0.6))


def test_shaped_selection_sweep(W):
    """wb_rf_tc_shaped(desc, 0 / 1) equals the mirror on 3000 seeded descriptors: L 1..32, F 1 / 2 / 4 / 8, 'cat' / 'sum', lod_idx,
    position / view modes and frequencies, dout 1..17, hidden widths 47..66, bias on / off.  Host calls only."""
    rng = np.random.default_rng(SWEEP_SEED)
    buf = torch.zeros(64, dtype=torch.float32, device="cuda")
    found = {k: [0, 0] for k in FAMILY_CLASSES}                # members whose forward / fused backward is shaped
    totals = [0, 0]
    refusals = set()
    bad = []
    for i in range(SWEEP_N):
        c = _sweep_case(rng, i)
        desc, keep = host_desc(W, c, buf)
        family_geometry = padded_dims(c) == (NERF64_ND, NERF64_NC, NERF64_KP, NERF64_NP)
        for b in (0, 1):
            got, err = shaped_or_refused(W, desc, b)
            want = nerf64_expected(c, b)
            if err:
                refusals.add(err.split(": ", 1)[-1])
                if family_geometry and not tc_refuses(c):
                    bad.append((c, b, "refused", err))
            if got != want:
                bad.append((c, b, got, want))
        f0, f1 = nerf64_expected(c, 0), nerf64_expected(c, 1)
        totals[0] += f0; totals[1] += f1
        for k, (fused, pred) in FAMILY_CLASSES.items():
            if (f1 if fused else (f0 and not f1)) and pred(c):
                found[k][0] += f0; found[k][1] += f1
    assert not bad, bad[:5]
    print(f"TCREPORT sweep: {SWEEP_N} descriptors, shaped forward {totals[0]}, shaped fused backward {totals[1]}")
    for k, (nf, nb) in found.items():
        print(f"TCREPORT sweep class {k}: {nf} shaped forward, {nb} shaped fused backward")
    print("TCREPORT sweep refusals: " + " | ".join(sorted(refusals)))
    assert all(nf > 0 for nf, _ in found.values()), found
    assert all(nb > 0 for k, (_, nb) in found.items() if FAMILY_CLASSES[k][0]), found


# ---- 2. members of the family inside the interval reference ----------------------------------------------------------------
def _fam(name, **kw):
    kw.setdefault("view", (3, 4))
    kw.setdefault("L", 16)
    return Case(name, kw.pop("dens_hidden", [64]), kw.pop("col_hidden", [64, 64]), **kw)


FUSED_MEMBERS = [
    _fam("h56_nobias", dens_hidden=[56], col_hidden=[56, 56], bias=False),
    _fam("col52_64_dout9", col_hidden=[52, 64], dout=9, view=(3, 5)),
    _fam("dout2_view35", dout=2, view=(3, 5)),
    _fam("dout10_view24", dout=10, view=(2, 4)),
    _fam("L16_lod9", lod_idx=9),
    _fam("L16_lod1", lod_idx=1),
    _fam("L9_pos21", L=9, pos=(2, 1)),
    _fam("L12_pos21", L=12, pos=(2, 1)),
    _fam("L14_pos10", L=14, pos=(1, 0)),
    _fam("L15_nopos", L=15),
    _fam("bench_bw19", bw=19, res_min=16, res_max=2048),
    # res 16 at bitwidth 12: res^3 == 2^12, the first hashed level (rows = 2^bw) above dense levels 8..13
    _fam("res3_eq_T", bw=12, res_min=8, res_max=64),
]
FWD_MEMBERS = [
    _fam("F4cat_L8", L=8, F=4),
    _fam("F8sum_pos33", L=8, F=8, multiscale="sum", pos=(3, 3)),
    _fam("F1cat_L24", L=24, F=1),
]
CONTROLS = [
    _fam("ctl_h48", dens_hidden=[48], col_hidden=[48, 48]),
    _fam("ctl_h65", dens_hidden=[65], col_hidden=[65, 65]),
    _fam("ctl_in35", pos=(1, 0)),                          # 32 features + 3 = 35 -> Kp 48
]
MEMBERS = [(c, 1, 1) for c in FUSED_MEMBERS] + [(c, 1, 0) for c in FWD_MEMBERS] + [(c, 0, 0) for c in CONTROLS]


def three_tiles_per_group():
    """Samples for three tiles (and a partial fourth) per group of the decoder backward: one CTA of two groups per SM."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    return sms * 2 * 64 * 3 + 37


def _route_checks(s, report, rng, fused):
    """wb_rf_shade_bwd runs the fused backward (one decoder launch per pass) or the decoder backward and then the stand-alone scatter
    (one launch more), beside the per-ray rows; its table gradient lies inside the scatter bound of the planes the same decoder
    backward writes (run-time route: no extra rounding; fused: the fp32 dX, within 7/6 of the bound)."""
    c = s.c
    g = (rng.standard_normal((s.S, 4)) * 1e-2).astype(np.float32)
    scale_t = s.loss_scale(g)
    n0 = s.A.launch_count()
    _, _, gt = s.shade_bwd(g, scale_t)
    launched = s.A.launch_count() - n0
    assert launched == 1 + len(bwd_plan(c)) + (0 if fused else 1), (launched, bwd_plan(c), fused)
    report.append(f"shade_bwd launches {launched} ({'fused' if fused else 'stand-alone'} scatter)")
    if not fused:
        _, _, planes = s.decoder_bwd(g, scale_t)
        cen, rad = T.table_scatter_bound(planes, float(scale_t.item()), s.pos, s.table.shape[0], s.res, c.bw, s.lod_idx, c.multiscale)
        _check_inside("shade_bwd table_scatter", gt, cen, rad, report)


@pytest.mark.parametrize("S", ["700", "3tiles"])
@pytest.mark.parametrize("case, fwd, bwd", MEMBERS, ids=[m[0].name for m in MEMBERS])
def test_family_member_inside_interval_reference(W, case, fwd, bwd, S):
    n = 700 if S == "700" else three_tiles_per_group()
    case = Case(**{**case.__dict__, "S": n, "R": 40 if n < 1000 else 3000})
    assert nerf64_expected(case, 0) == fwd and nerf64_expected(case, 1) == bwd, "the case no longer has the geometry it names"
    s = Setup(W, case)
    assert tc_shaped(W, s.desc, 0) == fwd and tc_shaped(W, s.desc, 1) == bwd
    assert fusable(case) >= bool(bwd)
    report = [f"{case.name} S={n} shaped fwd={fwd} bwd={bwd}"]
    _forward_checks(s, report)
    rng = np.random.default_rng(case.seed + 7)
    _backward_checks(s, report, rng)
    _route_checks(s, report, rng, fused=fusable(case))
    print("TCREPORT " + " | ".join(report))


@pytest.mark.parametrize("case", [_fam("dout1_view35", dout=1, view=(3, 5)), _fam("ctl_dout17", dout=17)], ids=lambda c: c.name)
def test_head_width_outside_2_16_is_refused(W, case):
    """dout 1 with view (3, 5) pads to the family's geometry (colour input 0 + 33 -> 48) and dout 17 to a 32-wide head: the
    tensor-core path refuses both, naming the head width, so neither can reach a shaped (or run-time) tensor-core kernel untested."""
    buf = torch.zeros(64, dtype=torch.float32, device="cuda")
    desc, keep = host_desc(W, case, buf)
    L = W._cabi.lib()
    for b in (0, 1):
        with pytest.raises(W._cabi.WispB200Error, match="decoder_density output must be"):
            tc_shaped(W, desc, b)
        assert int(L.wb_rf_precision_supported(desc, 1, b)) == 0
    assert int(L.wb_rf_param_blob_floats(desc, 1)) <= 0
    assert "decoder_density output must be" in L.wb_last_error().decode()
    if case.dout < 2:
        assert padded_dims(case)[2:] == (NERF64_KP, NERF64_NP)
        assert int(L.wb_rf_param_blob_floats(desc, 0)) < 0                 # the fp32 decoders refuse it too
        assert ">= 2 wide" in L.wb_last_error().decode()


def _dropped_view_grad(s, g, X):
    """float64 |dL/d(colour input)| of the columns behind the density features, the ones the first colour layer's 16-wide data-grad
    chain computes and the backward drops (only the first dout - 1 columns are the density head's gradient)."""
    relu = lambda a: np.maximum(a, 0.0)
    dec, dout = s.dec, s.c.dout
    lin = lambda x, W, b: x @ W.astype(np.float64).T + (b.astype(np.float64) if b is not None else 0.0)
    h = X
    for l in range(len(dec.dens_W)):
        h = lin(h, dec.dens_W[l], dec.dens_b[l] if dec.dens_b else None)
        h = relu(h) if l < len(dec.dens_W) - 1 else h
    acts = [np.concatenate([h[:, 1:dout], s.view[0]], axis=1)]
    for l in range(len(dec.col_W)):
        a = lin(acts[-1], dec.col_W[l], dec.col_b[l] if dec.col_b else None)
        acts.append(relu(a) if l < len(dec.col_W) - 1 else a)
    sg = 1.0 / (1.0 + np.exp(-acts[-1]))
    dy = g[:, :3].astype(np.float64) * sg * (1.0 - sg) * float(s.loss_scale(g).item())
    for l in range(len(dec.col_W) - 1, 0, -1):
        dy = (dy @ dec.col_W[l].astype(np.float64)) * (acts[l] > 0)
    dx = dy @ dec.col_W[0].astype(np.float64)
    return np.abs(dx[:, dout - 1:15])


def test_dropped_view_gradient_stays_out_of_the_density_head(W):
    """The first colour layer's data-grad chain is 16 wide, so it also computes the gradient of the view-embedding columns behind the
    dout - 1 density features; the backward must drop those columns, not pass them on as dY of the density head's padded outputs.
    Dropping is only visible when they do not vanish on the way: here the raw-direction columns of that layer's weights are scaled by
    2^17 (the directions by 2^-18, so the forward stays the same size; the raw direction is exact in fp16, so the intervals stay tight)
    until the dropped columns exceed the fp16 range; an overflowing dY column times the zero padding of the density head's weights
    would be NaN in every density gradient."""
    case = Case(**{**SIZE_CASE.__dict__, "name": "view_gain", "dout": 9})
    rng = np.random.default_rng(47)
    R, S = 40, 700
    o = rng.uniform(-0.4, 0.4, (R, 3)).astype(np.float32)
    d = (_unit(rng.standard_normal((R, 3))) * np.float32(2.0 ** -18)).astype(np.float32)
    ray = np.sort(rng.integers(0, R, S)); ray[-1] = R - 1
    t = rng.uniform(0.0, 0.5, S)
    order = np.lexsort((t, ray))
    s = LayoutSetup(W, case, o, d, ray[order], t[order])
    s.dec.col_W[0][:, case.dout - 1:case.dout + 2] *= np.float32(2.0 ** 17)       # the raw direction: the first 3 view features
    s.dec.col_W[-1] *= np.float32(4.0)
    s.t_fc.copy_(torch.from_numpy(s.dec.flat()[1]).cuda())
    s.L.wb_rf_pack_params(s.desc, 1, s.A.ptr(s.blob), s.A.stream())
    torch.cuda.synchronize()
    assert tc_shaped(W, s.desc, 0) == 1 and tc_shaped(W, s.desc, 1) == 1 and fusable(s.c)
    report = [f"view_gain S={s.S}"]
    _forward_checks(s, report)
    g, X = _backward_checks(s, report, np.random.default_rng(48))
    over = float(np.mean(_dropped_view_grad(s, g, X).max(axis=1) > 65504.0))
    report.append(f"samples whose dropped columns exceed fp16: {over:.2f}")
    assert over > 0.05, over
    print("TCREPORT " + " | ".join(report))


# ---- 3. the shaped kernels at coordinate, run and tile edges ---------------------------------------------------------------
class LayoutSetup(Setup):
    """Setup with explicit rays and sample records: origins o [R, 3], directions d [R, 3], and per sample its ray (non-decreasing,
    the last sample on the last ray) and t (ordered within a ray)."""

    def __init__(self, W, c, o, d, ray, t):
        ray, t = np.asarray(ray, np.int32), np.asarray(t, np.float32)
        assert np.all(np.diff(ray) >= 0) and ray[-1] == len(o) - 1
        c = Case(**{**c.__dict__, "R": len(o), "S": len(t)})
        super().__init__(W, c)
        self.o, self.d = np.asarray(o, np.float32), np.asarray(d, np.float32)
        self.rec_ray, self.rec_t = ray, t
        self.pos = (self.o[ray].astype(np.float64) + self.d[ray].astype(np.float64) * t[:, None].astype(np.float64)).astype(np.float32)
        self.rays, self.rkeep = self.A.make_rays(torch.from_numpy(self.o).cuda(), torch.from_numpy(self.d).cuda(), 0.0, 1.0)
        self.t_rec_t, self.t_rec_ray = torch.from_numpy(self.rec_t).cuda(), torch.from_numpy(self.rec_ray).cuda()
        self.view = T.view_embedding(self.d[self.rec_ray], *c.view)


def _unit(v):
    v = np.asarray(v, np.float64)
    return (v / np.linalg.norm(v, axis=-1, keepdims=True)).astype(np.float32)


def _edge_coords(res):
    """Coordinates in [0, 1.5]: cell faces of the given resolutions (x = c * res / 2 + res / 2 an integer), 1 and its fp32
    neighbours, and points outside the cube from 1 + 2^-23 to 1.5."""
    out = {0.0, 1.0, float(np.nextafter(np.float32(1), np.float32(0))), 1.0 + 2.0 ** -23, 1.0 + 2.0 ** -22, 1.0001, 1.25, 1.5}
    for r in res:
        for k in range(r // 2, r + 1):
            out.add(float(np.float32((2.0 * k - r) / r)))
    return sorted(out)


def layout_faces(rng):
    """Axis-aligned rays through the origin (p = t d exactly) at every edge coordinate, and t = 0 samples at origins whose
    coordinates are edge coordinates of either sign."""
    res = O.geometric_resolutions(SIZE_CASE.L, SIZE_CASE.res_min, SIZE_CASE.res_max)
    ec = np.asarray(_edge_coords(sorted(set(res))[::3] + [res[-1]]), np.float32)
    o, d, ray, t = [], [], [], []
    for axis in range(3):
        for sign in (1.0, -1.0):
            v = np.zeros(3, np.float32); v[axis] = sign
            o.append(np.zeros(3, np.float32)); d.append(v)
            ray += [len(o) - 1] * len(ec); t += list(ec)
    n = 400
    pts = rng.choice(ec, (n, 3)) * rng.choice([-1.0, 1.0], (n, 3))
    pts[:8] = [[sx, sy, sz] for sx in (-1, 1) for sy in (-1, 1) for sz in (-1, 1)]         # the cube's corners
    pts[8:14] = [[1.5, 0, 0], [-1.5, 0, 0], [0, 1.5, 0], [0, -1.5, 0], [0, 0, 1.5], [0, 0, -1.5]]
    for p in pts.astype(np.float32):
        o.append(p); d.append(_unit(rng.standard_normal(3))); ray.append(len(o) - 1); t.append(0.0)
    return np.asarray(o), np.asarray(d), np.asarray(ray), np.asarray(t)


def layout_one_cell(rng, S):
    """One ray with S samples at the same t: every lane of every warp in one cell at every LOD."""
    o = rng.uniform(-0.4, 0.4, (1, 3)).astype(np.float32)
    return o, _unit(rng.standard_normal((1, 3))), np.zeros(S, np.int32), np.full(S, 0.3, np.float32)


def layout_runs(rng):
    """Rays of 2..40 samples at one t each, in shuffled order: runs of lanes in one cell that straddle the two 32-lane warps of a tile
    and the tiles."""
    lengths = rng.permutation(np.arange(2, 41))
    R = len(lengths)
    o = rng.uniform(-0.6, 0.6, (R, 3)).astype(np.float32)
    ray = np.repeat(np.arange(R), lengths).astype(np.int32)
    t = np.repeat(rng.uniform(0.0, 0.3, R), lengths).astype(np.float32)
    starts = np.concatenate([[0], np.cumsum(lengths)[:-1]])
    straddle = int(np.sum((starts // 32) != ((starts + lengths - 1) // 32)))
    assert straddle >= 10, straddle
    return o, _unit(rng.standard_normal((R, 3))), ray, t


def _layout_case(name, S):
    return Case(**{**SIZE_CASE.__dict__, "name": name, "S": S})


def _run_layout(W, name, o, d, ray, t, seed):
    s = LayoutSetup(W, _layout_case(name, len(t)), o, d, ray, t)
    assert tc_shaped(W, s.desc, 0) == 1 and tc_shaped(W, s.desc, 1) == 1 and fusable(s.c)
    report = [f"{name} S={s.S}"]
    _forward_checks(s, report)
    _backward_checks(s, report, np.random.default_rng(seed))
    print("TCREPORT " + " | ".join(report))
    return s


def test_edge_coordinates(W):
    """Samples at +-1, on cell faces of several LODs, just outside and up to 1.5 outside the cube: the saved X0 rows are fp16 of the
    clamped gather bit for bit and both scatters lie inside the bound of the same clamped cells."""
    o, d, ray, t = layout_faces(np.random.default_rng(41))
    s = _run_layout(W, "edge_coords", o, d, ray, t, 41)
    assert np.any(np.abs(s.pos) == 1.0) and np.any(np.abs(s.pos) > 1.0) and np.any(np.abs(s.pos) == np.float32(1 + 2.0 ** -23))


@pytest.mark.parametrize("S", [64 * 4 + 1, 64 * 4 + 31, 64 * 4 + 33, 64 * 4 + 63])
def test_one_cell_run(W, S):
    """Every sample in one cell: the warp run merging sums 32-lane runs, and the clamped lanes of the tail tile repeat the last
    sample's position (the scatter must not count them)."""
    o, d, ray, t = layout_one_cell(np.random.default_rng(S), S)
    _run_layout(W, f"one_cell_r{S % 64}", o, d, ray, t, S)


def test_runs_straddling_warps(W):
    o, d, ray, t = layout_runs(np.random.default_rng(43))
    _run_layout(W, "runs_2_40", o, d, ray, t, 43)


def _tile_counts():
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    per = sms * 2 * 64                                     # one tile for every group of the backward's grid
    return [2 * per + dd for dd in (-64, -1, 0, 1, 64)] + [per - 64 - 1]


@pytest.mark.parametrize("i", range(6))
def test_prefetch_tile_edges(W, i):
    """S = grid * 2 * 64 * 2 + d, d in {-64, -1, 0, 1, 64} (grid = SM count): the backward's next-tile prefetch lands exactly on, just
    before or just past the last tile of each group; the last count leaves the last group of the grid without a tile."""
    S = _tile_counts()[i]
    case = Case(**{**SIZE_CASE.__dict__, "name": f"tiles{i}", "S": S, "R": 3000})
    s = Setup(W, case)
    assert tc_shaped(W, s.desc, 0) == 1 and tc_shaped(W, s.desc, 1) == 1
    ntiles = -(-S // 64)
    report = [f"tiles S={S} ntiles={ntiles}"]
    _forward_checks(s, report)
    _backward_checks(s, report, np.random.default_rng(S))
    print("TCREPORT " + " | ".join(report))


def test_ray_rows_flag_before_shaped_shade_bwd(W):
    """wb_rf_workspace_holds_ray_rows(1) before wb_rf_shade_bwd of a shaped decoder: the fused backward reads the per-ray colour-input
    rows the previous call left in the workspace; the hint covers that call only, so a later call into a fresh workspace writes them."""
    s = Setup(W, _layout_case("rows_shaped", 700))
    assert tc_shaped(W, s.desc, 1) == 1
    rng = np.random.default_rng(5)
    X = T.f16(rng.standard_normal((s.S, s.dens_dims[0])) * 0.7)
    s.set_x0_rows(X.astype(np.float16))
    g = (rng.standard_normal((s.S, 4)) * 1e-2).astype(np.float32)
    scale = s.loss_scale(g)
    sc = float(scale.item())
    bw = T.Reference(s.dec, X, s.view).backward(g, sc, s.planes, 2, wgrad_n=s.wgrad_n())
    _, _, planes = s.decoder_bwd(g, scale)                  # writes the per-ray rows
    cen, rad = T.table_scatter_bound(planes, sc, s.pos, s.table.shape[0], s.res, s.c.bw, s.lod_idx, s.c.multiscale)
    report = ["rows_shaped"]

    def check(tag, got):
        gd, gc, gt = got
        _check_inside(f"{tag} grad_dens", gd, *bw["dens"], report)
        _check_inside(f"{tag} grad_col", gc, *bw["col"], report)
        _check_inside(f"{tag} table_scatter", gt, cen, rad * (7.0 / 6.0), report)
    L, A, p = s.L, s.A, s.A.ptr
    L.wb_rf_workspace_holds_ray_rows(1)
    check("rows held", s.shade_bwd(g, scale))
    gd, gc, gt = s.zeros_grads()
    L.wb_rf_workspace_holds_ray_rows(1)
    L.wb_rf_shade_bwd(s.desc, p(s.blob), 1, s.rays, p(s.t_rec_t), p(s.t_rec_ray), 0, p(gd), p(scale), p(s.feat), p(s.ws),
                      p(gt), p(gd), p(gc), A.stream())
    s.ws.fill_(0xFF)                                      # a fresh workspace: 0xFFFF is an fp16 NaN
    check("fresh", s.shade_bwd(g, scale))
    print("TCREPORT " + " | ".join(report))
