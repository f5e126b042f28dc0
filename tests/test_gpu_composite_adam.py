"""The compositing kernels, the image loss fused into the compositing backward and the one-launch Adam through the C ABI, against
the float64 interval reference tests/composite_reference.py: every output must lie in centre +- radius.

Covers what test_composite_vs_oracle and the trainer comparisons cannot resolve at their tolerances:
  - wb_composite_fwd / wb_composite_bwd over rays of 0, 1, 31, 32, 33, 63, 64, 65, 1024 and 2048 samples, warps with 1-5 and 32
    sampled rays, R = 1, R < 32, R not a multiple of 32, and SMs x 32 x 256 + 4099 rays (a second grid-stride pass); sigma 0,
    tau below 2^-25, opaque rays (T underflows), tau 1e4, delta 0; bg black, white and arbitrary; depth_out, g_depth and g_alpha
    null and set; hit; absmax bit-equal to max |g_shaded| (0 without samples); rows past S untouched;
  - wb_composite_bwd_loss: l2 / l1 / huber, the 'rays' and 'samples' denominators, d = 0 and +-1 exactly, rays without samples;
  - wb_adam_step: numel 0 .. 1 000 003, misaligned segments (scalar path), 64 segments and the ABI's refusals, grad_scale,
    weight decay with zero gradients, eps 1e-15 with tiny gradients, steps 1, 2 and 10 000, zero_grad off;
  - a host running steps ahead of the stream (NativeAdam, SDFStep) computes what a synchronised host computes;
  - MultiviewStep's l2 / l1 losses with both denominators against the autograd route.
Each interval check prints one CMPREPORT line: max|k - c| / r and the median radius."""
import ctypes as C

import numpy as np
import pytest
import torch

import composite_reference as CR

pytestmark = pytest.mark.gpu
f32 = np.float32
SENTINEL = 7.25


@pytest.fixture(scope="module")
def W():
    import wisp_b200
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return wisp_b200


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _sms():
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


def _check(name, k, c, r):
    k, c, r = (np.asarray(x, np.float64) for x in (k, c, r))
    d = np.abs(k - c)
    ok = d <= r
    ratio = float(np.max(np.where(r > 0, d / np.where(r > 0, r, 1.0), np.where(d > 0, np.inf, 0.0)), initial=0.0))
    print(f"CMPREPORT {name}: max|k-c|/r={ratio:.3g} median_r={float(np.median(r)) if r.size else 0.0:.3g}")
    bad = np.argwhere(~ok)
    assert ok.all(), (name, bad[:4].tolist(), k[tuple(bad[0])], c[tuple(bad[0])], r[tuple(bad[0])])


class _Bufs:
    def __init__(self, case):
        self.case = case
        self.R, self.S = case["n"].shape[0], int(case["offsets"][-1])
        self.sh, self.dp, self.dl = dev(case["shaded"]), dev(case["depth"]), dev(case["deltas"])
        self.off = dev(case["offsets"])


def _bg3(bg):
    return (C.c_float * 3)(*[float(x) for x in bg])


def _fwd(W, b, bg, with_depth=True):
    A = W._cabi
    rgb = torch.full((b.R, 3), SENTINEL, device="cuda")
    dout = torch.full((b.R,), SENTINEL, device="cuda") if with_depth else None
    alpha = torch.full((b.R,), SENTINEL, device="cuda")
    hit = torch.full((b.R,), 3, dtype=torch.uint8, device="cuda")
    A.lib().wb_composite_fwd(A.ptr(b.sh), A.ptr(b.dp), A.ptr(b.dl), A.ptr(b.off), b.R, _bg3(bg), A.ptr(rgb), A.ptr(dout),
                             A.ptr(alpha), A.ptr(hit), A.stream())
    return rgb, dout, alpha, hit


def _gsh(b):
    return torch.full((b.S + 40, 4), SENTINEL, device="cuda")


def _tail_ok(g, b):
    assert bool((g[b.S:] == SENTINEL).all()), "rows past S written"


def _bwd(W, b, bg, g_rgb, g_depth, g_alpha):
    A = W._cabi
    g = _gsh(b)
    absmax = torch.zeros(1, device="cuda")
    A.lib().wb_composite_bwd(A.ptr(b.sh), A.ptr(b.dp), A.ptr(b.dl), A.ptr(b.off), b.R, _bg3(bg), A.ptr(g_rgb),
                             A.ptr(g_depth), A.ptr(g_alpha), A.ptr(g), A.ptr(absmax), A.stream())
    _tail_ok(g, b)
    return g[:b.S], absmax


def _bwd_loss(W, b, bg, rgb_pred, target, loss_type, inv):
    A = W._cabi
    g = _gsh(b)
    absmax, loss = torch.zeros(1, device="cuda"), torch.zeros(1, device="cuda")
    A.lib().wb_composite_bwd_loss(A.ptr(b.sh), A.ptr(b.dp), A.ptr(b.dl), A.ptr(b.off), b.R, _bg3(bg), A.ptr(rgb_pred),
                                  A.ptr(target), loss_type, inv, A.ptr(g), A.ptr(absmax), A.ptr(loss), A.stream())
    _tail_ok(g, b)
    return g[:b.S], absmax, loss


def _absmax_ok(g, absmax):
    want = float(g.abs().max()) if g.numel() else 0.0
    assert float(absmax) == want, (float(absmax), want)


def _run_composite(W, name, case, bg, seed=1):
    b = _Bufs(case)
    fw = CR.forward(case["offsets"], case["shaded"], case["depth"], case["deltas"], bg)
    rgb, dout, alpha, hit = _fwd(W, b, bg, True)
    rgb2, _, alpha2, hit2 = _fwd(W, b, bg, False)
    assert torch.equal(rgb, rgb2) and torch.equal(alpha, alpha2) and torch.equal(hit, hit2)
    _check(f"{name} rgb", rgb.cpu().numpy(), fw.rgb, fw.rgb_r)
    _check(f"{name} depth", dout.cpu().numpy(), fw.depth, fw.depth_r)
    ak = alpha.cpu().numpy()
    _check(f"{name} alpha", ak, fw.alpha, fw.alpha_r)
    assert CR.hit_ok(fw.alpha, fw.alpha_r, hit.cpu().numpy(), ak).all() and int(hit.max()) <= 1
    rng = np.random.default_rng(seed)
    gr, gd, ga = rng.standard_normal((b.R, 3)).astype(f32), rng.standard_normal(b.R).astype(f32), rng.standard_normal(b.R).astype(f32)
    for label, gdv, gav in (("set", gd, ga), ("null", None, None)):
        g, absmax = _bwd(W, b, bg, dev(gr), None if gdv is None else dev(gdv), None if gav is None else dev(gav))
        bw = CR.backward(case["offsets"], case["shaded"], case["depth"], case["deltas"], bg, gr, gdv, gav)
        gk = g.cpu().numpy()
        _check(f"{name} g_rgb[{label}]", gk[:, :3], bw.g[:, :3], bw.r[:, :3])
        _check(f"{name} g_sigma[{label}]", gk[:, 3], bw.g[:, 3], bw.r[:, 3])
        _absmax_ok(g, absmax)


BGS = {"black": (0.0, 0.0, 0.0), "white": (1.0, 1.0, 1.0), "arb": (0.3, 0.6, 0.1)}


@pytest.mark.parametrize("regime", CR.REGIMES)
@pytest.mark.parametrize("bg", list(BGS))
def test_composite_regimes(W, regime, bg):
    """205 rays: every length of RAY_LENGTHS, then warps with 1-5 and 32 sampled rays (205 is not a multiple of 32)."""
    rng = np.random.default_rng(0)
    case = CR.make_case(CR.ray_lengths(205, rng), regime, seed=0)
    _run_composite(W, f"R205 {regime} {bg}", case, BGS[bg])


@pytest.mark.parametrize("n", [[0], [1], [31], [33], [2048], "R17", "empty"])
def test_composite_small_batches(W, n):
    """R = 1 with each ray kind, 17 rays (< 32), and 100 rays without samples (absmax stays 0)."""
    if n == "R17":
        n = CR.ray_lengths(17, np.random.default_rng(2))
    elif n == "empty":
        n = np.zeros(100, np.int64)
    case = CR.make_case(n, "mixed", seed=3)
    _run_composite(W, f"R{len(n)} n={int(np.max(n))}", case, BGS["arb"])


def _big_case(seed=4):
    """SMs x 32 x 256 + 4099 rays of 0-2 samples (the grid-stride loop's second pass), a few long rays among them."""
    rng = np.random.default_rng(seed)
    R = _sms() * 32 * 256 + 4099
    n = rng.integers(0, 3, R)
    n[[5, 1000, R - 4000, R - 1]] = [1024, 65, 2048, 33]
    return CR.make_case(n, "mixed", seed)


def test_composite_second_grid_stride_pass(W):
    _run_composite(W, "Rbig", _big_case(), BGS["arb"])


# ---- fused loss ---------------------------------------------------------------------------------------------------------------
def _targets(rgb_k, rng):
    """Targets with d = rgb - target exactly 0, +1 (rgb >= 0.5: rgb - 1 is exact) and -1 (where rgb + 1 is exact), the rest random."""
    tgt = (rgb_k + rng.uniform(-1.5, 1.5, rgb_k.shape)).astype(f32)
    pick = rng.integers(0, 4, rgb_k.shape)
    plus = (rgb_k + f32(1)).astype(f32)
    tgt = np.where(pick == 0, rgb_k, tgt)
    tgt = np.where((pick == 1) & (rgb_k >= 0.5), (rgb_k - f32(1)).astype(f32), tgt)
    tgt = np.where((pick == 2) & (plus - rgb_k == 1), plus, tgt)
    d = rgb_k - tgt
    assert (d == 0).any() and (d == 1).any() and (d == -1).any()
    return tgt.astype(f32)


@pytest.mark.parametrize("loss,denom,shape", [(l, d, "R205") for l in ("l2", "l1", "huber") for d in ("rays", "samples")]
                         + [("huber", "rays", "Rbig")])                   # one loss at scale: the loss value's atomics
def test_composite_bwd_loss(W, loss, denom, shape):
    case = _big_case() if shape == "Rbig" else CR.make_case(CR.ray_lengths(205, np.random.default_rng(0)), "mixed", seed=0)
    bg = BGS["arb"]
    b = _Bufs(case)
    rgb, _, _, _ = _fwd(W, b, bg, False)
    rgb_k = rgb.cpu().numpy()
    tgt = _targets(rgb_k, np.random.default_rng(6))
    inv = float(f32(1.0 / (3 * b.R) if denom == "rays" else 1.0 / max(b.S, 1)))
    t = CR.LOSS_TYPES[loss]
    g, absmax, lv = _bwd_loss(W, b, bg, rgb, dev(tgt), t, inv)
    gl = CR.loss_grad(rgb_k, tgt, t, inv)
    bw = CR.backward(case["offsets"], case["shaded"], case["depth"], case["deltas"], bg, gl)
    gk = g.cpu().numpy()
    name = f"{shape} {loss}/{denom}"
    _check(f"{name} g_rgb", gk[:, :3], bw.g[:, :3], bw.r[:, :3])
    _check(f"{name} g_sigma", gk[:, 3], bw.g[:, 3], bw.r[:, 3])
    _absmax_ok(g, absmax)
    c, r = CR.loss_value(rgb_k, tgt, t, inv, b.R, sms=_sms())
    _check(f"{name} loss", np.array([float(lv)]), np.array([c]), np.array([r]))


# ---- Adam ---------------------------------------------------------------------------------------------------------------------
def _adam_call(W, segs, n, b1, b2, eps, step, gs, zero_grad):
    return W._cabi.lib().wb_adam_step(segs, n, b1, b2, eps, step, gs, zero_grad, W._cabi.stream())


def _addr(t):
    """Address of t's first element; also for an empty view, whose data_ptr() torch reports as 0."""
    return t.untyped_storage().data_ptr() + t.storage_offset() * t.element_size()


def _seg(A, p, g, m, v, lr, wd):
    s = A.AdamSegment()
    s.param, s.grad, s.exp_avg, s.exp_avg_sq = _addr(p), _addr(g), _addr(m), _addr(v)
    s.numel, s.lr, s.weight_decay = p.numel(), lr, wd
    return s


@pytest.mark.parametrize("step", [1, 2, 10000])
@pytest.mark.parametrize("zero_grad", [1, 0])
def test_adam_segments(W, step, zero_grad):
    """Segments of numel 0, 1, 3, 4, 5, 7 and 1 000 003, the same with p / g / m / v one float off 16-byte alignment (scalar
    path), weight decay with zero gradients, tiny gradients at eps 1e-15, grad_scale 0.5: m and v bit-exact, p one of the two
    contractions of the last line, all inside the interval; g cleared or untouched."""
    A = W._cabi
    rng = np.random.default_rng(step)
    b1, b2, eps, gs = 0.9, 0.999, 1e-15, 0.5
    plan = []                                   # (numel, misaligned operand or None, lr, wd, gradient scale)
    for n in (0, 1, 3, 4, 5, 7, 1000003):
        plan.append((n, None, 1e-3, 0.0, 1.0))
    for k, which in enumerate("pgmv"):
        plan.append((1027 + k, which, 2e-3, 1e-2, 1.0))
    plan += [(4099, None, 1e-3, 1e-2, 0.0), (4099, None, 1e-3, 0.0, 1e-14), (8, None, 5e-4, 0.0, 1e3)]
    segs = (A.AdamSegment * len(plan))()
    keep, host = [], []
    for i, (n, mis, lr, wd, scale) in enumerate(plan):
        h = dict(p=rng.standard_normal(n).astype(f32), g=(rng.standard_normal(n) * scale).astype(f32),
                 m=(rng.standard_normal(n) * 0.1 * max(scale, 1e-14)).astype(f32), v=(rng.random(n) * 0.01 * max(scale, 1e-14) ** 2).astype(f32))
        t = {}
        for key, a in h.items():
            off = 1 if mis == key else 0
            buf = torch.zeros(n + 4, device="cuda")
            buf[off:off + n] = dev(a)
            t[key] = buf[off:off + n]
        segs[i] = _seg(A, t["p"], t["g"], t["m"], t["v"], lr, wd)
        keep.append(t); host.append(h)
    _adam_call(W, segs, len(plan), b1, b2, eps, step, gs, zero_grad)
    torch.cuda.synchronize()
    for (n, mis, lr, wd, scale), t, h in zip(plan, keep, host):
        pk, mk, vk, gk = (t[x].cpu().numpy() for x in "pmvg")
        p_sep, p_fma, m1, v1 = CR.adam_fp32(h["p"], h["g"], h["m"], h["v"], lr, wd, b1, b2, eps, step, gs)
        assert np.array_equal(mk, m1) and np.array_equal(vk, v1), (n, mis)
        assert np.all((pk == p_sep) | (pk == p_fma)), (n, mis)
        (pc, pr), (mc, mr), (vc, vr) = CR.adam(h["p"], h["g"], h["m"], h["v"], lr, wd, b1, b2, eps, step, gs)
        name = f"adam n={n} mis={mis} wd={wd} scale={scale} step={step}"
        if n:
            _check(name + " p", pk, pc, pr)
            _check(name + " m", mk, mc, mr)
            _check(name + " v", vk, vc, vr)
        assert np.array_equal(gk, np.zeros_like(gk) if zero_grad else h["g"]), name


def test_adam_segment_count_and_raised_refusals(W):
    """64 segments in one launch; 65 segments, nseg 0 and step 0 raise WispB200Error with WB_ERR_INVALID and launch nothing."""
    A = W._cabi
    segs = (A.AdamSegment * 65)()
    ts = []
    for i in range(65):
        p = torch.full((i + 1,), float(i), device="cuda")
        t = (p, torch.ones_like(p), torch.zeros_like(p), torch.zeros_like(p))
        segs[i] = _seg(A, *t, 1e-3, 0.0)
        ts.append(t)
    before = A.launch_count()
    for n, step in ((65, 1), (0, 1), (64, 0)):
        with pytest.raises(A.WispB200Error) as e:
            _adam_call(W, segs, n, 0.9, 0.999, 1e-8, step, 1.0, 1)
        assert e.value.status == -1
    assert A.launch_count() == before
    _adam_call(W, segs, 64, 0.9, 0.999, 1e-8, 1, 1.0, 1)
    torch.cuda.synchronize()
    for i, (p, g, m, v) in enumerate(ts):
        pk = p.cpu().numpy()
        if i < 64:                                          # step 1 with g = 1: a sign step of lr, in the kernel's fp32 chain
            one = np.ones(i + 1, f32)
            p_sep, p_fma, _, _ = CR.adam_fp32(np.full(i + 1, i, f32), one, 0 * one, 0 * one, 1e-3, 0.0, 0.9, 0.999, 1e-8, 1)
            assert np.all((pk == p_sep) | (pk == p_fma)) and abs(float(i) - float(pk[0]) - 1e-3) <= 1e-5, i
        else:                                               # segment 65 untouched
            assert np.all(pk == i), i
        assert float(g.abs().max()) == (0.0 if i < 64 else 1.0)


# ---- a host running ahead of the stream -----------------------------------------------------------------------------------
SLEEP_CYCLES = 500_000_000          # ~0.3 s of GPU time: the host issues every step before the first one runs


def test_native_adam_host_run_ahead(W):
    """8 NativeAdam steps, each with its own gradient tensors, issued behind a ~0.3 s sleep without a host sync, equal the same
    8 steps with a sync after each (every step reads its own bias corrections and gradients)."""
    torch.manual_seed(0)
    shapes = [(4099,), (257, 3)]
    p0 = [torch.randn(s, device="cuda") for s in shapes]
    grads = [[torch.randn(s, device="cuda") for s in shapes] for _ in range(8)]

    def run(sync):
        ps = [p.clone() for p in p0]
        opt = W.NativeAdam([(p, 1e-3, 0.0) for p in ps], betas=(0.9, 0.999), eps=1e-8)
        gs = [[g.clone() for g in gg] for gg in grads]
        torch.cuda.synchronize()
        if not sync:
            torch.cuda._sleep(SLEEP_CYCLES)
        for t in range(8):
            opt.step(gs[t], zero_grad=False)
            if sync:
                torch.cuda.synchronize()
        torch.cuda.synchronize()
        return ps

    for a, b in zip(run(True), run(False)):
        assert torch.equal(a, b), float((a - b).abs().max())


def test_sdf_step_host_run_ahead(W):
    """6 SDFStep steps at the config-3 shape issued behind a ~0.3 s sleep without a host sync against 6 steps with a sync after
    each, at test_sdf_step_trajectory's bounds: losses 1e-4 relative, parameters 1e-6 per 1e-3 of the group's learning rate except
    entries whose gradient was ever below 1e-4 of max."""
    from oracle import octree_grid as OG
    from gpu_util import sdf_nef_from_case
    lr, wd, glw, eps, steps = 1e-3, 1e-2, 5.0, 1e-15, 6
    case = OG.make_sdf_case(level=7, num_lods=6, feature_dim=16, hidden_dim=128, multiscale="sum", res=4, seed=11, feature_std=0.02)
    rng = np.random.default_rng(3)
    L = case["level"]; spc = case["spc"]
    pts = spc.points[spc.pyramid[1, L]: spc.pyramid[1, L] + spc.pyramid[0, L]].astype(np.float32)
    c = ((pts[rng.integers(0, pts.shape[0], 16384)] + rng.random((16384, 3)).astype(np.float32)) / (2.0 ** (L - 1)) - 1.0).astype(np.float32)
    coords = dev(c)
    gt = dev(((np.abs(c).sum(-1, keepdims=True) - 0.5) / np.sqrt(3.0)).astype(np.float32))

    def make():
        nef = sdf_nef_from_case(case)
        st = W.SDFStep(W.Pipeline(nef), lr=lr, eps=eps, weight_decay=wd, grid_lr_weight=glw)
        assert st.fused
        return st

    sync_step, ahead = make(), make()
    tensors = lambda st: [f.data for f in st._grid_tensors(st.nef.grid)] + [st.dec_flat]
    lrs = [lr * glw] * (len(tensors(sync_step)) - 1) + [lr]
    small = [torch.zeros_like(t, dtype=torch.bool) for t in tensors(sync_step)]
    loss_a = []
    for _ in range(steps):                      # what SDFStep.step does, with the gradients read before Adam consumes them
        loss_a.append(float(sync_step.step(coords, gt, update=False)))
        for s_, g in zip(small, sync_step.g_feats + [sync_step.g_dec]):
            s_ |= g.abs() < 1e-4 * g.abs().max()
        sync_step.opt.step(sync_step.g_feats + [sync_step.g_dec], grad_scale=1.0, zero_grad=True)
        torch.cuda.synchronize()
    torch.cuda.synchronize()
    torch.cuda._sleep(SLEEP_CYCLES)
    loss_b = [ahead.step(coords, gt) for _ in range(steps)]
    torch.cuda.synchronize()
    for s, (a, b) in enumerate(zip(loss_a, loss_b)):
        assert abs(float(b) - a) <= 1e-4 * abs(a), (s, float(b), a)
    for k, (ta, tb, sm, lr_g) in enumerate(zip(tensors(sync_step), tensors(ahead), small, lrs)):
        d = (ta - tb).abs()
        assert float(d[~sm].max()) <= 1e-6 * lr_g / 1e-3 if bool((~sm).any()) else True, k
        assert float(d.max()) <= 2 * lr_g * steps, k


# ---- MultiviewStep loss variants ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("loss", ["l2", "l1"])
@pytest.mark.parametrize("denom", ["rays", "samples"])
def test_multiview_step_loss_variants(W, loss, denom):
    """MultiviewStep's native route (the loss inside wb_composite_bwd_loss) against its autograd route for l2 / l1 and both
    denominators, at test_multiview_step_matches_autograd_step's precision-0 bounds: loss 1e-6, gradients 2e-3 of max."""
    from oracle import oracle as O
    from gpu_util import nef_from_oracle, packed_grads
    onef = O.make_nef(num_lods=8, codebook_bitwidth=14, min_res=8, max_res=128, hidden_dim=64, feature_std=0.3, seed=1)
    spc = O.octree_to_spc(O.points_to_octree(O.lego_like_points(5), 5))
    o, d = O.look_at_rays([-3.0, 0.65, -3.0], [0, 0, 0], 48, 48, 30.0)
    tgt = torch.sigmoid(torch.randn(o.shape[0], 3, generator=torch.Generator().manual_seed(3))).cuda()
    rays = W.Rays(torch.from_numpy(o).cuda(), torch.from_numpy(d).cuda(), 0.0, 10.0)
    nef_a, _ = nef_from_oracle(onef, spc)
    tr_a = W.PackedRFTracer('ray', 128, bg_color=(1.0, 1.0, 1.0)); tr_a.precision = 0; tr_a.seed = 21
    rb = W.Pipeline(nef_a, tr_a)(rays=rays, channels=["rgb"])
    l = torch.nn.functional.mse_loss(rb.rgb, tgt, reduction='none') if loss == "l2" else torch.abs(rb.rgb - tgt)
    loss_a = l.mean() if denom == "rays" else l.sum() / max(tr_a.get_prev_num_samples(), 1)
    loss_a.backward()
    gt, gd, gc = packed_grads(nef_a)
    nef_b, _ = nef_from_oracle(onef, spc)
    tr_b = W.PackedRFTracer('ray', 128, bg_color=(1.0, 1.0, 1.0)); tr_b.precision = 0
    ms = W.MultiviewStep(W.Pipeline(nef_b, tr_b), lr=1e-3, eps=1e-8, rgb_loss_type=loss, rgb_loss_denom=denom)
    assert ms.fused
    loss_b = ms.step(rays, tgt, seed=21, update=False)
    assert tr_b.get_prev_num_samples() == tr_a.get_prev_num_samples() > 0
    loss_a = float(loss_a.detach())
    assert abs(float(loss_b) - loss_a) <= 1e-6 * max(1.0, abs(loss_a))
    for mine, ref in ((ms.g_grid[0].cpu().numpy(), gt), (ms.g_dens.cpu().numpy(), gd), (ms.g_col.cpu().numpy(), gc)):
        assert np.abs(mine.reshape(-1) - ref.reshape(-1)).max() <= 2e-3 * np.abs(ref).max()
