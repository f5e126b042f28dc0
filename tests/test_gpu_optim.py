"""The one-launch AdamW and RMSprop steps (wb_adamw_step / wb_rmsprop_step), their host classes and the optimiser / schedule
arguments of MultiviewStep and SDFStep, on the GPU:
  - through the C ABI both rules BIT-EXACT with tests/optim_reference.py's fp32 chain and inside its float64 interval: numel 0, 1,
    3, 4, 1 000 003, misaligned pointers (scalar path), weight decay on and off, grad_scale 0.5, zero_grad on and off, AdamW at steps
    1 and 1000, RMSprop with and without momentum; 64 segments and the refusals;
  - 5-step trajectories of NativeAdamW / NativeRMSprop against torch.optim on the device with init_optimizer's three groups;
  - a host running steps ahead of the stream;
  - MultiviewStep(optimizer=..., scheduler_milestones=(3,)) over a hash, an octree and a triplanar field against the package's
    autograd route stepped by the torch optimiser and MultiStepLR, with the library launch count of the "adam" step;
  - SDFStep(optimizer="rmsprop") against the reference trainer's own eight steps (tests/golden/optim_groups.npz);
  - the defaults take the steps optimizer="adam" takes, bit for bit."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

import optim_reference as OR

pytestmark = pytest.mark.gpu
f32 = np.float32
RULES = ("adamw", "rmsprop", "rmsprop_m")
B1, B2, ALPHA, MOM = 0.9, 0.999, 0.99, 0.9


@pytest.fixture(scope="module")
def W():
    import wisp_b200
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return wisp_b200


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _addr(t):
    """Address of t's first element; also for an empty view, whose data_ptr() torch reports as 0."""
    return 0 if t is None else t.untyped_storage().data_ptr() + t.storage_offset() * t.element_size()


def _seg(A, rule, p, g, s0, s1, lr, wd):
    s = A.AdamSegment() if rule == "adamw" else A.RMSpropSegment()
    s.param, s.grad, s.numel, s.lr, s.weight_decay = _addr(p), _addr(g), p.numel(), lr, wd
    names = ("exp_avg", "exp_avg_sq") if rule == "adamw" else ("square_avg", "momentum_buffer")
    setattr(s, names[0], _addr(s0)); setattr(s, names[1], _addr(s1) or None)
    return s


def _array(A, rule, n):
    return ((A.AdamSegment if rule == "adamw" else A.RMSpropSegment) * n)()


def _call(W, rule, segs, n, eps, step, gs, zero_grad, momentum=None):
    L, f = W._cabi.lib(), C.c_float
    if rule == "adamw":
        return L.wb_adamw_step(segs, C.c_int32(n), f(B1), f(B2), f(eps), C.c_int32(step), f(gs), C.c_int32(zero_grad), W._cabi.stream())
    mom = (MOM if rule == "rmsprop_m" else 0.0) if momentum is None else momentum
    return L.wb_rmsprop_step(segs, C.c_int32(n), f(ALPHA), f(eps), f(mom), f(gs), C.c_int32(zero_grad), W._cabi.stream())


def _emulate(rule, h, lr, wd, eps, step, gs):
    """-> (fp32 chain, interval) as lists over (p, s0, s1); s1 entries None for RMSprop without momentum."""
    if rule == "adamw":
        return OR.adamw_fp32(h["p"], h["g"], h["a"], h["b"], lr, wd, B1, B2, eps, step, gs), OR.adamw(h["p"], h["g"], h["a"], h["b"], lr, wd, B1, B2, eps, step, gs)
    mom = MOM if rule == "rmsprop_m" else 0.0
    return OR.rmsprop_fp32(h["p"], h["g"], h["a"], h["b"], lr, wd, ALPHA, eps, mom, gs), OR.rmsprop(h["p"], h["g"], h["a"], h["b"], lr, wd, ALPHA, eps, mom, gs)


# ---- the kernels through the C ABI ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("rule,step", [("adamw", 1), ("adamw", 1000), ("rmsprop", 1), ("rmsprop_m", 1)])
@pytest.mark.parametrize("zero_grad", [1, 0])
def test_segments_bit_exact(W, rule, step, zero_grad):
    """Every segment's parameters and state equal the fp32 chain bit for bit and lie inside the interval; the gradient is cleared
    or untouched; without momentum the second state tensor of RMSprop is not passed at all."""
    A = W._cabi
    rng = np.random.default_rng(step + zero_grad)
    eps, gs = 1e-8, 0.5
    plan = [(n, None, 1e-3, 0.0, 1.0) for n in (0, 1, 3, 4, 5, 7, 1000003)]      # (numel, misaligned operand, lr, wd, gradient scale)
    plan += [(1027 + k, which, 2e-3, 1e-2, 1.0) for k, which in enumerate("pgab")]
    plan += [(4099, None, 1e-3, 1e-2, 0.0), (4099, None, 1e-3, 0.0, 1e-14), (8, None, 5e-4, 1e-2, 1e3)]
    has_b = rule != "rmsprop"
    segs = _array(A, rule, len(plan))
    keep, host = [], []
    for i, (n, mis, lr, wd, scale) in enumerate(plan):
        h = dict(p=rng.standard_normal(n).astype(f32), g=(rng.standard_normal(n) * scale).astype(f32),
                 a=(rng.random(n) * 0.01 * max(scale, 1e-14) ** 2).astype(f32), b=(rng.random(n) * 0.01 * max(scale, 1e-14) ** 2).astype(f32))
        if rule == "adamw":
            h["a"] = (rng.standard_normal(n) * 0.1 * max(scale, 1e-14)).astype(f32)
        if rule == "rmsprop_m":
            h["b"] = (rng.standard_normal(n) * 0.5).astype(f32)
        t = {}
        for key, a in h.items():
            off = 1 if mis == key else 0
            buf = torch.zeros(n + 4, device="cuda")
            buf[off:off + n] = dev(a)
            t[key] = buf[off:off + n]
        segs[i] = _seg(A, rule, t["p"], t["g"], t["a"], t["b"] if has_b else None, lr, wd)
        keep.append(t); host.append(h)
    before = A.launch_count()
    A.check(_call(W, rule, segs, len(plan), eps, step, gs, zero_grad))
    assert A.launch_count() == before + 1
    torch.cuda.synchronize()
    for (n, mis, lr, wd, scale), t, h in zip(plan, keep, host):
        got = [t[x].cpu().numpy() for x in "pab"]
        emu, ivl = _emulate(rule, h, lr, wd, eps, step, gs)
        name = f"{rule} n={n} mis={mis} wd={wd} scale={scale} step={step}"
        for key, k, e, cr in zip("pab", got, emu, ivl):
            if e is None:
                assert np.array_equal(k, h["b"]), name             # momentum 0: the buffer is never written
                continue
            assert np.array_equal(k, e), (name, key, int((k != e).sum()))
            assert np.all(np.abs(k.astype(np.float64) - cr[0]) <= cr[1]), (name, key)
        assert np.array_equal(t["g"].cpu().numpy(), np.zeros(n, f32) if zero_grad else h["g"]), name


@pytest.mark.parametrize("rule", RULES)
def test_segment_count_and_refusals(W, rule):
    """64 segments in one launch; 65 segments, nseg 0, a null pointer, AdamW's step 0 and momentum > 0 without a buffer return
    WB_ERR_INVALID and launch nothing."""
    A = W._cabi
    segs = _array(A, rule, 65)
    ts = []
    for i in range(65):
        p = torch.full((i + 1,), float(i), device="cuda")
        t = (p, torch.ones_like(p), torch.zeros_like(p), torch.zeros_like(p) if rule != "rmsprop" else None)
        segs[i] = _seg(A, rule, *t, 1e-3, 0.0)
        ts.append(t)
    before = A.launch_count()
    assert _call(W, rule, segs, 65, 1e-8, 1, 1.0, 1) == -1
    assert _call(W, rule, segs, 0, 1e-8, 1, 1.0, 1) == -1
    assert _call(W, rule, None, 1, 1e-8, 1, 1.0, 1) == -1
    if rule == "adamw":
        assert _call(W, rule, segs, 64, 1e-8, 0, 1.0, 1) == -1
    if rule == "rmsprop":
        assert _call(W, rule, segs, 64, 1e-8, 1, 1.0, 1, momentum=0.9) == -1
        assert b"momentum" in A.lib().wb_last_error()
    bad = _array(A, rule, 1)
    bad[0] = _seg(A, rule, *ts[3], 1e-3, 0.0)
    bad[0].grad = None
    assert _call(W, rule, bad, 1, 1e-8, 1, 1.0, 1) == -1
    assert A.launch_count() == before
    A.check(_call(W, rule, segs, 64, 1e-8, 1, 1.0, 1))
    torch.cuda.synchronize()
    for i, (p, g, a, b) in enumerate(ts):
        pk = p.cpu().numpy()
        if i < 64:
            one = np.ones(i + 1, f32)
            emu, _ = _emulate(rule, dict(p=np.full(i + 1, i, f32), g=one, a=0 * one, b=0 * one), 1e-3, 0.0, 1e-8, 1, 1.0)
            assert np.array_equal(pk, emu[0]) and float(pk[0]) < i, i
        else:
            assert np.all(pk == i), i
        assert float(g.abs().max()) == (0.0 if i < 64 else 1.0)


# ---- the host classes against torch.optim -------------------------------------------------------------------------------------
def _torch_opt(rule, groups, lr, eps, momentum):
    if rule == "adamw":
        return torch.optim.AdamW(groups, lr=lr, betas=(B1, B2), eps=eps, weight_decay=0.0)
    return torch.optim.RMSprop(groups, lr=lr, alpha=ALPHA, eps=eps, momentum=momentum)


@pytest.mark.parametrize("rule", RULES)
def test_native_trajectory_is_torch(W, rule):
    """5 steps over init_optimizer's groups (decoder: weight decay; grid: lr * 5; rest) with gradients scaled by 0.5 against
    torch.optim on the device: parameters to 1e-6 of max."""
    torch.manual_seed(1)
    lr, wd, glw, eps = 1e-3, 1e-2, 5.0, 1e-8
    mom = MOM if rule == "rmsprop_m" else 0.0
    shapes = {"decoder": (64, 33), "grid": (40003, 2), "rest": (17,)}
    p0 = {k: torch.randn(s, device="cuda") for k, s in shapes.items()}
    grads = [{k: torch.randn(s, device="cuda") * 0.1 for k, s in shapes.items()} for _ in range(5)]
    ref = {k: v.clone().requires_grad_(True) for k, v in p0.items()}
    topt = _torch_opt(rule, [{"params": [ref["decoder"]], "lr": lr, "weight_decay": wd}, {"params": [ref["grid"]], "lr": lr * glw},
                             {"params": [ref["rest"]], "lr": lr}], lr, eps, mom)
    mine = {k: v.clone() for k, v in p0.items()}
    entries = [(mine["decoder"], lr, wd), (mine["grid"], lr * glw, 0.0), (mine["rest"], lr, 0.0)]
    opt = W.NativeAdamW(entries, betas=(B1, B2), eps=eps) if rule == "adamw" else W.NativeRMSprop(entries, alpha=ALPHA, eps=eps, momentum=mom)
    for g in grads:
        for k in shapes:
            ref[k].grad = g[k].clone()
        topt.step()
        gs = [(2.0 * g[k]).contiguous() for k in ("decoder", "grid", "rest")]
        opt.step(gs, grad_scale=0.5)
        assert all(float(x.abs().max()) == 0.0 for x in gs)
    for k in shapes:
        err = float((mine[k] - ref[k].detach()).abs().max() / ref[k].detach().abs().max())
        print(f"OPTIM trajectory {rule} {k}: {err:.3g} of max")
        assert err <= 1e-6, (k, err)


SLEEP_CYCLES = 500_000_000          # ~0.3 s of GPU time: the host issues every step before the first one runs


@pytest.mark.parametrize("rule", RULES)
def test_host_run_ahead(W, rule):
    """8 steps with their own gradients and a changing lr_scale issued behind a ~0.3 s sleep without a host sync equal the same 8
    steps with a sync after each: every launch carries its own description."""
    torch.manual_seed(0)
    shapes = [(4099,), (257, 3)]
    p0 = [torch.randn(s, device="cuda") for s in shapes]
    grads = [[torch.randn(s, device="cuda") for s in shapes] for _ in range(8)]

    def run(sync):
        ps = [p.clone() for p in p0]
        entries = [(p, 1e-3, 1e-2) for p in ps]
        opt = W.NativeAdamW(entries) if rule == "adamw" else W.NativeRMSprop(entries, momentum=MOM if rule == "rmsprop_m" else 0.0)
        gs = [[g.clone() for g in gg] for gg in grads]
        torch.cuda.synchronize()
        if not sync:
            torch.cuda._sleep(SLEEP_CYCLES)
        for t in range(8):
            opt.lr_scale = 0.5 ** t
            opt.step(gs[t], zero_grad=False)
            if sync:
                torch.cuda.synchronize()
        torch.cuda.synchronize()
        return ps

    for a, b in zip(run(True), run(False)):
        assert torch.equal(a, b), float((a - b).abs().max())


# ---- MultiviewStep ------------------------------------------------------------------------------------------------------------
def _rays(W, res):
    from oracle import oracle as O
    o, d = O.look_at_rays([-3.0, 0.65, -3.0], [0, 0, 0], res, res, 30.0)
    tgt = torch.sigmoid(torch.randn(o.shape[0], 3, generator=torch.Generator().manual_seed(3))).cuda()
    return W.Rays(dev(o), dev(d), 0.0, 10.0), tgt


def _field(W, kind):
    """A small NeRF field and its tracer, identical at every call: 'hash' | 'octree' | 'triplanar'."""
    from oracle import oracle as O
    torch.manual_seed(7)
    if kind == "hash":
        blas = W.OctreeAS.from_quantized_points(dev(O.lego_like_points(5)), 5)
        grid = W.HashGrid.from_geometric(blas, 2, 8, 'cat', 0.3, 0.0, 12, 8, 64)
        tr = W.PackedRFTracer('ray', 96, bg_color=(1.0, 1.0, 1.0))
    elif kind == "octree":
        blas = W.OctreeAS.from_quantized_points(dev(O.lego_like_points(5)), 5)
        grid = W.OctreeGrid(blas, feature_dim=8, num_lods=3, multiscale_type='sum', feature_std=0.3)
        tr = W.PackedRFTracer('ray', 96, bg_color=(1.0, 1.0, 1.0))
    else:
        grid = W.TriplanarGrid(W.AxisAlignedBBoxAS(device="cuda"), feature_dim=4, log_base_resolution=4, num_lods=3, multiscale_type='sum', feature_std=0.3)
        tr = W.PackedRFTracer('voxel', 32, bg_color=(1.0, 1.0, 1.0))
    nef = W.NeuralRadianceField(grid, view_embedder='positional', view_multires=4, hidden_dim=64, num_layers=1, bias=True).cuda()
    tr.precision = 0
    return nef, tr


@pytest.mark.parametrize("kind", ["hash", "octree", "triplanar"])
@pytest.mark.parametrize("optimizer", ["rmsprop", "adamw"])
def test_multiview_step_takes_the_configs_steps(W, kind, optimizer):
    """5 native steps at precision 0 with a milestone at iteration 3 against the package's autograd route stepped by the torch
    optimiser over init_optimizer's groups and MultiStepLR: losses 1e-4 relative; parameters 1e-3 of the tensor's max except
    entries whose gradient was ever below 1e-2 of max (both rules divide by the gradient's own magnitude, so there the two
    routes' rounding decides the step), those bounded by the steps' total length; one optimiser launch, the "adam" step's count."""
    A = W._cabi
    lr, wd, glw, gamma, steps = 2e-4, 1e-2, 5.0, 0.333, 5
    eps = 1e-8
    rays, tgt = _rays(W, 32)
    nef_a, tr_a = _field(W, kind)
    named = dict(nef_a.named_parameters())
    dec = [p for n, p in named.items() if "decoder" in n]
    grid = [p for n, p in named.items() if "decoder" not in n and "grid" in n]
    rest = [p for n, p in named.items() if "decoder" not in n and "grid" not in n]
    topt = _torch_opt(optimizer, [{"params": dec, "lr": lr, "weight_decay": wd}, {"params": grid, "lr": lr * glw}, {"params": rest, "lr": lr}], lr, eps, 0.0)
    sched = torch.optim.lr_scheduler.MultiStepLR(topt, milestones=[3], gamma=gamma)
    pipe_a = W.Pipeline(nef_a, tr_a)
    nef_b, tr_b = _field(W, kind)
    ms = W.MultiviewStep(W.Pipeline(nef_b, tr_b), lr=lr, eps=eps, weight_decay=wd, grid_lr_weight=glw, optimizer=optimizer, scheduler_milestones=(3,),
                         scheduler_gamma=gamma)
    assert ms.fused
    nef_c, tr_c = _field(W, kind)
    adam = W.MultiviewStep(W.Pipeline(nef_c, tr_c), lr=lr, eps=eps, weight_decay=wd, grid_lr_weight=glw)
    small = {n: torch.zeros_like(p, dtype=torch.bool) for n, p in named.items()}
    moved = 0.0
    for s in range(steps):
        topt.zero_grad()
        tr_a.seed = 40 + s
        rb = pipe_a(rays=rays, channels=["rgb"])
        loss_a = torch.nn.functional.smooth_l1_loss(rb.rgb, tgt, reduction='none').mean()
        loss_a.backward()
        for n, p in named.items():
            g = p.grad if p.grad is not None else torch.zeros_like(p)
            small[n] |= g.abs() < 1e-2 * g.abs().max()
        moved += topt.param_groups[1]["lr"] * (1.0 / (1.0 - ALPHA) ** 0.5 if optimizer == "rmsprop" else 1.0 / (1.0 - B1))
        topt.step(); sched.step()
        before = A.launch_count()
        loss_b = ms.step(rays, tgt, seed=40 + s)
        n_rule = A.launch_count() - before
        before = A.launch_count()
        adam.step(rays, tgt, seed=40 + s)
        assert n_rule == A.launch_count() - before, (s, n_rule)
        la = float(loss_a.detach())
        assert abs(float(loss_b) - la) <= 1e-4 * abs(la), (s, float(loss_b), la)
        assert ms.opt.lr_scale == (1.0 if s < 3 else gamma)
    assert ms.opt.t == steps
    worst = 0.0
    for n, pb in nef_b.named_parameters():
        pa, sm = named[n].detach(), small[n]
        d = (pa - pb.detach()).abs()
        if bool((~sm).any()):
            worst = max(worst, float(d[~sm].max() / pa.abs().max()))
        assert float(d.max()) <= 2.0 * moved + 1e-3 * float(pa.abs().max()), n
    print(f"OPTIM multiview {kind} {optimizer}: parameters {worst:.3g} of max")
    assert worst <= 1e-3


def test_multiview_step_default_is_adam(W):
    """MultiviewStep() and MultiviewStep(optimizer="adam") build the same NativeAdam and, from the same gradients, take bit-identical
    optimiser steps (the backward's atomic sums differ from run to run, so the gradients are set, not computed); a real step
    leaves lr_scale at 1 and update=False leaves the step count where it was."""
    rays, tgt = _rays(W, 32)
    out = []
    for kw in ({}, {"optimizer": "adam"}):
        nef, tr = _field(W, "hash")
        ms = W.MultiviewStep(W.Pipeline(nef, tr), lr=1e-3, eps=1e-8, weight_decay=1e-2, grid_lr_weight=5.0, **kw)
        assert type(ms.opt) is W.NativeAdam and ms.milestones == []
        gen = torch.Generator(device="cuda").manual_seed(5)
        bufs = ms.g_grid + [ms.g_dens, ms.g_col] + ms.g_rest
        for s in range(3):
            for b in bufs:
                b.copy_(torch.randn(b.shape, device="cuda", generator=gen))
            ms.opt.step(bufs)
        out.append(([p.detach().clone() for p in nef.parameters()], [(lr, wd) for _, lr, wd in ms.opt.entries]))
        ms.step(rays, tgt, seed=9)
        ms.step(rays, tgt, seed=20, update=False)
        assert ms.opt.t == 4 and ms.opt.lr_scale == 1.0
    assert out[0][1] == out[1][1]
    for a, b in zip(out[0][0], out[1][0]):
        assert torch.equal(a, b)


# ---- SDFStep ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", ["rmsprop", "rmsprop_m"])
def test_sdf_step_rmsprop_golden(W, golden_dir, case):
    """SDFStep(optimizer="rmsprop") over the reference trainer's eight steps, the recorded learning rates applied through
    lr_scale: 2 library launches per step (wb_sdf_train + the optimiser); after step 1 the entries whose gradient is above a
    tenth of the tensor's largest are the reference's to 5e-2 of the rule's largest first step, the group's lr / sqrt(1 - alpha)
    (the reference's gradients pass through fp16 features: 2e-2 of max, test_sdf_step_golden; the grid's gradients are of the
    size of eps, so the step follows their magnitude and not only their sign); after step 8 nine entries in ten of every tensor
    are the reference's to a tenth of the tensor's largest total movement, every entry within twice that movement."""
    A = W._cabi
    g = np.load(os.path.join(golden_dir, "optim_groups.npz"))
    lr, wd, glw, alpha, mom = float(g["lr"]), float(g["weight_decay"]), float(g["grid_lr_weight"]), float(g["alpha"]), float(g[f"{case}_momentum"])
    grid = W.OctreeGrid(W.OctreeAS(dev(g["octree"])), feature_dim=8, num_lods=3, multiscale_type='sum', feature_std=0.0)
    nef = W.NeuralSDF(grid, pos_embedder='none', position_input=True, hidden_dim=16, num_layers=1).cuda()
    with torch.no_grad():
        for n, p in nef.named_parameters():
            p.copy_(dev(g[f"{case}_init_{n}"]))
    with pytest.raises(ValueError):
        W.SDFStep(W.Pipeline(nef), optimizer="sgd")
    step = W.SDFStep(W.Pipeline(nef), lr=lr, eps=float(g["eps"]), weight_decay=wd, grid_lr_weight=glw, optimizer="rmsprop", alpha=alpha, momentum=mom)
    assert step.fused and type(step.opt) is W.NativeRMSprop and (step.opt.momentum_buffer is None) == (mom == 0.0)
    coords, sdf = dev(g["coords"]), dev(g["sdf"])
    lrs = g[f"{case}_lrs"]
    for t in range(1, 9):
        step.opt.lr_scale = float(lrs[t - 1][0]) / lr
        before = A.launch_count()
        step.step(coords, sdf)
        assert A.launch_count() - before == 2, t
        if t == 1:
            for n, p in nef.named_parameters():
                init, ref, ref_g, now = g[f"{case}_init_{n}"], g[f"{case}_step1_{n}"], g[f"{case}_grad1_{n}"], p.detach().cpu().numpy()
                lr_g, eff = (lr * glw, ref_g) if n.startswith("grid.") else (lr, ref_g + wd * init)
                big = np.abs(eff) > 1e-1 * np.abs(eff).max()
                assert big.any() and np.abs(ref - init)[big].min() > 0, n
                np.testing.assert_allclose(now[big], ref[big], atol=5e-2 * lr_g / np.sqrt(1.0 - alpha), err_msg=n)
    for n, p in nef.named_parameters():
        init, ref, now = g[f"{case}_init_{n}"], g[f"{case}_step8_{n}"], p.detach().cpu().numpy()
        move = float(np.abs(ref - init).max())
        d = np.abs(now - ref)
        frac = float((d <= 1e-1 * move).mean())
        print(f"OPTIM sdf golden {case} {n}: max {d.max() / move:.3g} of the movement, {frac:.4f} within 1e-1")
        assert frac >= 0.9 and d.max() <= 2.0 * move, n
