"""CPU tests of the AdamW / RMSprop steps' reference (tests/optim_reference.py), of the learning-rate schedule and of the host side
of wb_adamw_step / wb_rmsprop_step:
  - 20 steps of torch.optim.AdamW / RMSprop (CPU, foreach=False, fp32): from torch's state before every step the bit-exact
    emulation lands inside the float64 interval and torch's own result within three radii (torch rounds in another order: lerp
    for exp_avg, mul_ then addcmul_ for the second moments); with rounding off the interval function is torch in float64;
  - the emulation fed the gradients and learning rates of tests/golden/optim_groups.npz (the reference's init_optimizer groups
    and MultiStepLR under its SDFTrainer.step) reproduces the golden's parameters after every step;
  - the schedule against torch.optim.lr_scheduler.MultiStepLR (a repeated milestone and a milestone at iteration 1 included) and
    against the golden's recorded rates;
  - the refusal without a device, optimizer="sgd"."""
import os

import numpy as np
import pytest
import torch

import wisp_b200 as W

import optim_reference as OR

f32 = np.float32
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "optim_groups.npz")


def _inside(k, c, r, slack=1.0):
    return np.abs(np.asarray(k, np.float64) - c) <= slack * r


def _torch_run(make_opt, state_keys, n=513, steps=20, dtype=torch.float32, seed=0):
    """-> per step (state before, gradient, state after) of a torch optimiser over one tensor; state = (p, *state_keys)."""
    rng = np.random.default_rng(seed)
    p = torch.tensor(rng.standard_normal(n), dtype=dtype, requires_grad=True)
    opt = make_opt([p])
    out = []
    for t in range(steps):
        g = torch.tensor(rng.standard_normal(n) * 0.1, dtype=dtype)
        st = opt.state[p]
        before = [p.detach().numpy().copy()] + [st[k].numpy().copy() if k in st else np.zeros(n, p.detach().numpy().dtype) for k in state_keys]
        p.grad = g
        opt.step()
        st = opt.state[p]
        out.append((before, g.numpy().copy(), [p.detach().numpy().copy()] + [st[k].numpy().copy() for k in state_keys if k in st]))
    return out


@pytest.mark.parametrize("wd", [0.0, 1e-2])
def test_adamw_against_torch(wd):
    # betas that are fp32 numbers: 1 - beta is then the same formed in fp32 (the kernels, as wb_adam_kernel) and in double (torch);
    # 1 - fl32(0.999) differs from 0.001 by 1.3e-5 of it
    lr, b1, b2, eps = 1e-3, 0.875, 1.0 - 2.0 ** -9, 1e-8
    mk = lambda ps: torch.optim.AdamW(ps, lr=lr, betas=(b1, b2), eps=eps, weight_decay=wd, foreach=False)
    for t, ((p, m, v), g, after) in enumerate(_torch_run(mk, ("exp_avg", "exp_avg_sq")), 1):
        emu = OR.adamw_fp32(p, g, m, v, lr, wd, b1, b2, eps, t)
        for e, (c, r), a in zip(emu, OR.adamw(p, g, m, v, lr, wd, b1, b2, eps, t), after):
            assert _inside(e, c, r).all() and _inside(a, c, r, 3.0).all(), t
    for t, ((p, m, v), g, after) in enumerate(_torch_run(mk, ("exp_avg", "exp_avg_sq"), dtype=torch.float64), 1):
        for (c, r), a in zip(OR.adamw(p, g, m, v, lr, wd, b1, b2, eps, t, exact=True), after):
            assert r.max() == 0 and np.abs(c - a).max() <= 1e-12, t


@pytest.mark.parametrize("wd,momentum", [(0.0, 0.0), (1e-2, 0.0), (0.0, 0.9), (1e-2, 0.9)])
def test_rmsprop_against_torch(wd, momentum):
    lr, alpha, eps = 1e-2, 1.0 - 2.0 ** -6, 1e-8                 # an fp32 number, as test_adamw_against_torch's betas
    mk = lambda ps: torch.optim.RMSprop(ps, lr=lr, alpha=alpha, eps=eps, weight_decay=wd, momentum=momentum, foreach=False)
    keys = ("square_avg", "momentum_buffer")
    for (p, sq, buf), g, after in _torch_run(mk, keys):
        emu = OR.rmsprop_fp32(p, g, sq, buf, lr, wd, alpha, eps, momentum)
        ref = OR.rmsprop(p, g, sq, buf, lr, wd, alpha, eps, momentum)
        assert (emu[2] is None) == (ref[2] is None) == (momentum == 0.0)
        for e, cr, a in zip(emu, ref, after):
            if e is not None:
                assert _inside(e, cr[0], cr[1]).all() and _inside(a, cr[0], cr[1], 3.0).all()
    for (p, sq, buf), g, after in _torch_run(mk, keys, dtype=torch.float64):
        for cr, a in zip(OR.rmsprop(p, g, sq, buf, lr, wd, alpha, eps, momentum, exact=True), after):
            if cr is not None:
                assert cr[1].max() == 0 and np.abs(cr[0] - a).max() <= 1e-12


def test_decoupled_decay_is_not_l2():
    """AdamW's step lies outside the interval of Adam with the same weight decay as an L2 term, and the other way round."""
    import composite_reference as CR
    rng = np.random.default_rng(3)
    n, lr, wd, b1, b2, eps = 100003, 1e-3, 1e-2, 0.9, 0.999, 1e-8
    p, g = rng.standard_normal(n).astype(f32), rng.standard_normal(n).astype(f32)
    m, v = (rng.standard_normal(n) * 0.1).astype(f32), (rng.random(n) * 0.01).astype(f32)
    (wc, wr), _, _ = OR.adamw(p, g, m, v, lr, wd, b1, b2, eps, 2)
    (ac, ar), _, _ = CR.adam(p, g, m, v, lr, wd, b1, b2, eps, 2)
    assert not _inside(OR.adamw_fp32(p, g, m, v, lr, wd, b1, b2, eps, 2)[0], ac, ar).all()
    assert not _inside(CR.adam_fp32(p, g, m, v, lr, wd, b1, b2, eps, 2)[1], wc, wr).all()


@pytest.mark.parametrize("case", ["rmsprop", "rmsprop_m", "adamw"])
def test_emulation_reproduces_golden(case):
    """The emulation over the golden's gradients at the golden's learning rates, state carried in fp32 from zero: the reference's
    parameters after each of the 8 steps to 1e-6 of the tensor's largest entry."""
    G = np.load(GOLDEN)
    names = [str(n) for n in G[f"{case}_names"]]
    wd, eps, alpha, (b1, b2), mom = float(G["weight_decay"]), float(G["eps"]), float(G["alpha"]), G["betas"], float(G[f"{case}_momentum"])
    p = {n: G[f"{case}_init_{n}"] for n in names}
    s0 = {n: np.zeros_like(p[n]) for n in names}
    s1 = {n: np.zeros_like(p[n]) for n in names}
    worst = 0.0
    for t in range(1, int(G["steps"]) + 1):
        groups = OR.golden_groups(names, G[f"{case}_lrs"][t - 1], wd)
        for n in names:
            lr, w = groups[n]
            g = G[f"{case}_grad{t}_{n}"]
            if case == "adamw":
                p[n], s0[n], s1[n] = OR.adamw_fp32(p[n], g, s0[n], s1[n], lr, w, b1, b2, eps, t)
            else:
                p[n], s0[n], b = OR.rmsprop_fp32(p[n], g, s0[n], s1[n], lr, w, alpha, eps, mom)
                s1[n] = b if b is not None else s1[n]
            ref = G[f"{case}_step{t}_{n}"]
            err = float(np.abs(p[n] - ref).max() / np.abs(ref).max())
            worst = max(worst, err)
            assert err <= 1e-6, (t, n, err)
    print(f"OPTIM golden {case}: worst relative-to-max error {worst:.3g}")


@pytest.mark.parametrize("milestones", [(), (3,), (4, 6), (2, 2, 5), (1, 4), (0, 3), (5, 3)])
def test_schedule_is_multisteplr(milestones):
    lr0, gamma, steps = 1e-3, 0.333, 9
    p = torch.zeros(1, requires_grad=True)
    opt = torch.optim.SGD([p], lr=lr0)
    sch = torch.optim.lr_scheduler.MultiStepLR(opt, milestones=list(milestones), gamma=gamma)
    for t, mine in enumerate(OR.multistep_lrs(lr0, milestones, gamma, steps), 1):
        ref = opt.param_groups[0]["lr"]
        if 0 not in milestones:      # MultiStepLR never tests last_epoch == 0; the package counts every milestone <= t - 1
            assert abs(mine - ref) <= 1e-15 * ref, (t, mine, ref)
        assert W.trainers.multistep_factor(milestones, gamma, t) * lr0 == mine
        opt.step(); sch.step()


def test_schedule_is_the_goldens():
    """The reference's float milestones 4.0, 6.0 and 7.2 over 8 steps: the iterations that fire are 4 and 6."""
    G = np.load(GOLDEN)
    assert G["rmsprop_milestone_iters"].tolist() == [4.0, 6.0, 7.2]
    fire = [int(m) for m in G["rmsprop_milestone_iters"] if float(m).is_integer()]
    lr0, glw, gamma = float(G["lr"]), float(G["grid_lr_weight"]), float(G["gamma"])
    for case in ("rmsprop", "rmsprop_m", "adamw"):
        lrs = G[f"{case}_lrs"]
        for t in range(1, 9):
            f = W.trainers.multistep_factor(fire, gamma, t)
            assert np.allclose(lrs[t - 1], [lr0 * f, lr0 * glw * f, lr0 * f], rtol=1e-15, atol=0.0), (case, t)


@pytest.mark.skipif(torch.cuda.is_available(), reason="the refusal of a machine without a device")
def test_no_device_is_an_error():
    A = W._cabi
    t = [torch.zeros(8) for _ in range(4)]
    a, r = (A.AdamSegment * 1)(), (A.RMSpropSegment * 1)()
    for s in (a[0], r[0]):
        s.param, s.grad, s.numel, s.lr, s.weight_decay = t[0].data_ptr(), t[1].data_ptr(), 8, 1e-3, 0.0
    a[0].exp_avg, a[0].exp_avg_sq, r[0].square_avg = t[2].data_ptr(), t[3].data_ptr(), t[2].data_ptr()
    with pytest.raises(A.WispB200Error):
        A.lib().wb_adamw_step(a, 1, 0.9, 0.999, 1e-8, 1, 1.0, 1, None)
    with pytest.raises(A.WispB200Error):
        A.lib().wb_rmsprop_step(r, 1, 0.99, 1e-8, 0.0, 1.0, 1, None)
    assert torch.equal(t[0], torch.zeros(8))
    for opt in (W.NativeAdamW([(t[0], 1e-3, 0.0)]), W.NativeRMSprop([(t[0], 1e-3, 0.0)]), W.NativeRMSprop([(t[0], 1e-3, 0.0)], momentum=0.9)):
        with pytest.raises(A.WispB200Error):
            opt.step([t[1]])


def test_unknown_optimizer_is_a_value_error():
    with pytest.raises(ValueError):
        W.trainers._make_optimizer("sgd", [], (0.9, 0.999), 1e-8, 0.99, 0.0)
    o = W.OctreeAS.make_dense(2, device="cpu")
    g = W.HashGrid.from_geometric(o, 2, 4, 'cat', 0.1, 0.0, 10, 4, 32)
    nef = W.NeuralRadianceField(g, hidden_dim=16)
    with pytest.raises(ValueError):
        W.MultiviewStep(W.Pipeline(nef, W.PackedRFTracer('ray', 8)), optimizer="sgd")
    with pytest.raises(ValueError):          # the reference's non-integer product: a milestone that never fires is not passed
        W.MultiviewStep(W.Pipeline(nef, W.PackedRFTracer('ray', 8)), scheduler_milestones=(4.0, 7.2))
    assert W.MultiviewStep(W.Pipeline(nef, W.PackedRFTracer('ray', 8)), scheduler_milestones=(4.0, 6)).milestones == [4, 6]
    with pytest.raises(ValueError):
        W.NativeRMSprop([], momentum=-0.1)
