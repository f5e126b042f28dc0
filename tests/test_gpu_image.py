"""GPU tests (-m gpu) of app/image natively (csrc/wb_image.cu) against tests/image_reference.py and the autograd route:
  - wb_hashgrid2d_fwd bit for bit against the fp32 emulation and wb_hashgrid2d_bwd inside its float64 interval, over F 2 / 4 / 8, 1 / 2 / 16
    LODs, bitwidths 8 / 12 / 19 / 22, res^2 == T, dense levels of res >= 258 at coordinates exactly +-1, coord_dim 2 and 3 tables,
    coordinates outside +-1, on cell lines and NaN, N = 1 and N = 2^20 + 3; guard rows between and after the levels show that no row
    outside a level is read or written;
  - ops.hashgrid (what install() patches into wisp.ops.grid) and HashGrid.interpolate on [N, 2] against the emulation;
  - wb_image_eval / wb_image_train inside the float64 intervals ('cat' / 'sum', lod below the finest, H 16 / 64 / 128, N from 1 to
    65 536 and three tiles per CTA, accumulation into non-zero buffers) and against the autograd route;
  - ImageStep: two native launches per step, a 5-step trajectory against autograd + torch.optim.AdamW with init_optimizer's groups and
    MultiStepLR, precision=1 against autograd under autocast, the fall-back of a two-hidden-layer field, and one fit of a procedural
    512^2 image (native and autograd on the same batches; prints an IMAGEFIT line with both PSNRs)."""

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

import image_reference as IR

f32 = np.float32


@pytest.fixture(scope="module")
def W():
    import wisp_b200
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return wisp_b200


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def special_coords(res_list, rng, n_random):
    one = f32(1.0)
    v = [0.0, -0.0, 1.0, -1.0, np.nextafter(one, f32(0)), np.nextafter(-one, f32(0)), np.nextafter(one, f32(2)), 1.7, -3.0, 1e30, np.nan]
    for r in res_list[:4]:
        v += [float(f32(2.0 * k / r - 1.0)) for k in (1, r // 3, r - 1)]            # cell lines
    v = np.array(v, f32)
    g = np.stack(np.meshgrid(v, v), -1).reshape(-1, 2)
    return np.concatenate([g, rng.uniform(-1.1, 1.1, (n_random, 2)).astype(f32)]).astype(f32)


def grid_desc(W, table_t, res, begin, bw, multiscale="cat"):
    return W._cabi.make_grid_desc(table_t, res, [int(b) for b in begin], 2 ** bw, multiscale)


HASH_CASES = [  # F, resolutions, bitwidth, coord_dim, N random
    (2, [16], 8, 3, 500),
    (4, [4, 16], 8, 2, 500),                           # res^2 == T on the second level
    (8, [7, 64], 12, 3, 500),                          # res^2 == T
    (2, [16, 20, 25, 32, 40, 50, 64, 80, 101, 128, 161, 203, 256, 322, 406, 512], 19, 3, 2000),
    (2, [258, 300, 724], 19, 2, 500),                  # dense, res >= 258: coordinates at +1 on the last cell
    (4, [258, 511, 1024, 2000], 22, 2, 500),
    (8, [258, 724], 22, 3, 500),
]


@pytest.mark.parametrize("F,res,bw,cd,nr", HASH_CASES)
def test_hashgrid2d_fwd_bwd(W, F, res, bw, cd, nr):
    rng = np.random.default_rng(F * 131 + bw)
    begin = IR.table_layout(res, bw, cd)
    table = rng.standard_normal((int(begin[-1]), F)).astype(f32)
    coords = special_coords(res, rng, nr)
    tt, ct = dev(table), dev(coords)                                # kept alive until the kernels have run
    desc = grid_desc(W, tt, res, begin, bw)
    L = len(res)
    out = torch.empty((coords.shape[0], L * F), dtype=torch.float32, device="cuda")
    W._cabi.lib().wb_hashgrid2d_fwd(W._cabi.ptr(ct), coords.shape[0], desc, W._cabi.ptr(out), W._cabi.stream())
    emu, cen, rad = IR.hashgrid2d_fwd(coords, table, res, bw, begin)
    got = out.cpu().numpy()
    assert np.array_equal(got.view(np.uint32), emu.view(np.uint32)), np.argwhere(got != emu)[:5]
    # backward, accumulated into a non-zero table gradient; some gradients zero (skipped)
    gf = rng.standard_normal((coords.shape[0], L * F)).astype(f32)
    gf[::7] = 0.0
    g0 = (rng.standard_normal(table.shape) * 0.1).astype(f32)
    gt, gft = dev(g0), dev(gf)
    W._cabi.lib().wb_hashgrid2d_bwd(W._cabi.ptr(ct), coords.shape[0], desc, W._cabi.ptr(gft),
                                    W._cabi.ptr(gt), W._cabi.stream())
    c, r, k = IR.hashgrid2d_bwd(coords, gf, g0, res, bw, begin)
    k_ = gt.cpu().numpy().astype(np.float64)
    assert np.all(np.abs(k_ - c) <= r), float((np.abs(k_ - c) - r).max())
    assert np.array_equal(k_[k == 0], g0.astype(np.float64)[k == 0])


def test_hashgrid2d_large_and_single(W):
    rng = np.random.default_rng(5)
    res, bw, F = [16, 64, 258, 1024], 19, 2
    begin = IR.table_layout(res, bw, 3)
    table = rng.standard_normal((int(begin[-1]), F)).astype(f32)
    tt = dev(table)
    desc = grid_desc(W, tt, res, begin, bw)
    for N in (1, 2 ** 20 + 3):
        coords = rng.uniform(-1.05, 1.05, (N, 2)).astype(f32)
        ct = dev(coords)
        out = torch.empty((N, len(res) * F), dtype=torch.float32, device="cuda")
        W._cabi.lib().wb_hashgrid2d_fwd(W._cabi.ptr(ct), N, desc, W._cabi.ptr(out), W._cabi.stream())
        emu, _, _ = IR.hashgrid2d_fwd(coords, table, res, bw, begin)
        assert np.array_equal(out.cpu().numpy(), emu)


@pytest.mark.parametrize("cd", [2, 3])
def test_hashgrid2d_rows_stay_inside_their_level(W, cd):
    """Levels laid out with 64 guard rows after each one.  Forward: guard rows hold NaN, so a read outside a level (even with weight 0)
    makes a feature NaN.  Backward: guard rows hold -0.0, which any add of +0.0 (a weight-0 corner) turns into +0.0."""
    res, bw, F, G = [16, 258, 400, 724], 19, 4, 64
    rows = [IR.level_rows(r, bw, cd) for r in res]
    begin = np.zeros(len(res) + 1, np.int64)
    for l, n in enumerate(rows):
        begin[l + 1] = begin[l] + n + G
    rng = np.random.default_rng(9)
    table = rng.standard_normal((int(begin[-1]), F)).astype(f32)
    guard = np.zeros(table.shape[0], bool)
    for l, n in enumerate(rows):
        guard[begin[l] + n:begin[l + 1]] = True
    table[guard] = np.nan
    coords = special_coords(res, rng, 3000)
    coords = coords[~np.isnan(coords).any(1)]
    edge = np.array([[1, 1], [-1, 1], [1, -1], [-1, -1], [1, 0.25], [0.25, 1]], f32)
    coords = np.concatenate([coords, edge])
    tt, ct = dev(table), dev(coords)
    desc = grid_desc(W, tt, res, begin, bw)
    out = torch.empty((coords.shape[0], len(res) * F), dtype=torch.float32, device="cuda")
    W._cabi.lib().wb_hashgrid2d_fwd(W._cabi.ptr(ct), coords.shape[0], desc, W._cabi.ptr(out), W._cabi.stream())
    assert torch.isfinite(out).all()
    g0 = np.zeros(table.shape, f32)
    g0[guard] = -0.0
    gt, gft = dev(g0), dev(np.ones((coords.shape[0], len(res) * F), f32))
    W._cabi.lib().wb_hashgrid2d_bwd(W._cabi.ptr(ct), coords.shape[0], desc, W._cabi.ptr(gft),
                                    W._cabi.ptr(gt), W._cabi.stream())
    k = gt.cpu().numpy()
    assert np.all(np.signbit(k[guard])) and np.all(k[guard] == 0)


def test_ops_hashgrid_2d_through_the_mirror(W):
    """ops.hashgrid (install()'s wisp.ops.grid.hashgrid) and HashGrid.interpolate on [N, 2]: the emulation, 'cat' zeroing from lod."""
    g = W.HashGrid.from_geometric(None, feature_dim=2, num_lods=6, multiscale_type='cat', feature_std=0.5, codebook_bitwidth=12,
                                  min_grid_res=8, max_grid_res=300).cuda()
    rng = np.random.default_rng(2)
    coords = rng.uniform(-1, 1, (4000, 2)).astype(f32)
    table = g.codebook.feats.detach().cpu().numpy()
    begin = g.codebook.begin_idxes.cpu().numpy()
    emu, _, _ = IR.hashgrid2d_fwd(coords, table, g.resolutions, 12, begin)
    raw = W.ops.hashgrid(dev(coords), 12, 5, g.codebook)
    assert np.array_equal(raw.detach().cpu().numpy(), emu)
    f = g.interpolate(dev(coords), 3).detach().cpu().numpy()
    want = emu.copy(); want[:, 3 * 2:] = 0
    assert np.array_equal(f, want)
    # backward through autograd equals the interval of the emulation
    c = dev(coords)
    g.codebook.feats.grad = None
    g.interpolate(c, 5).sum().backward()
    gf = np.ones((4000, 12), f32); gf[:, 10:] = 0
    cen, rad, _ = IR.hashgrid2d_bwd(coords, gf, np.zeros_like(table), g.resolutions, 12, begin)
    assert np.all(np.abs(g.codebook.feats.grad.cpu().numpy() - cen) <= rad)


# ---- ImageNeuralField -------------------------------------------------------------------------------------------------------
def make_field(W, F=2, L=16, bw=19, min_res=16, max_res=1024, ms='cat', H=64, num_layers=1, std=0.3, seed=0, cd=3):
    torch.manual_seed(seed)
    g = W.HashGrid.from_geometric(None, feature_dim=F, num_lods=L, multiscale_type=ms, feature_std=std, codebook_bitwidth=bw,
                                  min_grid_res=min_res, max_grid_res=max_res, coord_dim=cd)
    nef = W.ImageNeuralField(g, activation_type='relu', layer_type='linear', hidden_dim=H, num_layers=num_layers)
    return nef.cuda()


def field_arrays(nef):
    g = nef.grid
    params = torch.cat([p.detach().reshape(-1) for p in W_ops(nef)]).cpu().numpy()
    return (g.codebook.feats.detach().cpu().numpy(), params, g.resolutions, g.codebook_bitwidth, g.codebook.begin_idxes.cpu().numpy(),
            g.multiscale_type)


def W_ops(nef):
    d = nef.decoder
    return [d.layers[0].weight, d.layers[0].bias, d.lout.weight, d.lout.bias]


def inside(k, c, r, what):
    bad = np.abs(np.asarray(k, np.float64) - c) > r
    assert not bad.any(), (what, int(bad.sum()), float((np.abs(k - c) - r).max()))


EVAL_CASES = [  # F, L, ms, lod, H, N, max_res
    (2, 16, 'cat', None, 64, 4096, 1024),
    (2, 16, 'cat', 7, 16, 129, 1024),
    (4, 4, 'sum', None, 128, 127, 300),
    (8, 3, 'cat', 1, 64, 1, 64),
    (2, 8, 'sum', None, 16, 65536, 600),
]


@pytest.mark.parametrize("F,L,ms,lod,H,N,mr", EVAL_CASES)
def test_image_eval_inside_intervals(W, F, L, ms, lod, H, N, mr):
    nef = make_field(W, F=F, L=L, ms=ms, H=H, max_res=mr, seed=N)
    rng = np.random.default_rng(N)
    coords = rng.uniform(-1, 1, (N, 2)).astype(f32)
    coords[:min(N, 4)] = np.array([[1, 1], [-1, -1], [1, -1], [0, 0]], f32)[:min(N, 4)]
    table, params, res, bw, begin, _ = field_arrays(nef)
    lod_ = L - 1 if lod is None else lod
    before = W._cabi.launch_count()
    with torch.no_grad():
        rgb = nef.rgb(dev(coords), lod)
    torch.cuda.synchronize()
    assert W._cabi.launch_count() - before == 1                      # one launch: gather, embedding, decoder, sigmoid
    fw = IR.forward(coords, table, params, res, bw, begin, ms, lod_, H)
    inside(rgb.cpu().numpy(), fw["y"], fw["ry"], "rgb")
    ref = nef.rgb(dev(coords), lod)                                  # autograd route
    assert (ref.detach() - rgb).abs().max().item() < 1e-5


TRAIN_CASES = [  # F, L, ms, lod, H, N, max_res
    (2, 16, 'cat', None, 64, 4096, 1024),
    (2, 16, 'cat', 5, 16, 31, 512),
    (2, 16, 'cat', None, 64, 33, 1024),
    (4, 4, 'sum', None, 128, 129, 300),
    (8, 3, 'cat', 2, 64, 1, 64),
    (4, 6, 'cat', None, 16, 65536, 700),
]


def run_train(W, nef, coords, gt, lod, g_table=None, g_params=None):
    fd = W.ops.image_field(nef)
    assert fd is not None
    gt_t = torch.zeros_like(nef.grid.codebook.feats) if g_table is None else dev(g_table)
    gp_t = torch.zeros(sum(p.numel() for p in W_ops(nef)), device="cuda") if g_params is None else dev(g_params)
    loss = torch.zeros(1, device="cuda")
    before = W._cabi.launch_count()
    W.ops.image_train(fd, dev(coords), dev(gt), lod, gt_t, gp_t, loss)
    torch.cuda.synchronize()
    assert W._cabi.launch_count() - before == 1
    return float(loss), gt_t.cpu().numpy(), gp_t.cpu().numpy()


@pytest.mark.parametrize("F,L,ms,lod,H,N,mr", TRAIN_CASES)
def test_image_train_inside_intervals(W, F, L, ms, lod, H, N, mr):
    nef = make_field(W, F=F, L=L, ms=ms, H=H, max_res=mr, seed=N + 1)
    rng = np.random.default_rng(N + 1)
    coords = rng.uniform(-1, 1, (N, 2)).astype(f32)
    gt = rng.uniform(0, 1, (N, 3)).astype(f32)
    table, params, res, bw, begin, _ = field_arrays(nef)
    lod_ = L - 1 if lod is None else lod
    g0 = (rng.standard_normal(table.shape) * 1e-3).astype(f32) if N == 33 else None
    p0 = (rng.standard_normal(params.shape) * 1e-3).astype(f32) if N == 33 else None
    loss, gtab, gpar = run_train(W, nef, coords, gt, lod_, g0, p0)
    r = IR.train(coords, gt, table, params, res, bw, begin, ms, lod_, H, grad_table0=g0, grad_params0=p0)
    assert abs(loss - r["loss"]) <= r["rloss"]
    inside(gtab, r["gtable"], r["rgtable"], "table gradient")
    inside(gpar, r["gparams"], r["rgparams"], "decoder gradient")
    if g0 is None:                                                   # against the autograd route
        for p in nef.parameters():
            p.grad = None
        ref = torch.nn.functional.mse_loss(nef.rgb(dev(coords), lod_), dev(gt))
        ref.backward()
        agp = torch.cat([p.grad.reshape(-1) for p in W_ops(nef)]).cpu().numpy()
        agt = nef.grid.codebook.feats.grad.cpu().numpy()
        assert abs(loss - float(ref.detach())) <= 1e-5 * float(ref.detach())
        assert np.abs(agp - gpar).max() <= 1e-4 * np.abs(agp).max()
        assert np.abs(agt - gtab).max() <= 1e-4 * np.abs(agt).max()


def test_image_train_three_tiles_per_cta_and_empty_batch(W):
    nef = make_field(W, H=64, seed=11)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    N = 3 * 128 * sms                                                # 128-pixel tiles, one 130 KB CTA per SM: three tiles each
    rng = np.random.default_rng(3)
    coords = rng.uniform(-1, 1, (N, 2)).astype(f32)
    gt = rng.uniform(0, 1, (N, 3)).astype(f32)
    table, params, res, bw, begin, ms = field_arrays(nef)
    loss, gtab, gpar = run_train(W, nef, coords, gt, 15)
    r = IR.train(coords, gt, table, params, res, bw, begin, ms, 15, 64)
    assert abs(loss - r["loss"]) <= r["rloss"]
    inside(gtab, r["gtable"], r["rgtable"], "table gradient")
    inside(gpar, r["gparams"], r["rgparams"], "decoder gradient")
    fd = W.ops.image_field(nef)
    with pytest.raises(W.WispB200Error):
        W.ops.image_train(fd, torch.zeros((0, 2), device="cuda"), torch.zeros((0, 3), device="cuda"), 15,
                          torch.zeros_like(nef.grid.codebook.feats), torch.zeros(10, device="cuda"), torch.zeros(1, device="cuda"))
    with pytest.raises(W.WispB200Error):
        ct, out = dev(coords), torch.empty(3, device="cuda")
        W._cabi.lib().wb_image_eval(fd[0], 64, fd[2], 15, W._cabi.ptr(ct), 0,
                                    W._cabi.ptr(out), W._cabi.stream())


# ---- ImageStep --------------------------------------------------------------------------------------------------------------
APP = dict(lr=1e-3, eps=1e-16, weight_decay=1e-6, grid_lr_weight=500.0)


def torch_adamw(nef, lr, eps, weight_decay, grid_lr_weight, milestones, gamma=0.333):
    dec = [p for n, p in nef.named_parameters() if "decoder" in n and p.requires_grad]
    grid = [p for n, p in nef.named_parameters() if "decoder" not in n and "grid" in n and p.requires_grad]
    opt = torch.optim.AdamW([{"params": dec, "lr": lr, "eps": eps, "weight_decay": weight_decay},
                             {"params": grid, "eps": eps, "lr": lr * grid_lr_weight, "weight_decay": 0.0}], lr=lr, eps=eps)
    return opt, torch.optim.lr_scheduler.MultiStepLR(opt, milestones=milestones, gamma=gamma)


def test_image_step_two_launches_and_trajectory(W):
    nef = make_field(W, seed=21, std=0.05)
    ref = make_field(W, seed=21, std=0.05)
    ref.load_state_dict(nef.state_dict())
    step = W.ImageStep(W.Pipeline(nef), optimizer="adamw", scheduler_milestones=(3,), **{**APP, "grid_lr_weight": 10.0})
    assert step.fused
    opt, sched = torch_adamw(ref, APP["lr"], APP["eps"], APP["weight_decay"], 10.0, [3])
    rng = np.random.default_rng(4)
    for t in range(5):
        coords = dev(rng.uniform(-1, 1, (4096, 2)).astype(f32)); gt = dev(rng.uniform(0, 1, (4096, 3)).astype(f32))
        before = W._cabi.launch_count()
        loss = step.step(coords, gt)
        torch.cuda.synchronize()
        assert W._cabi.launch_count() - before == 2                  # wb_image_train + wb_adamw_step
        opt.zero_grad()
        rl = torch.nn.functional.mse_loss(ref.rgb(coords), gt)
        rl.backward(); opt.step(); sched.step()
        assert abs(float(loss) - float(rl)) <= 1e-4 * float(rl), (t, float(loss), float(rl))
    for (n, p), (_, q) in zip(nef.named_parameters(), ref.named_parameters()):
        d = (p.detach() - q.detach()).abs()
        if "decoder" in n:
            assert d.max().item() <= 2e-5, n
        else:
            assert d.median().item() <= 1e-6 and d.max().item() <= 2 * 5 * APP["lr"] * 10.0, n


def test_image_step_precision1_and_fallback(W):
    rng = np.random.default_rng(6)
    coords = dev(rng.uniform(-1, 1, (4096, 2)).astype(f32)); gt = dev(rng.uniform(0, 1, (4096, 3)).astype(f32))
    nef = make_field(W, seed=31)
    step = W.ImageStep(W.Pipeline(nef), precision=1, **APP)
    assert not step.fused
    loss = step.step(coords, gt, update=False)
    g16 = [p.grad.detach().clone() for p in W_ops(nef)] + [nef.grid.codebook.feats.grad.detach().clone()]
    for p in nef.parameters():
        p.grad = None
    with torch.autocast("cuda", torch.float16):
        ref = torch.nn.functional.mse_loss(nef.rgb(coords), gt)
    ref.backward()
    assert abs(float(loss) - float(ref)) <= 2e-3 * float(ref)
    for a, p in zip(g16, W_ops(nef) + [nef.grid.codebook.feats]):
        assert (a - p.grad).abs().max().item() <= 3e-2 * p.grad.abs().max().item()
    # two hidden layers: autograd + the native optimiser
    deep = make_field(W, seed=32, num_layers=2)
    sd = W.ImageStep(W.Pipeline(deep), **APP)
    assert not sd.fused
    w0 = deep.decoder.layers[1].weight.detach().clone()
    l0 = float(sd.step(coords, gt))
    for p in deep.parameters():
        p.grad = None
    with torch.no_grad():
        rgb = deep.rgb(coords)                                       # the kernel does not take it: the mirror body
    assert not torch.equal(w0, deep.decoder.layers[1].weight) and l0 > 0 and rgb.shape == (4096, 3)


def procedural_image(n):
    y, x = np.meshgrid(np.linspace(-1, 1, n), np.linspace(-1, 1, n), indexing="ij")
    r = 0.5 + 0.5 * np.sin(9 * x + 4 * y * y)
    g = 0.5 + 0.5 * np.cos(13 * np.hypot(x - 0.2, y + 0.1))
    b = ((np.floor(6 * (x + 1)) + np.floor(6 * (y + 1))) % 2) * 0.8 + 0.1
    img = np.stack([r, g, b], -1).astype(f32)
    coords = np.stack([x, y], -1).astype(f32)
    return coords.reshape(-1, 2), img.reshape(-1, 3)


def psnr(pred, gt):
    return float(-10 * torch.log10(((pred - gt) ** 2).mean()))


def test_image_step_fit_procedural_image(W):
    n, steps = 512, 2000
    coords, img = procedural_image(n)
    coords, img = dev(coords), dev(img)
    nef = make_field(W, F=2, L=16, bw=19, min_res=16, max_res=n // 2, std=1e-9, seed=41)
    ref = make_field(W, F=2, L=16, bw=19, min_res=16, max_res=n // 2, std=1e-9, seed=41)
    ref.load_state_dict(nef.state_dict())
    with torch.no_grad():
        p0 = psnr(nef.rgb(coords), img)
    step = W.ImageStep(W.Pipeline(nef), **APP)
    opt, _ = torch_adamw(ref, APP["lr"], APP["eps"], APP["weight_decay"], APP["grid_lr_weight"], [])
    gen = torch.Generator(device="cuda").manual_seed(0)
    for _ in range(steps):
        idx = torch.randint(0, n * n, (4096,), device="cuda", generator=gen)
        c, g = coords[idx], img[idx]
        step.step(c, g)
        opt.zero_grad()
        torch.nn.functional.mse_loss(ref.rgb(c), g).backward()
        opt.step()
    with torch.no_grad():
        pn, pa = psnr(nef.rgb(coords), img), psnr(ref.rgb(coords), img)
    print(f"IMAGEFIT {n}x{n} steps={steps}: initial {p0:.2f} dB, native {pn:.2f} dB, autograd {pa:.2f} dB")
    assert abs(pn - pa) <= 0.25 and pn >= p0 + 10 and pa >= p0 + 10


@pytest.mark.parametrize("name", ["cat3", "sum2"])
def test_image_step_reference_golden(W, name):
    """tests/golden/image_step.npz: the reference's own three ImageTrainer steps (AdamW groups of init_optimizer, MultiStepLR firing at
    iteration 2) replayed by ImageStep: step-1 gradients, the three losses and the parameters after step 3."""
    import os
    z = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "image_step.npz"))
    ms, F, cd = str(z[f"{name}_multiscale"]), int(z[f"{name}_feature_dim"]), int(z[f"{name}_coord_dim"])
    g = W.HashGrid.from_geometric(None, feature_dim=F, num_lods=4, multiscale_type=ms, feature_std=0.1, codebook_bitwidth=10,
                                  min_grid_res=4, max_grid_res=64, coord_dim=cd)
    assert g.resolutions == [int(r) for r in z[f"{name}_resolutions"]]
    nef = W.ImageNeuralField(g, activation_type='relu', layer_type='linear', hidden_dim=int(z["hidden_dim"]), num_layers=1)
    with torch.no_grad():
        for k, p in nef.named_parameters():
            if p.requires_grad:
                p.copy_(torch.from_numpy(z[f"{name}_init_{k}"]))
    nef = nef.cuda()
    step = W.ImageStep(W.Pipeline(nef), lr=float(z["lr"]), eps=float(z["eps"]), weight_decay=float(z["weight_decay"]),
                       grid_lr_weight=float(z["grid_lr_weight"]), optimizer="adamw", scheduler_milestones=tuple(int(m) for m in z["milestones"]),
                       scheduler_gamma=float(z["gamma"]))
    assert step.fused
    coords, rgb = dev(z["coords"]), dev(z["rgb"])
    step.step(coords, rgb, update=False)
    dec = ("decoder.layers.0.weight", "decoder.layers.0.bias", "decoder.lout.weight", "decoder.lout.bias")
    want = np.concatenate([z[f"{name}_grad1_{k}"].reshape(-1) for k in dec])
    assert np.abs(step.g_dec.cpu().numpy() - want).max() <= 1e-4 * np.abs(want).max()
    want = z[f"{name}_grad1_grid.codebook.feats"]
    assert np.abs(step.g_table.cpu().numpy() - want).max() <= 1e-4 * np.abs(want).max()
    step.zero_grads()
    losses = [float(step.step(coords, rgb)) for _ in range(3)]
    assert np.allclose(losses, z[f"{name}_losses"], rtol=1e-5, atol=0), (losses, z[f"{name}_losses"])
    for k, p in nef.named_parameters():
        if not p.requires_grad:
            continue
        d = np.abs(p.detach().cpu().numpy() - z[f"{name}_step3_{k}"])
        lr = float(z["lr"]) * (float(z["grid_lr_weight"]) if "grid" in k else 1.0)
        assert (d <= 1e-6).mean() >= 0.99 and d.max() <= 6 * lr, (k, float(d.max()), float((d <= 1e-6).mean()))
