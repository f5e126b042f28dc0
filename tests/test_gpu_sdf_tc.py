"""SDFStep(precision=1) on the GPU: the tensor-core training step (wb_sdf_train_tc) against the package's autograd route under
torch.autocast("cuda", torch.float16) -- the reference's enable_amp arithmetic -- on the same field, its accumulate-into semantics,
its launch count, its loss scale under large residuals, the autocast autograd route of the fields it does not take, and the
unchanged default.  Tolerances: loss 2e-3 relative, gradients 3e-2 of their max (the precision-1 bounds of DESIGN section 2)."""
import math

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def W():
    import wisp_b200
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return wisp_b200


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


_CASE = {}


def _case():
    from oracle import octree_grid as OG
    if not _CASE:
        _CASE["c"] = OG.make_sdf_case(level=7, num_lods=6, feature_dim=16, hidden_dim=128, multiscale="sum", res=4, seed=11, feature_std=0.02)
    return _CASE["c"]


# name: (grid, F, multiscale, num_lods, pos_embedder, position_input, H, hidden layers)
SHAPES = {
    "config3":    ("octree", 16, "sum", 6, "none", True, 128, 1),        # app/nglod nglod_octree.yaml: 19-128-1
    "octcat_pos": ("octree", 8, "cat", 6, "positional", True, 64, 1),    # 'cat' with a positional embedding, in 75
    "deep":       ("octree", 16, "sum", 6, "none", True, 128, 2),        # 19-128-128-1
    "h30":        ("octree", 4, "sum", 6, "none", False, 30, 1),         # H padded to 32
    "wide":       ("octree", 16, "cat", 6, "positional", True, 128, 1),  # in 3 + 24 + 96 = 123 -> K 128
    "in132":      ("octree", 21, "cat", 5, "positional", True, 32, 1),   # in 3 + 24 + 5 * 21 = 132 -> K 144
    "h96":        ("octree", 4, "sum", 6, "none", True, 96, 1),          # Hp 96: the second weight-gradient pass covers outputs 64..127
    "h80_deep":   ("octree", 16, "sum", 6, "none", True, 80, 2),         # Hp 80, two hidden layers
    "hash_cat8":  ("hash", 8, "cat", 4, "none", True, 128, 1),           # nglod_hash.yaml shape (scaled table)
    "hash_sum4":  ("hash", 4, "sum", 4, "none", True, 64, 2),
}


def _field(W, shape, seed=0):
    kind, F, ms, L, pe, pin, H, nh = SHAPES[shape]
    torch.manual_seed(seed)
    blas = W.OctreeAS(dev(_case()["octree"]))
    if kind == "hash":
        grid = W.HashGrid.from_geometric(blas, feature_dim=F, num_lods=L, multiscale_type=ms, feature_std=0.1, codebook_bitwidth=14,
                                         min_grid_res=16, max_grid_res=256)
    else:
        grid = W.OctreeGrid(blas, feature_dim=F, num_lods=L, multiscale_type=ms, feature_std=0.05)
    nef = W.NeuralSDF(grid, pos_embedder=pe, pos_multires=4, position_input=pin, hidden_dim=H, num_layers=nh).cuda()
    with torch.no_grad():                                                 # both relu sides populated
        for l in nef.decoder.layers:
            l.bias.uniform_(-0.3, 0.3)
    return nef


def _points(n, seed=5):
    case = _case()
    rng = np.random.default_rng(seed)
    spc, L = case["spc"], case["level"]
    pts = spc.points[spc.pyramid[1, L]: spc.pyramid[1, L] + spc.pyramid[0, L]].astype(np.float32)
    nn = (n + 1) // 2
    near = (pts[rng.integers(0, pts.shape[0], nn)] + rng.random((nn, 3)).astype(np.float32)) / (2.0 ** (L - 1)) - 1.0
    c = np.concatenate([near, rng.uniform(-1.05, 1.05, (n - nn, 3))]).astype(np.float32)[:n]
    gt = ((np.abs(c).sum(-1, keepdims=True) - 0.5) / np.sqrt(3.0)).astype(np.float32)
    return dev(c), dev(gt)


def _names(nef):
    return [n for n, p in nef.named_parameters() if p.requires_grad]


def _step_grads(nef, step):
    """{parameter name: gradient} of a fused step: grid tensors in order, then the flat decoder buffer in parameter order."""
    out, grid = {}, [n for n in _names(nef) if not n.startswith("decoder.")]
    for n, t in zip(grid, step.g_feats):
        out[n] = t
    o = 0
    for n, p in nef.named_parameters():
        if n.startswith("decoder."):
            out[n] = step.g_dec[o:o + p.numel()].view_as(p); o += p.numel()
    return {k: v.detach().double().cpu().numpy() for k, v in out.items()}


def _kernel(W, nef, coords, gt, lods):
    """ops.sdf_train(precision=1) (wb_sdf_train_tc) over the field's own tensors into fresh buffers -> (loss, {name: gradient})."""
    fd = W.ops.sdf_field(nef)
    feats = W.SDFStep._grid_tensors(nef.grid)
    g_feats = [torch.zeros_like(f.data) for f in feats]
    dparams = W.ops.decoder_params(nef.decoder)
    g_dec = torch.zeros(sum(p.numel() for p in dparams), dtype=torch.float32, device="cuda")
    loss = torch.zeros(1, dtype=torch.float32, device="cuda")
    c, g = coords.reshape(-1, 3).contiguous(), gt.reshape(-1).contiguous()
    for lod in lods:
        W.ops.sdf_train(fd, c, g, lod, 1.0 / c.shape[0], g_feats, g_dec, loss, precision=1)
    out, grid = {}, [n for n in _names(nef) if not n.startswith("decoder.")]
    for n, t in zip(grid, g_feats):
        out[n] = t
    o = 0
    for n, p in nef.named_parameters():
        if n.startswith("decoder."):
            out[n] = g_dec[o:o + p.numel()].view_as(p); o += p.numel()
    return float(loss), {k: v.detach().double().cpu().numpy() for k, v in out.items()}


def _autocast_autograd(nef, coords, gt, lods, scaled=True):
    """The reference's enable_amp step: autograd under torch.autocast(fp16).  scaled: with the kernel's power-of-two loss scale on
    the backward (loss * scale, gradients / scale, as a GradScaler does); the reference's unscaled fp16 dpred = 2 (y - gt) / N is
    subnormal below |y - gt| ~ 2 N 2^-14 / 2, which at N = 65 536 is most residuals, and its grid gradients are then off by more
    than the fp16 arithmetic both sides share (DESIGN section 2)."""
    N = coords.shape[0]
    scale = 2.0 ** -math.frexp(1.0 / N)[1] if scaled else 1.0
    while True:                         # as a GradScaler backs off: the fp16 batch sums of the weight gradients must stay finite
        for p in nef.parameters():
            p.grad = None
        with torch.autocast("cuda", torch.float16):
            loss = 0.0
            for lod in lods:
                loss = loss + ((nef(coords=coords, lod_idx=lod, channels="sdf") - gt) ** 2).sum()
            loss = loss / N
        (loss * scale).backward()
        grads = {n: (p.grad.detach().double().cpu().numpy() / scale if p.grad is not None else np.zeros(tuple(p.shape)))
                 for n, p in nef.named_parameters() if p.requires_grad}
        if not scaled or scale < 1.0 or all(np.isfinite(g).all() for g in grads.values()):
            return float(loss.detach()), grads
        scale /= 16.0


def _compare(loss, got, ref_loss, ref, what):
    assert np.isfinite(loss) and abs(loss - ref_loss) <= 2e-3 * abs(ref_loss), (what, loss, ref_loss)
    worst = 0.0
    for n, r in ref.items():
        err = np.abs(got[n] - r).max() / max(np.abs(r).max(), 1e-30)
        worst = max(worst, err)
        assert np.isfinite(got[n]).all() and err <= 3e-2, (what, n, err)
    print(f"{what}: loss rel {abs(loss - ref_loss) / abs(ref_loss):.2e}, worst gradient err / max {worst:.2e}")


@pytest.mark.parametrize("shape", list(SHAPES))
def test_tc_kernel_vs_autocast_autograd(W, shape):
    """wb_sdf_train_tc at 65 536 samples against autograd under torch.autocast on the same field."""
    nef = _field(W, shape)
    coords, gt = _points(65536)
    lods = [nef.grid.num_lods - 1]
    loss, got = _kernel(W, nef, coords, gt, lods)
    ref_loss, ref = _autocast_autograd(nef, coords, gt, lods)
    _compare(loss, got, ref_loss, ref, shape)


@pytest.mark.parametrize("shape", ["hash_cat8", "hash_sum4", "config3", "deep"])
def test_tc_step_route(W, shape):
    """SDFStep(precision=1) trains hash fields with wb_sdf_train_tc (its gradients are the kernel's) and octree fields by autograd
    under autocast (the kernel is slower there, DESIGN section 7)."""
    nef = _field(W, shape)
    step = W.SDFStep(W.Pipeline(nef), precision=1)
    assert step.precision == 1 and step.fused == (SHAPES[shape][0] == "hash")
    coords, gt = _points(4096, seed=2)
    loss = float(step.step(coords, gt, update=False))
    if step.fused:
        k_loss, k = _kernel(W, nef, coords, gt, step.loss_lods)
        got = _step_grads(nef, step)
        assert abs(loss - k_loss) <= 1e-6 * abs(k_loss)
        for n, v in k.items():
            assert np.abs(got[n] - v).max() <= 1e-5 * max(np.abs(v).max(), 1e-30), n


@pytest.mark.parametrize("N", [1, 63, 64, 65, 1000, 3 * 64 * 132 * 3 + 17])
@pytest.mark.parametrize("shape", ["config3", "deep"])
def test_tc_step_batch_sizes(W, shape, N):
    """Partial tiles, one tile, tiles straddling CTAs and several tiles per CTA."""
    nef = _field(W, shape, seed=1)
    coords, gt = _points(N, seed=N)
    lods = [nef.grid.num_lods - 1]
    loss, got = _kernel(W, nef, coords, gt, lods)
    ref_loss, ref = _autocast_autograd(nef, coords, gt, lods)
    _compare(loss, got, ref_loss, ref, f"{shape} N={N}")


def test_tc_step_all_lods(W):
    nef = _field(W, "config3", seed=2)
    coords, gt = _points(65536, seed=7)
    lods = list(range(nef.grid.num_lods))
    loss, got = _kernel(W, nef, coords, gt, lods)
    ref_loss, ref = _autocast_autograd(nef, coords, gt, lods)
    _compare(loss, got, ref_loss, ref, "all LODs")


def test_tc_accumulates_and_empty_batch(W):
    """wb_sdf_train_tc adds into non-zero buffers (a second call doubles them), and N = 0 leaves everything untouched."""
    nef = _field(W, "hash_sum4", seed=3)
    step = W.SDFStep(W.Pipeline(nef), precision=1)
    assert step.fused
    coords, gt = _points(4096, seed=3)
    c, g = coords.reshape(-1, 3).contiguous(), gt.reshape(-1).contiguous()
    lod = nef.grid.num_lods - 1
    W.ops.sdf_train(step.fd, c, g, lod, 1.0 / 4096, step.g_feats, step.g_dec, step.loss_buf, precision=1)
    once = [t.clone() for t in step.g_feats + [step.g_dec, step.loss_buf]]
    W.ops.sdf_train(step.fd, c, g, lod, 1.0 / 4096, step.g_feats, step.g_dec, step.loss_buf, precision=1)
    for a, b in zip(once, step.g_feats + [step.g_dec, step.loss_buf]):
        torch.testing.assert_close(b, 2 * a, rtol=1e-5, atol=1e-6 * float(a.abs().max()))
    before = [t.clone() for t in step.g_feats + [step.g_dec, step.loss_buf]]
    W.ops.sdf_train(step.fd, c[:0], g[:0], lod, 1.0, step.g_feats, step.g_dec, step.loss_buf, precision=1)
    for a, b in zip(before, step.g_feats + [step.g_dec, step.loss_buf]):
        assert torch.equal(a, b)
    with pytest.raises(W._cabi.WispB200Error):
        W.ops.sdf_train(step.fd, c, g, lod, 1.0 / 4096, step.g_feats, step.g_dec, step.loss_buf, precision=2)


def test_tc_step_launch_count(W):
    """An only_last precision-1 step is two library launches: wb_sdf_train_tc and wb_adam_step."""
    nef = _field(W, "hash_cat8")
    step = W.SDFStep(W.Pipeline(nef), precision=1)
    assert step.fused
    coords, gt = _points(512)
    step.step(coords, gt)
    before = W._cabi.launch_count()
    step.step(coords, gt)
    assert W._cabi.launch_count() - before == 2
    torch.cuda.synchronize()


def test_tc_step_large_residuals(W):
    """Residuals near 1e3 at N = 512 and 65 536: the loss-scaled fp16 dY stays finite, and so does everything it feeds."""
    for N in (512, 65536):
        for shape in ("deep", "hash_sum4"):
            nef = _field(W, shape, seed=4)
            coords, gt = _points(N, seed=11)
            lods = [nef.grid.num_lods - 1]
            loss, got = _kernel(W, nef, coords, gt + 1e3, lods)
            assert np.isfinite(loss) and loss > 1e5
            assert all(np.isfinite(v).all() for v in got.values())
            ref_loss, ref = _autocast_autograd(nef, coords, gt + 1e3, lods)
            _compare(loss, got, ref_loss, ref, f"{shape} residual 1e3, N={N}")


def _torch_adam(nef, lr, wd, glw, eps):
    dec, grd, rest = [], [], []
    for n, p in nef.named_parameters():
        if p.requires_grad:
            (dec if "decoder" in n else grd if "grid" in n else rest).append(p)
    return torch.optim.Adam([{"params": dec, "lr": lr, "eps": eps, "weight_decay": wd}, {"params": grd, "eps": eps, "lr": lr * glw},
                             {"params": rest, "eps": eps, "lr": lr}], lr=lr, eps=eps)


def test_tc_step_trajectory(W):
    """Five precision-1 steps against autocast autograd + torch.optim.Adam with init_optimizer's groups: losses 3e-2 relative at
    every step; parameters within 3 learning-rate steps of each other per step (bias-corrected Adam steps exceed lr where
    the fp16 differences of small gradients change their sign) and, where the gradient stays above 0.3 of its max, within half a step per step."""
    lr, wd, glw, eps, steps = 1e-3, 1e-2, 5.0, 1e-15, 5
    nef, ref_nef = _field(W, "hash_sum4", seed=5), _field(W, "hash_sum4", seed=5)
    step = W.SDFStep(W.Pipeline(nef), lr=lr, eps=eps, weight_decay=wd, grid_lr_weight=glw, precision=1)
    opt = _torch_adam(ref_nef, lr, wd, glw, eps)
    coords, gt = _points(65536, seed=3)
    small = {n: np.zeros(tuple(p.shape), bool) for n, p in ref_nef.named_parameters()}
    for s in range(steps):
        loss = float(step.step(coords, gt))
        ref_loss, grads = _autocast_autograd(ref_nef, coords, gt, step.loss_lods)
        opt.step()
        assert abs(loss - ref_loss) <= 3e-2 * abs(ref_loss), (s, loss, ref_loss)      # after Adam steps on differently rounded gradients
        for n, gr in grads.items():
            small[n] |= np.abs(gr) < 0.3 * np.abs(gr).max()        # 3e-2 of max is at most a 10 % error here: same Adam sign
    ref_p = dict(ref_nef.named_parameters())
    for n, p in nef.named_parameters():
        d = np.abs(p.detach().cpu().numpy() - ref_p[n].detach().cpu().numpy())
        lr_g = lr * (glw if n.startswith("grid.") else 1.0)
        assert d.max() <= 3 * lr_g * steps, n
        assert d[~small[n]].max(initial=0.0) <= 0.5 * lr_g * steps, n


@pytest.mark.parametrize("kind", ["triplanar", "hash_f2", "deep3x128", "octree"])
def test_tc_step_autocast_fallback(W, kind):
    """Fields outside wb_sdf_train_tc take autograd under torch.autocast(fp16) + NativeAdam: one step matches autocast autograd +
    torch.optim.Adam to 1e-6."""
    lr, wd, glw, eps = 1e-3, 1e-2, 5.0, 1e-15
    nets = []
    for _ in range(2):
        torch.manual_seed(3)
        blas = W.OctreeAS(dev(_case()["octree"]))
        nh, H = 1, 64
        if kind == "triplanar":
            grid = W.TriplanarGrid(blas, feature_dim=4, log_base_resolution=5, num_lods=1, multiscale_type='sum', feature_std=0.01)
        elif kind == "hash_f2":
            grid = W.HashGrid.from_geometric(blas, feature_dim=2, num_lods=8, multiscale_type='cat', feature_std=0.01, codebook_bitwidth=14,
                                             min_grid_res=16, max_grid_res=256)
        else:
            grid = W.OctreeGrid(blas, feature_dim=16, num_lods=6, multiscale_type='sum', feature_std=0.05)
            nh, H = (3, 128) if kind == "deep3x128" else (1, 128)
        nets.append(W.NeuralSDF(grid, pos_embedder='positional', pos_multires=4, position_input=True, hidden_dim=H, num_layers=nh).cuda())
    nef, ref_nef = nets
    step = W.SDFStep(W.Pipeline(nef), lr=lr, eps=eps, weight_decay=wd, grid_lr_weight=glw, precision=1)
    assert not step.fused and step.precision == 1
    if kind == "deep3x128":
        assert W.ops.sdf_field(nef) is not None and W.ops.sdf_train_tc_smem_bytes(W.ops.sdf_field(nef)) < 0
    opt = _torch_adam(ref_nef, lr, wd, glw, eps)
    coords, gt = _points(4096, seed=4)
    loss = float(step.step(coords, gt))
    ref_loss, _ = _autocast_autograd(ref_nef, coords, gt, [ref_nef.grid.num_lods - 1], scaled=False)
    opt.step()
    assert abs(loss - ref_loss) <= 1e-6 * abs(ref_loss)
    ref_p = dict(ref_nef.named_parameters())
    for n, p in nef.named_parameters():
        np.testing.assert_allclose(p.detach().cpu().numpy(), ref_p[n].detach().cpu().numpy(), atol=1e-6, err_msg=n)


def test_default_precision_unchanged_under_autocast(W):
    """SDFStep() keeps the fp32 kernels inside an autocast region: its gradients equal a second SDFStep() run outside autocast
    bit for bit, and precision values other than 0 and 1 are refused."""
    nef = _field(W, "config3", seed=6)
    coords, gt = _points(8192, seed=6)
    step = W.SDFStep(W.Pipeline(nef))
    assert step.fused and step.precision == 0
    l0 = step.step(coords, gt, update=False)
    g0 = [t.clone() for t in step.g_feats + [step.g_dec]]
    step.zero_grads()
    with torch.autocast("cuda", torch.float16):
        l1 = step.step(coords, gt, update=False)
    g1 = step.g_feats + [step.g_dec]
    # the same kernel, same inputs: equal up to the order of its atomic additions
    assert abs(float(l0) - float(l1)) <= 1e-6 * abs(float(l0))
    for a, b in zip(g0, g1):
        torch.testing.assert_close(a, b, rtol=1e-5, atol=1e-6 * float(a.abs().max()))
    for bad in (2, -1, True):
        with pytest.raises(ValueError):
            W.SDFStep(W.Pipeline(nef), precision=bad)


# ---------------------------------------------------------------------------------------------------------------
# the kernel inside the float64 fp16-faithful intervals (tests/sdf_tc_reference.py)
# ---------------------------------------------------------------------------------------------------------------
# octree: tests/sdf_shapes.py / sdf_deep_shapes.py fields (+ H 96 over config 3's grid); hash: this module's fields
INTERVAL_SHAPES = ["config3", "sum_pos3", "cat_id", "fast_h30", "widest", "l2_h128", "l2_h64", "h96", "hash_cat8", "hash_sum4"]


def _interval_field(W, name, seed=1):
    """-> (reference field, nef, points(n, seed) -> (coords, gt) numpy)."""
    import sdf_deep_shapes as DS
    import sdf_hash_reference as HR
    import sdf_shapes as SS
    from oracle import sdf_reference as S
    from test_gpu_sdf_kernels import nef_of
    if name.startswith("hash"):
        nef = _field(W, name, seed)
        g = nef.grid
        layers = list(nef.decoder.layers) + [nef.decoder.lout]
        field = HR.hash_field(g.codebook.feats.detach().cpu().numpy(), g.codebook.begin_idxes.tolist(), g.resolutions, g.codebook_bitwidth,
                              g.multiscale_type, [l.weight.detach().cpu().numpy() for l in layers], [l.bias.detach().cpu().numpy() for l in layers], 1, 0)

        def pts(n, s):
            c, t = _points(n, s)
            return c.cpu().numpy(), t.cpu().numpy()[:, 0]
        return field, nef, pts
    if name == "h96":
        level, nl, F, ms, pm, pf, H, layers, half = SS.SHAPES["config3"]
        case = SS.case_of(level, nl, F, ms)
        rng = np.random.default_rng(seed)
        feats = [(rng.standard_normal(f.shape) * 0.05).astype(np.float32) for f in case["feats"]]
        Ws, bs = S.random_decoder(rng, 3 + F, pm, 96, 1, scale=0.2)
        field = S.Field(case["spc"], case["trinkets"], feats, case["active_lods"][0], ms, Ws, bs, pm, pf, half)
    elif name in DS.DEEP_SHAPES:
        field, case = DS.make_field(name, seed=seed)
    else:
        field, case = SS.make_field(name, seed=seed)
    return field, nef_of(W, field, case), lambda n, s: SS.points(case, n, seed=s)


def _inside(k, c, r, what):
    k, c, r = np.asarray(k, np.float64), np.asarray(c, np.float64), np.asarray(r, np.float64)
    err = np.abs(k - c)
    assert (err <= r).all(), (what, float((err - r).max()), float(np.abs(c).max()))
    q = err[r > 0] / r[r > 0]
    return float(q.max(initial=0.0)), float(np.median(r[r > 0])) if (r > 0).any() else 0.0


@pytest.mark.parametrize("N", [1, 63, 64, 65, 1000, "tiles3", 65536])
@pytest.mark.parametrize("name", INTERVAL_SHAPES)
def test_tc_kernel_inside_intervals(W, name, N):
    """wb_sdf_train_tc's loss, decoder gradients and grid gradients inside the float64 fp16-faithful intervals; samples whose relu
    mask the intervals leave open are dropped.  Prints max|k - c| / r and the median radius per output.  'tiles3': every CTA runs
    three or more tiles."""
    import sdf_tc_reference as TR
    if N in (1, 63, 64, 65, 65536) and name not in ("config3", "l2_h128", "hash_cat8", "h96"):
        pytest.skip("every batch size on four shapes; the others at 1000 and three tiles per CTA")
    field, nef, pts = _interval_field(W, name)
    if N == "tiles3":
        fd = W.ops.sdf_field(nef)
        smem = W.ops.sdf_train_tc_smem_bytes(fd)
        sms = torch.cuda.get_device_properties(0).multi_processor_count
        N = 3 * 64 * sms * max(1, min(16, (228 * 1024) // (smem + 1024)))
    coords, gt = pts(N, N % 97 + 1)
    lods = [field.num_lods - 1]
    ref = TR.train_tc(field, coords, gt, lods)
    assert ref.amb.mean() <= 0.05, ref.amb.mean()
    if ref.amb.any():
        coords, gt = coords[~ref.amb], gt[~ref.amb]
        ref = TR.train_tc(field, coords, gt, lods)
    loss, got = _kernel(W, nef, dev(coords.astype(np.float32)), dev(gt.astype(np.float32)), lods)
    out = [("loss", *_inside(loss, ref.loss, ref.loss_r, (name, N, "loss")))]
    dec = np.concatenate([got[n].reshape(-1) for n, _ in nef.named_parameters() if n.startswith("decoder.")])
    out.append(("decoder", *_inside(dec, ref.dec, ref.dec_r, (name, N, "decoder"))))
    grid = [v for n, v in got.items() if not n.startswith("decoder.")]
    if name.startswith("hash"):
        tc = np.concatenate([c for c, _ in ref.grid]); tr = np.concatenate([r for _, r in ref.grid])
        out.append(("table", *_inside(grid[0], tc, tr, (name, N, "table"))))
    else:
        for k, (g, (c, r)) in enumerate(zip(grid, ref.grid)):
            out.append((f"grid{k}", *_inside(g, c, r, (name, N, "grid", k))))
    print(f"{name} N={N}: " + ", ".join(f"{w} max|k-c|/r {q:.2f} median r {m:.1e}" for w, q, m in out))
