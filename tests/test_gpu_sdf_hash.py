"""NeuralSDF(HashGrid) on the native SDF route, on the GPU: wb_sdf_eval's features against wb_hashgrid_fwd (bit for bit), its
predictions against a float64 evaluation with an fp32 error bound, wb_sdf_train (1 to 4 hidden layers) against the package's
autograd route (wb_hashgrid_fwd/bwd + torch decoder and loss), SDFStep against autograd + torch.optim.Adam, and PackedSDFTracer over
a hash field against the same trace through the torch field."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

EPS32 = 2.0 ** -24


@pytest.fixture(scope="module")
def W():
    import wisp_b200
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return wisp_b200


_CASE = {}


def _case():
    from oracle import octree_grid as OG
    if not _CASE:
        _CASE.update(OG.make_sdf_case(level=5, num_lods=3, feature_dim=8, hidden_dim=32, res=32, seed=3))
    return _CASE


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


# pos: 0 none, 1 identity (nglod_hash.yaml), 2 positional, 3 positional + input
_POS = {0: ('none', False), 1: ('none', True), 2: ('positional', False), 3: ('positional', True)}
# name: (F, multiscale, num_lods, bitwidth, min_res, max_res, pos mode, H, hidden layers)
SHAPES = {
    "nglod_hash": (8, 'cat', 4, 19, 16, 2048, 1, 128, 1),
    "sum4": (4, 'sum', 4, 10, 4, 32, 1, 64, 1),
    "cat4_pos3": (4, 'cat', 3, 10, 4, 32, 3, 32, 1),
    "cat8_pos0": (8, 'cat', 3, 10, 4, 32, 0, 32, 1),
    "sum8_pos2": (8, 'sum', 4, 10, 4, 32, 2, 16, 1),
    "l2_h64": (8, 'cat', 4, 10, 4, 32, 1, 64, 2),
    "l3_h32": (4, 'sum', 4, 10, 4, 32, 3, 32, 3),
    "l4_h16": (8, 'cat', 3, 10, 4, 32, 1, 16, 4),
}


def _field(W, shape, seed=0, std=0.1):
    F, ms, L, bw, rmin, rmax, pm, H, nh = SHAPES[shape]
    torch.manual_seed(seed)
    blas = W.OctreeAS(dev(_case()["octree"]))
    grid = W.HashGrid.from_geometric(blas, feature_dim=F, num_lods=L, multiscale_type=ms, feature_std=std, codebook_bitwidth=bw,
                                     min_grid_res=rmin, max_grid_res=rmax)
    pe, pin = _POS[pm]
    nef = W.NeuralSDF(grid, pos_embedder=pe, pos_multires=4, position_input=pin, hidden_dim=H, num_layers=nh).cuda()
    with torch.no_grad():                                           # both relu sides populated
        for l in nef.decoder.layers:
            l.bias.uniform_(-0.3, 0.3)
    return nef


def _points(n, seed=5, res=(16, 2048)):
    """Uniform points in [-1.2, 1.2]^3 plus: points outside [-1.1, 1.1], exact +-1, cell faces of a dense (res[0]) and of a hashed
    level (res[1]: 2k/res - 1 is exact), and duplicates."""
    rng = np.random.default_rng(seed)
    c = rng.uniform(-1.2, 1.2, (n, 3)).astype(np.float32)
    extra = [rng.uniform(1.1, 1.6, (8, 3)) * rng.choice([-1, 1], (8, 3)), np.array([[1, 1, 1], [-1, -1, -1], [1, -1, 0.5], [-1, 0.25, 1]]),
             2.0 * rng.integers(0, res[0] + 1, (8, 3)) / res[0] - 1.0, 2.0 * rng.integers(0, res[1] + 1, (8, 3)) / res[1] - 1.0]
    c = np.concatenate([np.concatenate(extra).astype(np.float32), c])[:n]
    if n > 16:
        c[-8:] = c[:8]
    gt = ((np.abs(c).sum(-1, keepdims=True) - 0.5) / np.sqrt(3.0)).astype(np.float32)
    return dev(c), dev(gt)


def _hash_feats(W, nef, coords, lod_idx):
    """wb_hashgrid_fwd ([N, L*F], fp32) followed by the 'cat' zeroing / the 'sum' over all LODs in LOD order (fp32)."""
    g = nef.grid
    with torch.no_grad():
        raw = W.ops.hashgrid(coords, g.codebook_bitwidth, lod_idx, g.codebook).cpu().numpy()
    F, L = g.feature_dim, g.num_lods
    if g.multiscale_type == 'cat':
        raw[:, lod_idx * F:] = 0.0
        return raw
    r = raw.reshape(-1, L, F)
    acc = np.zeros((raw.shape[0], F), np.float32)
    for l in range(L):
        acc = (acc + r[:, l]).astype(np.float32)
    return acc


def _embed(nef, c):
    """float64 position embedding of fp32 coordinates (positional_embedder.py:51-66)."""
    pe = nef.pos_embedder
    if pe is None:
        return np.zeros((c.shape[0], 0))
    if isinstance(pe, torch.nn.Identity):
        return c
    out = [c] if pe.include_input else []
    bands = [2.0 ** f for f in range(pe.num_freq)]
    wind = np.concatenate([c * b for b in bands], -1)
    return np.concatenate(out + [np.sin(wind), np.cos(wind)], -1)


def _f64_sdf(nef, c, feats):
    """float64 BasicDecoder on [embedding, features] and the bound of an fp32 evaluation of it: per layer |a - a64| <= (n+1) u
    sum|w x| + the propagated input error; sinf/cosf inputs carry 2 ulp."""
    x = np.concatenate([_embed(nef, c), feats.astype(np.float64)], -1)
    pd = x.shape[1] - feats.shape[1]
    err = np.zeros_like(x)
    if nef.pos_embedder is not None and not isinstance(nef.pos_embedder, torch.nn.Identity):
        err[:, (3 if nef.pos_embedder.include_input else 0):pd] = 2 * EPS32 * 2
    layers = list(nef.decoder.layers) + [nef.decoder.lout]
    h, e = x, err
    for i, l in enumerate(layers):
        Wt, b = l.weight.detach().double().cpu().numpy(), l.bias.detach().double().cpu().numpy()
        a = h @ Wt.T + b
        mag = np.abs(h) @ np.abs(Wt).T + np.abs(b)
        e = (Wt.shape[1] + 2) * EPS32 * 1.01 * mag + e @ np.abs(Wt).T
        if i < len(layers) - 1:
            h = np.maximum(a, 0.0)
        else:
            h = a
    return h[:, 0], e[:, 0]


# ---------------------------------------------------------------------------------------------------------------
# wb_sdf_eval
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("shape", ["nglod_hash", "sum4", "cat4_pos3"])
def test_eval_features_are_hashgrid_fwd(W, shape):
    """A decoder of one unit that passes feature f through (W0 = +-e_f, zero biases, wout = 1) returns relu(+-feat_f) exactly, so
    wb_sdf_eval's features are read out bit for bit: equal to wb_hashgrid_fwd + the 'cat'/'sum' rule at every lod_idx."""
    F, ms, L, bw, rmin, rmax, pm, H, nh = SHAPES[shape]
    nef = _field(W, shape)
    c, _ = _points(2000, seed=1, res=(nef.grid.resolutions[0], nef.grid.resolutions[-1]))
    pe, pin = _POS[pm]
    probe = W.NeuralSDF(nef.grid, pos_embedder=pe, pos_multires=4, position_input=pin, hidden_dim=1, num_layers=1).cuda()
    width = F if ms == 'sum' else F * L
    pd = probe.decoder.layers[0].in_features - width
    for lod in range(L):
        ref = _hash_feats(W, nef, c, lod)
        got = np.zeros_like(ref)
        for f in range(width):
            vals = []
            for sgn in (1.0, -1.0):
                with torch.no_grad():
                    probe.decoder.layers[0].weight.zero_(); probe.decoder.layers[0].weight[0, pd + f] = sgn
                    probe.decoder.layers[0].bias.zero_(); probe.decoder.lout.weight.fill_(1.0); probe.decoder.lout.bias.zero_()
                    vals.append(W.ops.sdf_eval(probe, c, lod).cpu().numpy()[:, 0])
            got[:, f] = vals[0] - vals[1]
        assert np.array_equal(got, ref), (lod, np.abs(got - ref).max())
        if ms == 'cat' and lod == 0:
            assert not got.any()


@pytest.mark.parametrize("shape", list(SHAPES))
def test_eval_inside_f64_bound(W, shape):
    """wb_sdf_eval at every lod_idx against a float64 decoder over the exact fp32 features, within the fp32 error bound; and
    NeuralSDF.sdf under no_grad takes this route."""
    nef = _field(W, shape)
    c, _ = _points(3000, seed=2, res=(nef.grid.resolutions[0], nef.grid.resolutions[-1]))
    cn = c.cpu().numpy().astype(np.float64)
    for lod in range(nef.grid.num_lods):
        with torch.no_grad():
            y = W.ops.sdf_eval(nef, c, lod)
        assert y is not None
        y = y.cpu().numpy()[:, 0].astype(np.float64)
        ref, bound = _f64_sdf(nef, cn, _hash_feats(W, nef, c, lod))
        assert (np.abs(y - ref) <= bound).all(), (lod, np.abs(y - ref).max(), float(bound[np.argmax(np.abs(y - ref))]))
    with torch.no_grad():
        before = W._cabi.launch_count()
        y2 = nef(coords=c, lod_idx=nef.grid.num_lods - 1, channels="sdf")
        assert W._cabi.launch_count() - before == 1
    assert torch.equal(y2.reshape(-1), W.ops.sdf_eval(nef, c).reshape(-1))


# ---------------------------------------------------------------------------------------------------------------
# wb_sdf_train / SDFStep against the autograd route
# ---------------------------------------------------------------------------------------------------------------
def _autograd(nef, coords, gt, lods):
    for p in nef.parameters():
        p.grad = None
    loss = 0.0
    for lod in lods:
        loss = loss + ((nef(coords=coords, lod_idx=lod, channels="sdf") - gt) ** 2).sum()
    loss = loss / coords.shape[0]
    loss.backward()
    return float(loss.detach()), {n: p.grad.detach().clone() if p.grad is not None else torch.zeros_like(p)
                                  for n, p in nef.named_parameters() if p.requires_grad}


def _fused_grads(nef, step):
    g = {"grid.codebook.feats": step.g_feats[0]}
    o = 0
    for n, p in nef.named_parameters():
        if n.startswith("decoder."):
            g[n] = step.g_dec[o:o + p.numel()].view_as(p); o += p.numel()
    return g


def _close(got, ref, loss, ref_loss, tol_loss=1e-5, tol_grad=1e-4):
    assert abs(loss - ref_loss) <= tol_loss * abs(ref_loss), (loss, ref_loss)
    for n, r in ref.items():
        err = float((got[n] - r).abs().max())
        assert err <= tol_grad * max(float(r.abs().max()), 1e-30), (n, err, float(r.abs().max()))


_BIG = 3 * 132 * 4 * 128          # at least three 128-sample tiles per CTA at up to 4 resident CTAs per SM


@pytest.mark.parametrize("shape,N,only_last", [("nglod_hash", 1, True), ("nglod_hash", 127, True), ("nglod_hash", 129, True),
                                               ("nglod_hash", 65536, True), ("nglod_hash", 65536, False), ("nglod_hash", _BIG, True),
                                               ("sum4", 1000, True), ("sum4", 1000, False), ("cat4_pos3", 1000, False),
                                               ("sum8_pos2", 1000, True), ("cat8_pos0", 128, False),
                                               ("l2_h64", 1, True), ("l2_h64", 129, False), ("l2_h64", _BIG, True),
                                               ("l3_h32", 1000, False), ("l4_h16", 1000, True), ("l4_h16", 33, False)])
def test_sdf_step_fused_vs_autograd(W, shape, N, only_last):
    """SDFStep.step(update=False) (one wb_sdf_train per loss LOD) against nef(...) + torch loss + .backward(): loss 1e-5 relative,
    table and decoder gradients 1e-4 of their max.  'cat' over all LODs trains (the hash grid keeps its width)."""
    nef = _field(W, shape)
    step = W.SDFStep(W.Pipeline(nef), only_last=only_last)
    assert step.fused
    coords, gt = _points(N, seed=N)
    loss = float(step.step(coords, gt, update=False))
    got = _fused_grads(nef, step)
    ref_loss, ref = _autograd(nef, coords, gt, step.loss_lods)
    _close(got, ref, loss, ref_loss)


def test_sdf_train_accumulates_and_n0(W):
    """wb_sdf_train adds to non-zero buffers (twice the same batch = 2x), and N = 0 leaves them untouched."""
    nef = _field(W, "l2_h64")
    step = W.SDFStep(W.Pipeline(nef))
    coords, gt = _points(1000, seed=7)
    c, g = coords.contiguous(), gt.reshape(-1).contiguous()
    lod = nef.grid.num_lods - 1
    W.ops.sdf_train(step.fd, c, g, lod, 1e-3, step.g_feats, step.g_dec, step.loss_buf)
    once = [t.clone() for t in step.g_feats + [step.g_dec, step.loss_buf]]
    W.ops.sdf_train(step.fd, c, g, lod, 1e-3, step.g_feats, step.g_dec, step.loss_buf)
    for a, b in zip(step.g_feats + [step.g_dec, step.loss_buf], once):
        assert float((a - 2 * b).abs().max()) <= 1e-5 * max(float(b.abs().max()), 1e-30)
    twice = [t.clone() for t in step.g_feats + [step.g_dec, step.loss_buf]]
    import ctypes as C
    A = W._cabi
    d, _, _ = step.fd
    gptrs = (C.c_void_p * 1)(step.g_feats[0].data_ptr())
    A.check(A.lib().wb_sdf_train(None, C.byref(d), C.c_int32(lod), A.ptr(c), A.ptr(g), C.c_int64(0), C.c_float(1e-3), gptrs,
                                 A.ptr(step.g_dec), A.ptr(step.loss_buf), A.stream()))
    torch.cuda.synchronize()
    for a, b in zip(step.g_feats + [step.g_dec, step.loss_buf], twice):
        assert torch.equal(a, b)


@pytest.mark.parametrize("lod", [0, 1, 3])
def test_sdf_train_lower_lods(W, lod):
    """One wb_sdf_train at a lower lod_idx against autograd of nef(lod_idx=lod): 'cat' zeroes LODs >= lod (lod 0: no grid gradient)."""
    nef = _field(W, "nglod_hash")
    step = W.SDFStep(W.Pipeline(nef))
    coords, gt = _points(4096, seed=11)
    step.loss_buf.zero_()
    W.ops.sdf_train(step.fd, coords, gt.reshape(-1).contiguous(), lod, 1.0 / 4096, step.g_feats, step.g_dec, step.loss_buf)
    ref_loss, ref = _autograd(nef, coords, gt, [lod])
    _close(_fused_grads(nef, step), ref, float(step.loss_buf[0]), ref_loss)
    if lod == 0:
        assert not step.g_feats[0].any()


def test_sdf_step_loss_is_eval_loss(W):
    nef = _field(W, "nglod_hash")
    step = W.SDFStep(W.Pipeline(nef))
    coords, gt = _points(65536, seed=9)
    loss = float(step.step(coords, gt, update=False))
    with torch.no_grad():
        y = W.ops.sdf_eval(nef, coords).double()
    ref = float(((y - gt.double()) ** 2).sum() / coords.shape[0])
    assert abs(loss - ref) <= 1e-6 * ref, (loss, ref)


def _torch_adam(nef, lr, wd, glw, eps):
    dec = [p for n, p in nef.named_parameters() if p.requires_grad and "decoder" in n]
    grd = [p for n, p in nef.named_parameters() if p.requires_grad and "decoder" not in n and "grid" in n]
    return torch.optim.Adam([{"params": dec, "lr": lr, "eps": eps, "weight_decay": wd}, {"params": grd, "eps": eps, "lr": lr * glw}],
                            lr=lr, eps=eps)


@pytest.mark.parametrize("only_last", [True, False])
def test_sdf_step_trajectory(W, only_last):
    """Five SDFStep steps against autograd + torch.optim.Adam with init_optimizer's groups (table: lr * grid_lr_weight, no decay;
    decoder: weight decay): losses 1e-4 relative, parameters 1e-6 per 1e-3 of their group's lr where the gradient was never below
    1e-4 of max, within 2 lr steps everywhere."""
    lr, wd, glw, eps, steps = 1e-3, 1e-2, 5.0, 1e-15, 5
    nef, ref_nef = _field(W, "nglod_hash"), _field(W, "nglod_hash")
    step = W.SDFStep(W.Pipeline(nef), lr=lr, eps=eps, weight_decay=wd, grid_lr_weight=glw, only_last=only_last)
    opt = _torch_adam(ref_nef, lr, wd, glw, eps)
    coords, gt = _points(16384, seed=3)
    small = {n: torch.zeros_like(p, dtype=torch.bool) for n, p in ref_nef.named_parameters()}
    for s in range(steps):
        loss = float(step.step(coords, gt))
        ref_loss, grads = _autograd(ref_nef, coords, gt, step.loss_lods)
        opt.step()
        assert abs(loss - ref_loss) <= 1e-4 * abs(ref_loss), (s, loss, ref_loss)
        for n, gr in grads.items():
            small[n] |= gr.abs() < 1e-4 * gr.abs().max()
    ref_p = dict(ref_nef.named_parameters())
    for n, p in nef.named_parameters():
        d = (p.detach() - ref_p[n].detach()).abs()
        lr_g = lr * (glw if n.startswith("grid.") else 1.0)
        assert float(d[~small[n]].max()) <= 1e-6 * lr_g / 1e-3, n
        assert float(d.max()) <= 2 * lr_g * steps, n


def test_sdf_step_launch_count(W):
    nef = _field(W, "nglod_hash")
    step = W.SDFStep(W.Pipeline(nef))
    coords, gt = _points(512, seed=1)
    step.step(coords, gt)
    before = W._cabi.launch_count()
    step.step(coords, gt)
    assert W._cabi.launch_count() - before == 2
    torch.cuda.synchronize()


def test_sdf_step_footprint_fallback(W):
    """A hash field whose training footprint exceeds shared memory (3 hidden layers of 128) trains through autograd, matching it."""
    SHAPES["l3_h128"] = (8, 'cat', 4, 10, 4, 32, 1, 128, 3)
    try:
        nef = _field(W, "l3_h128")
    finally:
        del SHAPES["l3_h128"]
    assert W.ops.sdf_field(nef) is not None and W.ops.sdf_train_smem_bytes(W.ops.sdf_field(nef)) < 0
    step = W.SDFStep(W.Pipeline(nef))
    assert not step.fused
    coords, gt = _points(1000, seed=4)
    loss = float(step.step(coords, gt, update=False))
    ref_loss, _ = _autograd(nef, coords, gt, step.loss_lods)
    assert abs(loss - ref_loss) <= 1e-6 * ref_loss


# ---------------------------------------------------------------------------------------------------------------
# PackedSDFTracer over a hash field
# ---------------------------------------------------------------------------------------------------------------
def test_tracer_over_hash_field(W, monkeypatch):
    """PackedSDFTracer over an nglod_hash-shaped field (phase-by-phase tracer, field through wb_sdf_eval) against the same trace
    with ops.sdf_eval forced to None (the torch field): at most 0.2 % of the rays flip, depths agree to 1e-4."""
    case = _case()
    nef = _field(W, "nglod_hash", std=0.01)
    with torch.no_grad():                                           # (|x|+|y|+|z| - 0.52)/sqrt(3) plus a small grid part
        nef.decoder.layers[0].weight.mul_(0.05)
        nef.decoder.layers[0].weight[:6, :3] = torch.tensor([[1, 0, 0], [-1, 0, 0], [0, 1, 0], [0, -1, 0], [0, 0, 1], [0, 0, -1.0]])
        nef.decoder.layers[0].bias.zero_()
        nef.decoder.lout.weight.mul_(0.01); nef.decoder.lout.weight[0, :6] = 1.0 / np.sqrt(3.0)
        nef.decoder.lout.bias.fill_(-0.52 / np.sqrt(3.0))      # the case's octree: |x|+|y|+|z| = 0.52
    tracer = W.PackedSDFTracer(num_steps=64, step_size=0.8, min_dis=1e-3)
    rays = W.Rays(dev(case["origins"]), dev(case["dirs"]), 0.0, 6.0)
    native, evals = W.ops.sdf_eval, []

    def counted(*a, **k):
        out = native(*a, **k)
        evals.append(out is not None)
        return out
    monkeypatch.setattr(W.ops, "sdf_eval", counted)
    rb = W.Pipeline(nef, tracer)(rays=rays, channels=["depth", "hit", "normal"])
    torch.cuda.synchronize()
    assert len(evals) > 10 and all(evals)          # every field evaluation (the march and the 6 of the normals) went to wb_sdf_eval
    monkeypatch.setattr(W.ops, "sdf_eval", lambda *a, **k: None)
    ref = W.Pipeline(nef, tracer)(rays=rays, channels=["depth", "hit", "normal"])
    hit, rhit = rb.hit.cpu().numpy(), ref.hit.cpu().numpy()
    assert rhit.sum() > 50
    assert (hit != rhit).sum() <= max(1, 0.002 * hit.size), int((hit != rhit).sum())
    both = hit & rhit
    assert np.abs(rb.depth.cpu().numpy()[both] - ref.depth.cpu().numpy()[both]).max() <= 1e-4


# ---------------------------------------------------------------------------------------------------------------
# the reference trainer's own steps, and the float64 interval reference
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", ["cat", "sum", "cat_all", "cat_l2"])
def test_sdf_step_hash_golden(W, golden_dir, case):
    """tests/golden/sdf_train_hash.npz (the reference's SDFTrainer.step + init_optimizer over its NeuralSDF(HashGrid), 3 steps):
    step-1 table and decoder gradients 1e-4 of max (fp32 both, summation orders differ), Adam's first step a sign step of each group's
    learning rate where the gradient is not negligible, and the three losses to 1e-4 relative."""
    import os
    g = np.load(os.path.join(golden_dir, "sdf_train_hash.npz"))
    ms, F, nh = str(g[f"{case}_multiscale"]), int(g[f"{case}_feature_dim"]), int(g[f"{case}_num_layers"])
    lr, wd, glw = float(g["lr"]), float(g["weight_decay"]), float(g["grid_lr_weight"])
    blas = W.OctreeAS(dev(g["octree"]))
    grid = W.HashGrid.from_geometric(blas, feature_dim=F, num_lods=4, multiscale_type=ms, codebook_bitwidth=int(g[f"{case}_codebook_bitwidth"]),
                                     min_grid_res=4, max_grid_res=32)
    assert grid.resolutions == [int(r) for r in g[f"{case}_resolutions"]]
    nef = W.NeuralSDF(grid, pos_embedder='none', position_input=True, hidden_dim=16, num_layers=nh).cuda()
    with torch.no_grad():
        for n, p in nef.named_parameters():
            p.copy_(dev(g[f"{case}_init_{n}"]))
    step = W.SDFStep(W.Pipeline(nef), lr=lr, eps=float(g["eps"]), weight_decay=wd, grid_lr_weight=glw, only_last=len(g[f"{case}_loss_lods"]) == 1)
    assert step.fused
    coords, sdf = dev(g["coords"]), dev(g["sdf"])
    step.step(coords, sdf, update=False)
    got = {k: v.detach().cpu().numpy() for k, v in _fused_grads(nef, step).items()}
    for n in got:
        ref = g[f"{case}_grad1_{n}"]
        assert np.abs(got[n] - ref).max() <= 1e-4 * np.abs(ref).max(), n
    step.zero_grads()
    losses = []
    for s in range(3):
        losses.append(float(step.step(coords, sdf)))
        if s == 0:
            for n, p in nef.named_parameters():
                init, ref_g, now = g[f"{case}_init_{n}"], g[f"{case}_grad1_{n}"], p.detach().cpu().numpy()
                lr_g, eff = (lr * glw, ref_g) if n.startswith("grid.") else (lr, ref_g + wd * init)
                big = np.abs(eff) > 1e-3 * np.abs(eff).max()
                assert big.any(), n
                np.testing.assert_allclose(now[big], (init - lr_g * np.sign(eff))[big], atol=1e-6, err_msg=n)
    np.testing.assert_allclose(losses, g[f"{case}_losses"], rtol=1e-4)


@pytest.mark.parametrize("shape,N,only_last", [("nglod_hash", 1, True), ("nglod_hash", 129, True), ("nglod_hash", 5000, False),
                                               ("sum4", 1000, False), ("cat4_pos3", 1000, True), ("l2_h64", 1000, False),
                                               ("l3_h32", 129, True), ("l4_h16", 1000, True)])
def test_sdf_train_inside_intervals(W, shape, N, only_last):
    """wb_sdf_train's loss, decoder gradient and table gradient inside the float64 interval reference (oracle/sdf_reference.py with
    the hash hook of tests/sdf_hash_reference.py; tests/sdf_deep_reference.py for 2-4 layers); samples whose relu decision the
    reference cannot settle are dropped."""
    import sdf_deep_reference as D
    import sdf_hash_reference as HR
    nef = _field(W, shape)
    g = nef.grid
    Ws = [l.weight.detach().cpu().numpy() for l in list(nef.decoder.layers) + [nef.decoder.lout]]
    bs = [l.bias.detach().cpu().numpy() for l in list(nef.decoder.layers) + [nef.decoder.lout]]
    pm = SHAPES[shape][6]
    field = HR.hash_field(g.codebook.feats.detach().cpu().numpy(), g.codebook.begin_idxes.tolist(), g.resolutions, g.codebook_bitwidth,
                          g.multiscale_type, Ws, bs, pm, 4 if pm >= 2 else 0)
    coords, gt = _points(N, seed=N + 1)
    c, t = coords.cpu().numpy(), gt.cpu().numpy()[:, 0]
    lods = [g.num_lods - 1] if only_last else list(range(g.num_lods))
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    ref = D.train(field, c, t, lods, sms=sms)
    keep = ~ref.amb
    if not keep.all():
        c, t = c[keep], t[keep]
        ref = D.train(field, c, t, lods, sms=sms)
    step = W.SDFStep(W.Pipeline(nef), only_last=only_last)
    loss = float(step.step(dev(c), dev(t[:, None].astype(np.float32)), update=False))
    assert abs(loss - ref.loss) <= ref.loss_r, (loss, ref.loss, ref.loss_r)
    dec = step.g_dec.cpu().numpy()
    assert (np.abs(dec - ref.dec) <= ref.dec_r).all(), np.abs(dec - ref.dec).max()
    tc, tr = HR.table_grad(ref)
    tab = step.g_feats[0].cpu().numpy()
    assert (np.abs(tab - tc) <= tr).all(), (np.abs(tab - tc) - tr).max()
