"""SDFStep's fused route for decoders with 2 to 4 hidden layers (wb_sdf_train_deep_kernel): against the reference trainer's own
three steps (tests/golden/sdf_train_deep.npz), against the float64 interval reference tests/sdf_deep_reference.py on the fields of
tests/sdf_deep_shapes.py (batch sizes around the kernel's sample tile, and batches of >= 3 tiles per CTA), against the evaluation
kernel's loss, against the package's autograd route and torch.optim.Adam at the BASELINE config-3 shape with num_layers = 2, and
on both sides of the shared-memory footprint that decides native or autograd."""
import os

import numpy as np
import pytest
import torch

from oracle import octree_grid as OG
from oracle import sdf_reference as S

import sdf_deep_reference as DR
import sdf_deep_shapes as DS
from test_gpu_sdf_kernels import drop_ambiguous, fused_step, inside, nef_of

pytestmark = pytest.mark.gpu

SMEM_PER_SM, SMEM_PER_CTA_RESERVED = 228 * 1024, 1024       # H100


@pytest.fixture(scope="module")
def W():
    import wisp_b200
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return wisp_b200


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _dec_names(nef):
    return [n for n, _ in nef.named_parameters() if n.startswith("decoder.")]


def _step_grads(nef, step):
    g = {f"grid.features.{k}": t for k, t in enumerate(step.g_feats)}
    o = 0
    for n, p in nef.named_parameters():
        if n.startswith("decoder."):
            g[n] = step.g_dec[o:o + p.numel()].view_as(p); o += p.numel()
    return {k: v.detach().cpu().numpy() for k, v in g.items()}


# ---------------------------------------------------------------------------------------------------------------
# the reference trainer's own steps
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", ["sum", "cat", "sum_all"])
def test_deep_golden(W, golden_dir, case):
    """Step-1 gradients 2e-2 of max (the fp16-feature tolerance of test_sdf_step_golden), three losses 2e-3 relative."""
    g = np.load(os.path.join(golden_dir, "sdf_train_deep.npz"))
    ms = str(g[f"{case}_multiscale"])
    only_last = len(g[f"{case}_loss_lods"]) == 1
    layers = len([k for k in g.files if k.startswith(f"{case}_init_decoder.layers.") and k.endswith(".weight")])
    blas = W.OctreeAS(dev(g["octree"]))
    grid = W.OctreeGrid(blas, feature_dim=8, num_lods=3, multiscale_type=ms, feature_std=0.0)
    nef = W.NeuralSDF(grid, pos_embedder='none', position_input=True, hidden_dim=16, num_layers=layers).cuda()
    with torch.no_grad():
        for n, p in nef.named_parameters():
            p.copy_(dev(g[f"{case}_init_{n}"]))
    step = W.SDFStep(W.Pipeline(nef), lr=float(g["lr"]), eps=float(g["eps"]), weight_decay=float(g["weight_decay"]),
                     grid_lr_weight=float(g["grid_lr_weight"]), only_last=only_last)
    assert step.fused
    coords, sdf = dev(g["coords"]), dev(g["sdf"])
    step.step(coords, sdf, update=False)
    got = _step_grads(nef, step)
    for n, p in nef.named_parameters():
        ref = g[f"{case}_grad1_{n}"]
        assert np.abs(got[n] - ref).max() <= 2e-2 * max(np.abs(ref).max(), 1e-12), n
    step.zero_grads()
    losses = [float(step.step(coords, sdf)) for _ in range(3)]
    np.testing.assert_allclose(losses, g[f"{case}_losses"], rtol=2e-3)


# ---------------------------------------------------------------------------------------------------------------
# the interval reference
# ---------------------------------------------------------------------------------------------------------------
def _smem(W, nef):
    return W.ops.sdf_train_smem_bytes(W.ops.sdf_field(nef))


def check_deep(W, field, case, coords, gt, only_last=True, what=""):
    lods = [field.num_lods - 1] if only_last else list(range(field.num_lods))
    tile = DS.tile_of(field)
    ref = DR.train(field, coords, gt, lods, sms=_sms(), tile=tile)
    assert ref.amb.mean() <= 0.02, ref.amb.mean()
    if ref.amb.any():
        coords, gt = coords[~ref.amb], gt[~ref.amb]
        ref = DR.train(field, coords, gt, lods, sms=_sms(), tile=tile)
        assert not ref.amb.any()
    nef = nef_of(W, field, case)
    loss, dec, grid, _ = fused_step(W, nef, coords, gt, only_last)
    inside(loss, ref.loss, ref.loss_r, ("loss", what))
    inside(dec, ref.dec, ref.dec_r, ("decoder", what))
    for k, (g, (c, r)) in enumerate(zip(grid, ref.grid)):
        inside(g, c, r, ("grid", k, what))
        assert np.all(g[c == 0][r[c == 0] == 0] == 0), ("untouched rows", k, what)


@pytest.mark.parametrize("name", sorted(DS.DEEP_SHAPES))
@pytest.mark.parametrize("N", [1, "tile-1", "tile", "tile+1", 1000, "tiles3"])
def test_deep_train_vs_reference(W, name, N):
    field, case = DS.make_field(name, seed=1)
    tile = DS.tile_of(field)
    assert tile is not None
    if isinstance(N, str):
        if N == "tiles3":       # every CTA runs >= 3 tiles: CTAs <= SMs x (CTAs per SM by shared memory and by 2048 threads)
            nef = nef_of(W, field, case)
            smem = _smem(W, nef)
            assert smem == (2 * ((S_img(field) + 3) & ~3) + tile * S_row(field) + 16) * 4      # the host formula, restated
            per_sm = max(1, min(2048 // 256, SMEM_PER_SM // (smem + SMEM_PER_CTA_RESERVED)))
            N = 3 * tile * _sms() * per_sm
        else:
            N = tile + {"tile-1": -1, "tile": 0, "tile+1": 1}[N]
    coords, gt = DS.points(case, N, seed=N % 97)
    check_deep(W, field, case, coords, gt, what=(name, N))
    if N == 1000 and field.multiscale == "sum":
        check_deep(W, field, case, coords, gt, only_last=False, what=(name, "all LODs"))


def S_img(field):
    H, nh, in_dim = field.Ws[0].shape[0], len(field.Ws) - 1, field.Ws[0].shape[1]
    return H * ((in_dim + 3) & ~3) + H + (nh - 1) * (H * H + H) + H + 4


def S_row(field):
    H, nh, in_dim = field.Ws[0].shape[0], len(field.Ws) - 1, field.Ws[0].shape[1]
    st = lambda n: ((n + 31) & ~31) + 4
    return st((in_dim + 3) & ~3) + nh * st(H) + 1


def test_deep_contract(W):
    """Accumulates into the buffers passed in; N = 0 changes nothing."""
    field, case = DS.make_field("l2_h64", seed=1)
    nef = nef_of(W, field, case)
    coords, gt = DS.points(case, 700, seed=8)
    coords, gt = drop_ambiguous(field, coords, gt, [field.num_lods - 1])
    fd = W.ops.sdf_field(nef)
    c, g = dev(coords), dev(gt)
    lod = field.num_lods - 1
    rng = np.random.default_rng(0)
    init_f = [np.float32(2.0 ** -8) * rng.integers(-64, 64, f.shape).astype(np.float32) for f in field.feats]
    init_p = np.float32(2.0 ** -8) * rng.integers(-64, 64, field.packed().size).astype(np.float32)
    gf, gp, loss = [dev(f) for f in init_f], dev(init_p), torch.full((1,), 0.25, device="cuda")
    import ctypes as C
    A = W._cabi
    gptrs = (C.c_void_p * len(gf))(*[t.data_ptr() for t in gf])
    A.lib().wb_sdf_train(fd[1].desc(), fd[0], lod, A.ptr(c), A.ptr(g), 0,
                         1.0, gptrs, A.ptr(gp), A.ptr(loss), A.stream())
    torch.cuda.synchronize()
    assert all(np.array_equal(a.cpu().numpy(), b) for a, b in zip(gf, init_f)) and np.array_equal(gp.cpu().numpy(), init_p)
    assert float(loss) == 0.25
    W.ops.sdf_train(fd, c, g, lod, 1.0 / coords.shape[0], gf, gp, loss)
    torch.cuda.synchronize()
    ref = DR.train(field, coords, gt, [lod], sms=_sms(), tile=DS.tile_of(field))
    inside(float(loss) - 0.25, ref.loss, ref.loss_r + S.g32(ref.atomics) * 0.25, "loss")
    inside(gp.cpu().numpy().astype(np.float64) - init_p, ref.dec, ref.dec_r + S.g32(ref.atomics) * np.abs(init_p), "decoder")
    for k, (a, (cc, r)) in enumerate(zip(gf, ref.grid)):
        inside(a.cpu().numpy().astype(np.float64) - init_f[k], cc, r + S.g32(ref.grid_n[k])[:, None] * np.abs(init_f[k]), ("grid", k))


@pytest.mark.parametrize("name", ["l2_h128", "cat_l3"])
def test_deep_loss_is_eval_loss(W, name):
    """The kernel's forward is wb_sdf_eval's: its loss equals the loss of ops.sdf_eval's predictions to 1e-6 relative."""
    field, case = DS.make_field(name, seed=1)
    nef = nef_of(W, field, case)
    step = W.SDFStep(W.Pipeline(nef))
    assert step.fused
    coords, gt = DS.points(case, 65536, seed=9)
    c, g = dev(coords), dev(gt)
    loss = float(step.step(c, g, update=False))
    with torch.no_grad():
        y = W.ops.sdf_eval(nef, c, nef.grid.num_lods - 1).double()
    ref = float(((y[:, 0] - g.double()) ** 2).sum() / coords.shape[0])
    assert abs(loss - ref) <= 1e-6 * ref, (loss, ref)


# ---------------------------------------------------------------------------------------------------------------
# the package's autograd route and torch.optim.Adam at the config-3 shape with two hidden layers
# ---------------------------------------------------------------------------------------------------------------
_CASE = {}


def _config3_l2(W):
    """BASELINE config 3 (level-7 octahedron, F = 16, 6 LODs 'sum', identity position input) with num_layers = 2, H = 128."""
    from gpu_util import sdf_nef_from_case
    if "c" not in _CASE:
        _CASE["c"] = OG.make_sdf_case(level=7, num_lods=6, feature_dim=16, hidden_dim=128, multiscale="sum", res=4, seed=11, feature_std=0.02)
    case = dict(_CASE["c"])
    case["W"], case["b"] = S.random_decoder(np.random.default_rng(4), 19, 1, 128, 2, scale=0.2)
    return sdf_nef_from_case(case), case


def _points(case, n, seed=5):
    rng = np.random.default_rng(seed)
    spc = case["spc"]; L = case["level"]
    pts = spc.points[spc.pyramid[1, L]: spc.pyramid[1, L] + spc.pyramid[0, L]].astype(np.float32)
    nn = (n + 1) // 2
    near = (pts[rng.integers(0, pts.shape[0], nn)] + rng.random((nn, 3)).astype(np.float32)) / (2.0 ** (L - 1)) - 1.0
    c = np.concatenate([near, rng.uniform(-1.05, 1.05, (n - nn, 3))]).astype(np.float32)[:n]
    gt = ((np.abs(c).sum(-1, keepdims=True) - 0.5) / np.sqrt(3.0)).astype(np.float32)
    return dev(c), dev(gt)


def _autograd(nef, coords, gt, lods):
    for p in nef.parameters():
        p.grad = None
    loss = 0.0
    for lod in lods:
        loss = loss + ((nef(coords=coords, lod_idx=lod, channels="sdf") - gt) ** 2).sum()
    loss = loss / coords.shape[0]
    loss.backward()
    return float(loss.detach()), {n: p.grad.detach().cpu().numpy() if p.grad is not None else np.zeros(tuple(p.shape), np.float32)
                                  for n, p in nef.named_parameters() if p.requires_grad}


def _vs_autograd(W, nef, coords, gt, only_last, fused):
    step = W.SDFStep(W.Pipeline(nef), only_last=only_last)
    assert step.fused == fused
    loss = float(step.step(coords, gt, update=False))
    got = _step_grads(nef, step) if fused else {n: p.grad.detach().cpu().numpy() for n, p in nef.named_parameters()}
    ref_loss, ref = _autograd(nef, coords, gt, step.loss_lods)
    assert abs(loss - ref_loss) <= 1e-5 * abs(ref_loss), (loss, ref_loss)
    for n, r in ref.items():
        assert np.abs(got[n] - r).max() <= 1e-4 * max(np.abs(r).max(), 1e-30), (n, np.abs(got[n] - r).max(), np.abs(r).max())


@pytest.mark.parametrize("N,only_last", [(64, True), (1000, True), (65536, True), (65536, False)])
def test_deep_fused_vs_autograd(W, N, only_last):
    """step(update=False) against nef(...) + torch loss + .backward(): loss 1e-5 relative, every gradient 1e-4 of its max.  (A
    single sample whose prediction nearly equals its target loses the loss's relative accuracy to cancellation in y - gt: batch
    1 is checked against the interval reference instead, test_deep_train_vs_reference.)"""
    nef, case = _config3_l2(W)
    coords, gt = _points(case, N)
    _vs_autograd(W, nef, coords, gt, only_last, True)


def _torch_adam(nef, lr, wd, glw, eps):
    dec, grd, rest = [], [], []
    for n, p in nef.named_parameters():
        if p.requires_grad:
            (dec if "decoder" in n else grd if "grid" in n else rest).append(p)
    return torch.optim.Adam([{"params": dec, "lr": lr, "eps": eps, "weight_decay": wd}, {"params": grd, "eps": eps, "lr": lr * glw},
                             {"params": rest, "eps": eps, "lr": lr}], lr=lr, eps=eps)


def test_deep_trajectory(W):
    """Five SDFStep steps against autograd + torch.optim.Adam with the reference's groups (test_sdf_step_trajectory's bounds)."""
    lr, wd, glw, eps, steps = 1e-3, 1e-2, 5.0, 1e-15, 5
    nef, case = _config3_l2(W)
    ref_nef, _ = _config3_l2(W)
    step = W.SDFStep(W.Pipeline(nef), lr=lr, eps=eps, weight_decay=wd, grid_lr_weight=glw)
    assert step.fused
    opt = _torch_adam(ref_nef, lr, wd, glw, eps)
    coords, gt = _points(case, 16384, seed=3)
    small = {n: np.zeros(tuple(p.shape), bool) for n, p in ref_nef.named_parameters()}
    for s in range(steps):
        loss = float(step.step(coords, gt))
        ref_loss, grads = _autograd(ref_nef, coords, gt, [nef.grid.num_lods - 1])
        opt.step()
        assert abs(loss - ref_loss) <= 1e-4 * abs(ref_loss), (s, loss, ref_loss)
        for n, gr in grads.items():
            small[n] |= np.abs(gr) < 1e-4 * np.abs(gr).max()
    ref_p = dict(ref_nef.named_parameters())
    for n, p in nef.named_parameters():
        d = np.abs(p.detach().cpu().numpy() - ref_p[n].detach().cpu().numpy())
        lr_g = lr * (glw if n.startswith("grid.") else 1.0)
        assert d[~small[n]].max(initial=0.0) <= 1e-6 * lr_g / 1e-3, n
        assert d.max() <= 2 * lr_g * steps, n


def test_deep_launch_count(W):
    """An only_last fused step is two library launches: wb_sdf_train and wb_adam_step."""
    nef, case = _config3_l2(W)
    step = W.SDFStep(W.Pipeline(nef))
    assert step.fused
    coords, gt = _points(case, 512)
    step.step(coords, gt)
    before = W._cabi.launch_count()
    step.step(coords, gt)
    assert W._cabi.launch_count() - before == 2
    torch.cuda.synchronize()


@pytest.mark.parametrize("F,native", [(16, True), (17, False)])
def test_deep_footprint_boundary(W, F, native):
    """'cat' of 3 LODs + identity input, 2 hidden layers of 128: in 51 (in_pad 52) fits with a 32-sample tile, in 54 (in_pad 56)
    does not; the native route and the autograd fallback both agree with autograd and neither raises."""
    case = DS.case_of(5, 3, F, "cat")
    blas = W.OctreeAS(dev(case["octree"]))
    torch.manual_seed(0)
    grid = W.OctreeGrid(blas, feature_dim=F, num_lods=3, multiscale_type="cat", feature_std=0.05)
    nef = W.NeuralSDF(grid, pos_embedder="none", position_input=True, hidden_dim=128, num_layers=2).cuda()
    lin = list(nef.decoder.layers) + [nef.decoder.lout]
    Ws, bs = S.random_decoder(np.random.default_rng(0), lin[0].in_features, 1, 128, 2, scale=0.2)
    with torch.no_grad():
        for l, Wm, b in zip(lin, Ws, bs):
            l.weight.copy_(dev(Wm)); l.bias.copy_(dev(b))
    assert W.ops.sdf_field(nef) is not None                      # wb_sdf_eval evaluates both
    assert (_smem(W, nef) > 0) == native
    coords, gt = DS.points(case, 3000, seed=2)
    _vs_autograd(W, nef, dev(coords), dev(gt[:, None]), True, native)
