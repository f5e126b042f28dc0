"""SDFStep (SDFTrainer.step + BaseTrainer.init_optimizer) on the GPU: the fused wb_sdf_train route against the reference trainer's
own three steps (tests/golden/sdf_train.npz), against this package's autograd route at BASELINE config-3 shapes, against the
evaluation kernel, over a 5-step trajectory, and the autograd fallback for fields outside the fused kernel."""
import os

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


def _dec_parts(nef, flat):
    """flat decoder buffer -> {reference parameter name: tensor} in the packed order [W0, b0, Wout, bout]."""
    out, o = {}, 0
    for n, p in nef.named_parameters():
        if n.startswith("decoder."):
            out[n] = flat[o:o + p.numel()].view_as(p); o += p.numel()
    return out


def _step_grads(nef, step):
    g = {f"grid.features.{k}": t for k, t in enumerate(step.g_feats)}
    g.update(_dec_parts(nef, step.g_dec))
    return {k: v.detach().cpu().numpy() for k, v in g.items()}


# ---------------------------------------------------------------------------------------------------------------
# 1. the reference trainer's own steps
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", ["sum", "cat", "sum_all"])
def test_sdf_step_golden(W, golden_dir, case):
    """Step-1 gradients (2e-2 of max: the fp16-feature tolerance of test_octree_grid_golden), three losses (2e-3 relative),
    untouched grid rows bit-identical after step 1, and Adam's first step a sign step of every group's learning rate."""
    g = np.load(os.path.join(golden_dir, "sdf_train.npz"))
    ms = str(g[f"{case}_multiscale"])
    only_last = len(g[f"{case}_loss_lods"]) == 1
    lr, wd, glw = float(g["lr"]), float(g["weight_decay"]), float(g["grid_lr_weight"])
    blas = W.OctreeAS(dev(g["octree"]))
    grid = W.OctreeGrid(blas, feature_dim=8, num_lods=3, multiscale_type=ms, feature_std=0.0)
    nef = W.NeuralSDF(grid, pos_embedder='none', position_input=True, hidden_dim=16, num_layers=1).cuda()
    names = [n for n, p in nef.named_parameters() if p.requires_grad]
    with torch.no_grad():
        for n, p in nef.named_parameters():
            p.copy_(dev(g[f"{case}_init_{n}"]))
    step = W.SDFStep(W.Pipeline(nef), lr=lr, eps=float(g["eps"]), weight_decay=wd, grid_lr_weight=glw, only_last=only_last)
    assert step.fused
    coords, sdf = dev(g["coords"]), dev(g["sdf"])
    step.step(coords, sdf, update=False)
    got = _step_grads(nef, step)
    for n in names:
        ref = g[f"{case}_grad1_{n}"]
        assert np.abs(got[n] - ref).max() <= 2e-2 * max(np.abs(ref).max(), 1e-12), n
    step.zero_grads()
    losses = []
    for s in range(3):
        losses.append(float(step.step(coords, sdf)))
        if s == 0:
            for n, p in nef.named_parameters():
                init, ref_g, now = g[f"{case}_init_{n}"], g[f"{case}_grad1_{n}"], p.detach().cpu().numpy()
                if n.startswith("grid."):
                    # the scatter wrote nothing else: where the reference's gradient is zero, ours is zero too, or below the fp16
                    # underflow of the reference's gradient (each loss LOD's gradient flows through feats.half(), octree_grid.py:147,
                    # which flushes magnitudes below 2^-25 to zero); untouched rows keep their initial bits (no weight decay on grids)
                    zero = ref_g == 0
                    assert np.abs(got[n][zero]).max(initial=0.0) <= len(g[f"{case}_loss_lods"]) * 2.0 ** -24, n
                    untouched = zero & (got[n] == 0)
                    assert untouched.any() and np.array_equal(now[untouched], init[untouched]), n
                    lr_g, eff = lr * glw, ref_g
                else:
                    lr_g, eff = lr, ref_g + wd * init
                big = np.abs(eff) > 1e-3 * np.abs(eff).max()
                assert big.any(), n
                np.testing.assert_allclose(now[big], (init - lr_g * np.sign(eff))[big], atol=1e-6, err_msg=n)
    np.testing.assert_allclose(losses, g[f"{case}_losses"], rtol=2e-3)


# ---------------------------------------------------------------------------------------------------------------
# 2.-6. the package's own autograd route
# ---------------------------------------------------------------------------------------------------------------
_CASES = {}


def _octahedron(level):
    from oracle import octree_grid as OG
    if level not in _CASES:
        _CASES[level] = OG.make_sdf_case(level=level, num_lods=6, feature_dim=16, hidden_dim=128, multiscale="sum", res=4, seed=11, feature_std=0.02)
    return _CASES[level]


def _field(W, shape, seed=0):
    """'config3': BASELINE config 3 (level-7 octahedron, F = 16, 6 LODs 'sum', 19-128-1); 'cat8': 'cat', F = 8, positional
    embedding with the input, H = 64; 'sum4': 'sum', F = 4, no position input, H = 32."""
    from gpu_util import sdf_nef_from_case
    case = _octahedron(7)
    if shape == "config3":
        return sdf_nef_from_case(case), case
    torch.manual_seed(seed)
    blas = W.OctreeAS(dev(case["octree"]))
    if shape == "cat8":
        grid = W.OctreeGrid(blas, feature_dim=8, num_lods=6, multiscale_type='cat', feature_std=0.05)
        nef = W.NeuralSDF(grid, pos_embedder='positional', pos_multires=4, position_input=True, hidden_dim=64, num_layers=1)
    else:
        grid = W.OctreeGrid(blas, feature_dim=4, num_lods=6, multiscale_type='sum', feature_std=0.05)
        nef = W.NeuralSDF(grid, pos_embedder='none', position_input=False, hidden_dim=32, num_layers=1)
    return nef.cuda(), case


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


@pytest.mark.parametrize("shape,N,only_last", [("config3", 1, True), ("config3", 1000, True), ("config3", 65536, True), ("config3", 65536, False),
                                               ("cat8", 1, True), ("cat8", 1000, True), ("cat8", 65536, True),
                                               ("sum4", 1, True), ("sum4", 1000, True), ("sum4", 65536, True), ("sum4", 65536, False)])
def test_sdf_step_fused_vs_autograd(W, shape, N, only_last):
    """step(update=False) against nef(...) + torch loss + .backward(): loss 1e-5 relative, every gradient 1e-4 of its max
    (fp32, atomic summation order).  N = 1 and 1000 leave partial tiles."""
    nef, case = _field(W, shape)
    step = W.SDFStep(W.Pipeline(nef), only_last=only_last)
    assert step.fused
    coords, gt = _points(case, N)
    loss = float(step.step(coords, gt, update=False))
    got = _step_grads(nef, step)
    ref_loss, ref = _autograd(nef, coords, gt, step.loss_lods)
    assert abs(loss - ref_loss) <= 1e-5 * abs(ref_loss), (loss, ref_loss)
    for n, r in ref.items():
        assert np.abs(got[n] - r).max() <= 1e-4 * max(np.abs(r).max(), 1e-30), (n, np.abs(got[n] - r).max(), np.abs(r).max())


def test_sdf_step_cat_all_lods_refused(W):
    nef, case = _field(W, "cat8")
    step = W.SDFStep(W.Pipeline(nef), only_last=False)
    coords, gt = _points(case, 64)
    with pytest.raises(RuntimeError, match="cannot be multiplied"):
        step.step(coords, gt)


@pytest.mark.parametrize("shape", ["config3", "cat8"])
def test_sdf_step_loss_is_eval_loss(W, shape):
    """The kernel's forward is wb_sdf_eval: its loss equals the loss of ops.sdf_eval's predictions to 1e-6 relative."""
    nef, case = _field(W, shape)
    step = W.SDFStep(W.Pipeline(nef))
    coords, gt = _points(case, 65536, seed=9)
    loss = float(step.step(coords, gt, update=False))
    with torch.no_grad():
        y = W.ops.sdf_eval(nef, coords, nef.grid.num_lods - 1).double()
    ref = float(((y - gt.double()) ** 2).sum() / coords.shape[0])
    assert abs(loss - ref) <= 1e-6 * ref, (loss, ref)


def _torch_adam(nef, lr, wd, glw, eps):
    """BaseTrainer.init_optimizer's groups (base_trainer.py:205-239) over torch.optim.Adam."""
    dec, grd, rest = [], [], []
    for n, p in nef.named_parameters():
        if not p.requires_grad:
            continue
        (dec if "decoder" in n else grd if "grid" in n else rest).append(p)
    return torch.optim.Adam([{"params": dec, "lr": lr, "eps": eps, "weight_decay": wd}, {"params": grd, "eps": eps, "lr": lr * glw},
                             {"params": rest, "eps": eps, "lr": lr}], lr=lr, eps=eps)


def test_sdf_step_trajectory(W):
    """Five SDFStep steps against autograd + torch.optim.Adam with the reference's groups: losses 1e-4 relative at every step,
    parameters 1e-6 per 1e-3 of their group's learning rate, except entries whose gradient was ever below 1e-4 of max (Adam's
    normalisation amplifies atomic-order noise there): within 2 lr steps."""
    lr, wd, glw, eps, steps = 1e-3, 1e-2, 5.0, 1e-15, 5
    nef, case = _field(W, "config3")
    ref_nef, _ = _field(W, "config3")
    step = W.SDFStep(W.Pipeline(nef), lr=lr, eps=eps, weight_decay=wd, grid_lr_weight=glw)
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
        assert d.max() <= 2 * lr * (glw if n.startswith("grid.") else 1.0) * steps, n


@pytest.mark.parametrize("kind", ["hash", "triplanar"])
def test_sdf_step_fallback(W, kind):
    """A NeuralSDF over a HashGrid (nglod_hash.yaml, scaled down) or a TriplanarGrid (nglod_triplanar.yaml) trains through
    SDFStep's autograd route: one step matches autograd + torch.optim.Adam with the reference's groups to 1e-6."""
    lr, wd, glw, eps = 1e-3, 1e-2, 5.0, 1e-15
    case = _octahedron(7)
    nets = []
    for _ in range(2):
        torch.manual_seed(3)
        blas = W.OctreeAS(dev(case["octree"]))
        if kind == "hash":
            grid = W.HashGrid.from_geometric(blas, feature_dim=2, num_lods=8, multiscale_type='cat', feature_std=0.01, codebook_bitwidth=14,
                                             min_grid_res=16, max_grid_res=256)
        else:
            grid = W.TriplanarGrid(blas, feature_dim=4, log_base_resolution=5, num_lods=1, multiscale_type='sum', feature_std=0.01)
        nets.append(W.NeuralSDF(grid, pos_embedder='positional', pos_multires=4, position_input=True, hidden_dim=64, num_layers=1).cuda())
    nef, ref_nef = nets
    step = W.SDFStep(W.Pipeline(nef), lr=lr, eps=eps, weight_decay=wd, grid_lr_weight=glw)
    assert not step.fused
    opt = _torch_adam(ref_nef, lr, wd, glw, eps)
    coords, gt = _points(case, 4096, seed=4)
    loss = float(step.step(coords, gt))
    ref_loss, _ = _autograd(ref_nef, coords, gt, [ref_nef.grid.num_lods - 1])
    opt.step()
    assert abs(loss - ref_loss) <= 1e-6 * abs(ref_loss)
    ref_p = dict(ref_nef.named_parameters())
    for n, p in nef.named_parameters():
        np.testing.assert_allclose(p.detach().cpu().numpy(), ref_p[n].detach().cpu().numpy(), atol=1e-6, err_msg=n)


def test_sdf_step_launch_count(W):
    """An only_last fused step is two library launches: wb_sdf_train and wb_adam_step (counted, not timed)."""
    nef, case = _field(W, "config3")
    step = W.SDFStep(W.Pipeline(nef))
    coords, gt = _points(case, 512)
    step.step(coords, gt)
    before = W._cabi.launch_count()
    step.step(coords, gt)
    assert W._cabi.launch_count() - before == 2
    torch.cuda.synchronize()
