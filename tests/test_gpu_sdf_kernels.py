"""The NeuralSDF(OctreeGrid) kernels -- wb_sdf_eval, wb_sdf_trace, wb_sdf_train -- and wb_octree_interp_bwd against the float64
interval reference oracle/sdf_reference.py, over the field shapes ops.sdf_field sends to them: both compiled instances (<16,1> for
the app/nglod shape, <0,0> for everything else), position embeddings, 'cat' and 'sum', F up to 64, 1 to 4 hidden layers,
half_features on and off, every lod_idx.  Samples the reference flags as ambiguous (a relu decision within the rounding radius) are
dropped before the launch; every remaining output must lie in centre +- radius."""
import numpy as np
import pytest
import torch

from oracle import octree_grid as OG
from oracle import sdf_reference as S

pytestmark = pytest.mark.gpu

SMEM_PER_SM, SMEM_PER_CTA_RESERVED = 228 * 1024, 1024       # H100


@pytest.fixture(scope="module")
def W():
    import wisp_b200
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return wisp_b200


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


from sdf_shapes import SHAPES, TRAINABLE, case_of, make_field, points


def nef_of(W, field, case):
    """W.NeuralSDF with the field's octree, features and decoder."""
    blas = W.OctreeAS(dev(case["octree"]))
    grid = W.OctreeGrid(blas, feature_dim=field.F, num_lods=field.num_lods, multiscale_type=field.multiscale, feature_std=0.0)
    assert grid.base_lod == field.base_lod and np.array_equal(grid.trinkets.cpu().numpy(), field.trinkets)
    grid.half_features = field.half
    pos = {0: ("none", False), 1: ("none", True), 2: ("positional", False), 3: ("positional", True)}[field.pos_mode]
    nef = W.NeuralSDF(grid, pos_embedder=pos[0], pos_multires=max(field.pos_freq, 1), position_input=pos[1], hidden_dim=field.Ws[0].shape[0],
                      num_layers=len(field.Ws) - 1).cuda()
    with torch.no_grad():
        for f, ref in zip(grid.features, field.feats):
            f.copy_(dev(ref))
        for l, Wm, b in zip(list(nef.decoder.layers) + [nef.decoder.lout], field.Ws, field.bs):
            l.weight.copy_(dev(Wm)); l.bias.copy_(dev(b))
    return nef


def inside(got, c, r, what):
    err = np.abs(np.asarray(got, np.float64) - c)
    bad = err > r
    assert not bad.any(), (what, int(bad.sum()), float(err.max()), float((err - r).max()), float(np.abs(c).max()))


def drop_ambiguous(field, coords, gt, lods):
    amb = np.zeros(coords.shape[0], bool)
    for lod in lods:
        amb |= S.forward(field, coords, lod).amb
    assert amb.mean() <= 0.02, amb.mean()
    return coords[~amb], gt[~amb]


# ---------------------------------------------------------------------------------------------------------------
# wb_sdf_eval
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(SHAPES))
def test_sdf_eval_vs_reference(W, name):
    field, case = make_field(name)
    nef = nef_of(W, field, case)
    lods = range(field.num_lods) if field.multiscale == "sum" else [field.num_lods - 1]
    for lod in lods:
        coords, _ = points(case, 1000, seed=lod)
        coords, _ = drop_ambiguous(field, coords, coords[:, 0], [lod])
        got = W.ops.sdf_eval(nef, dev(coords), lod)
        assert got is not None, name
        fw = S.forward(field, coords, lod)
        inside(got.cpu().numpy()[:, 0], fw.y, fw.y_r, (name, lod))


# ---------------------------------------------------------------------------------------------------------------
# wb_sdf_train
# ---------------------------------------------------------------------------------------------------------------
def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _ctas_per_sm_bound(field):
    """Upper bound of wb_sdf_train's occupancy: its shared memory (the launch's formula) and the 2048 threads of an SM."""
    H, in_dim = field.Ws[0].shape[0], field.Ws[0].shape[1]
    in_pad = (in_dim + 3) & ~3
    fast = field.multiscale == "sum" and field.F == 16 and field.pos_mode == 1
    smem_floats = H * in_pad + H + H + 4
    xs = (smem_floats + 3) & ~3
    red = xs + S.TILE * in_pad + S.TILE + (0 if fast else H * (in_pad + 1))
    smem = (red + 2 * (S.TILE // 32)) * 4
    return max(1, min(S.MAX_CTAS_PER_SM, SMEM_PER_SM // (smem + SMEM_PER_CTA_RESERVED)))


def fused_step(W, nef, coords, gt, only_last=True):
    step = W.SDFStep(W.Pipeline(nef), only_last=only_last)
    assert step.fused
    loss = float(step.step(dev(coords), dev(gt), update=False))
    torch.cuda.synchronize()
    return loss, step.g_dec.cpu().numpy().astype(np.float64), [g.cpu().numpy().astype(np.float64) for g in step.g_feats], step


def check_train(W, field, case, coords, gt, only_last=True, what=""):
    lods = [field.num_lods - 1] if only_last else list(range(field.num_lods))
    ref = S.train(field, coords, gt, lods, sms=_sms())
    assert ref.amb.mean() <= 0.02, ref.amb.mean()
    if ref.amb.any():                                  # drop the ambiguous samples from the batch
        coords, gt = coords[~ref.amb], gt[~ref.amb]
        ref = S.train(field, coords, gt, lods, sms=_sms())
        assert not ref.amb.any()
    nef = nef_of(W, field, case)
    loss, dec, grid, _ = fused_step(W, nef, coords, gt, only_last)
    inside(loss, ref.loss, ref.loss_r, ("loss", what))
    inside(dec, ref.dec, ref.dec_r, ("decoder", what))
    for k, (g, (c, r)) in enumerate(zip(grid, ref.grid)):
        inside(g, c, r, ("grid", k, what))
        assert np.all(g[c == 0][r[c == 0] == 0] == 0), ("untouched rows", k, what)      # rows no sample reaches stay 0


@pytest.mark.parametrize("name", TRAINABLE)
def test_sdf_train_vs_reference(W, name):
    field, case = make_field(name)
    coords, gt = points(case, 1000, seed=3)
    check_train(W, field, case, coords, gt, what=name)
    if field.multiscale == "sum":
        check_train(W, field, case, coords, gt, only_last=False, what=name + " all LODs")


@pytest.mark.parametrize("name", ["fast_1lod", "widest"])
@pytest.mark.parametrize("N", [1, 127, 128, 129, 1000, "tiles3"])
def test_sdf_train_batch_sizes(W, name, N):
    """Partial tiles, and a batch in which every CTA of the launch runs at least three 128-sample tiles."""
    field, case = make_field(name, seed=1)
    if N == "tiles3":
        N = 3 * S.TILE * _sms() * _ctas_per_sm_bound(field)
    coords, gt = points(case, N, seed=N % 97)
    check_train(W, field, case, coords, gt, what=(name, N))


def test_sdf_train_contract(W):
    """Accumulates into the buffers passed in; N = 0 changes nothing; an all-LOD 'sum' loss is the sum of the per-LOD launches."""
    field, case = make_field("sum_pos3")
    nef = nef_of(W, field, case)
    coords, gt = points(case, 700, seed=8)
    coords, gt = drop_ambiguous(field, coords, gt, range(field.num_lods))
    fd = W.ops.sdf_field(nef)
    c, g = dev(coords), dev(gt)
    def launch(lod, gf, gp, loss, n=None):
        if n is None:
            W.ops.sdf_train(fd, c, g, lod, 1.0 / coords.shape[0], gf, gp, loss)
        else:                                                  # the C ABI with valid pointers and N = n
            import ctypes as C
            A = W._cabi
            gptrs = (C.c_void_p * len(gf))(*[t.data_ptr() for t in gf])
            A.check(A.lib().wb_sdf_train(C.byref(fd[1].desc()), C.byref(fd[0]), C.c_int32(lod), A.ptr(c), A.ptr(g), C.c_int64(n),
                                         C.c_float(1.0), gptrs, A.ptr(gp), A.ptr(loss), A.stream()))
        torch.cuda.synchronize()
    rng = np.random.default_rng(0)
    init_f = [np.float32(2.0 ** -8) * rng.integers(-64, 64, f.shape).astype(np.float32) for f in field.feats]
    init_p = np.float32(2.0 ** -8) * rng.integers(-64, 64, field.packed().size).astype(np.float32)
    gf, gp, loss = [dev(f) for f in init_f], dev(init_p), torch.full((1,), 0.25, device="cuda")
    launch(field.num_lods - 1, gf, gp, loss, n=0)
    assert all(np.array_equal(a.cpu().numpy(), b) for a, b in zip(gf, init_f)) and np.array_equal(gp.cpu().numpy(), init_p)
    assert float(loss) == 0.25
    for lod in range(field.num_lods):
        launch(lod, gf, gp, loss)
    ref = S.train(field, coords, gt, list(range(field.num_lods)), sms=_sms())
    # every atomic now also rounds relative to the initial value: n atomics add gamma(n) |init|
    inside(float(loss) - 0.25, ref.loss, ref.loss_r + S.g32(ref.atomics) * 0.25, "loss")
    inside(gp.cpu().numpy().astype(np.float64) - init_p, ref.dec, ref.dec_r + S.g32(ref.atomics) * np.abs(init_p), "decoder")
    for k, (a, (cc, r)) in enumerate(zip(gf, ref.grid)):
        inside(a.cpu().numpy().astype(np.float64) - init_f[k], cc, r + S.g32(ref.grid_n[k])[:, None] * np.abs(init_f[k]), ("grid", k))
    # the all-LOD step of SDFStep equals the sum of its per-LOD launches (to 2^-20: the CTAs' atomics add in any order)
    loss_all, *_ = fused_step(W, nef, coords, gt, only_last=False)
    per = torch.zeros(1, device="cuda")
    z = [torch.zeros_like(t) for t in gf]
    for lod in range(field.num_lods):
        launch(lod, z, torch.zeros_like(gp), per)
    assert abs(loss_all - float(per)) <= 2.0 ** -20 * abs(float(per))


# ---------------------------------------------------------------------------------------------------------------
# wb_sdf_trace, <0,0> instance
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name,lod", [("l3_h128", None), ("l2_h64", None), ("sum_pos3", 1), ("l4_h124", 0)])
def test_sdf_trace_generic_vs_reference(W, name, lod):
    field, case = make_field(name)
    # a field with |grad| ~ 1: where the SDF is steeper than 1 sphere tracing overshoots and fp32 differences change where it stops
    field.Ws[-1][:, 6:] *= 0.1
    field.Ws[0][:, 3:field.pos_dim] *= 0.02 if field.pos_mode == 3 else 1.0
    nef = nef_of(W, field, case)
    lod_idx = field.num_lods - 1 if lod is None else lod
    tracer = W.PackedSDFTracer(num_steps=32, step_size=0.8, min_dis=1e-3)
    rb = tracer(nef, rays=W.Rays(dev(case["origins"]), dev(case["dirs"]), dist_min=0.0, dist_max=6.0), lod_idx=lod_idx,
                channels=["depth", "hit", "normal", "xyz"])
    f32 = lambda x, l=None: S.forward(field, x, l).y.astype(np.float32)[:, None]
    ref = OG.sdf_trace(case, num_steps=32, step_size=0.8, min_dis=1e-3, lod_idx=lod_idx, field=f32)
    hit, ref_hit = rb.hit.cpu().numpy(), ref["hit"]
    assert ref_hit.sum() > 20 and (hit != ref_hit).mean() <= 0.002
    both = hit & ref_hit
    np.testing.assert_allclose(rb.xyz.cpu().numpy()[both], ref["xyz"][both], atol=1e-4)
    np.testing.assert_allclose(rb.depth.cpu().numpy()[both], ref["depth"][both], atol=1e-4)
    dots = (rb.normal.cpu().numpy()[both] * ref["normal"][both]).sum(-1)
    assert np.quantile(dots, 0.01) > 0.999


# ---------------------------------------------------------------------------------------------------------------
# wb_octree_interp_bwd in fp32
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("ms,F,num_lods", [("cat", 5, 3), ("sum", 7, 6), ("cat", 3, 6)])
def test_octree_interp_bwd_fp32(W, ms, F, num_lods):
    case = case_of(5, num_lods, F, ms)
    field = S.Field(case["spc"], case["trinkets"], case["feats"], case["active_lods"][0], ms, [], [], 1, 0, False)
    blas = W.OctreeAS(dev(case["octree"]))
    grid = W.OctreeGrid(blas, feature_dim=F, num_lods=num_lods, multiscale_type=ms, feature_std=0.0).cuda()
    grid.half_features = False
    with torch.no_grad():
        for f, ref in zip(grid.features, case["feats"]):
            f.copy_(dev(ref))
    coords, _ = points(case, 3000, seed=4)
    lod = num_lods - 1
    go = np.random.default_rng(5).standard_normal((coords.shape[0], F if ms == "sum" else F * num_lods)).astype(np.float32)
    grid.interpolate(dev(coords), lod).backward(dev(go))
    for k, (c, r) in enumerate(S.interp_backward(field, coords, go, lod)):
        g = grid.features[k].grad.cpu().numpy()
        inside(g, c, r, (ms, k))
        assert np.all(g[c == 0] == 0)


# ---------------------------------------------------------------------------------------------------------------
# native or fallback, never an error
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("layers,H,pos,native", [(4, 124, "id", True), (3, 128, "wide", True), (4, 128, "id", False), (4, 120, "wide", False)])
def test_decoder_shared_memory_boundary(W, layers, H, pos, native):
    """in 19 ('sum' F 16 + identity) or in 132 ('cat' F 23 x 3 + 10 frequencies with the input): images up to 200 KB run natively,
    larger ones fall back to the autograd route; neither raises."""
    case = case_of(5, 3, 16 if pos == "id" else 23, "sum" if pos == "id" else "cat")
    blas = W.OctreeAS(dev(case["octree"]))
    torch.manual_seed(0)
    grid = W.OctreeGrid(blas, feature_dim=case["feature_dim"], num_lods=3, multiscale_type=case["multiscale"], feature_std=0.05)
    nef = W.NeuralSDF(grid, pos_embedder="none" if pos == "id" else "positional", pos_multires=10, position_input=True, hidden_dim=H,
                      num_layers=layers).cuda()
    lin = list(nef.decoder.layers) + [nef.decoder.lout]
    Ws, bs = S.random_decoder(np.random.default_rng(0), lin[0].in_features, 1 if pos == "id" else 3, H, layers, scale=0.2)
    Ws[-1][:, 6:] *= 0.1                                             # an SDF-like field with a surface to trace
    Ws[0][:, 3:63] *= 1.0 if pos == "id" else 0.02
    with torch.no_grad():
        for l, Wm, b in zip(lin, Ws, bs):
            l.weight.copy_(dev(Wm)); l.bias.copy_(dev(b))
    coords, _ = points(case, 2000, seed=2)
    c = dev(coords)
    fused = W.ops.sdf_eval(nef, c, 2)
    assert (fused is not None) == native
    ref = nef(coords=c, lod_idx=2, channels="sdf").detach()          # autograd route: native grid kernel + torch decoder
    with torch.no_grad():
        got = nef(coords=c, lod_idx=2, channels="sdf")
    tol = 1e-5 * float(ref.abs().max())
    assert float((got - ref).abs().max()) <= (tol if native else 0.0)
    # PackedSDFTracer against the same tracer over the autograd route's SDF
    rays = W.Rays(dev(case["origins"]), dev(case["dirs"]), dist_min=0.0, dist_max=6.0)
    rb = W.PackedSDFTracer(num_steps=16, step_size=0.8, min_dis=1e-3)(nef, rays=rays, lod_idx=2, channels=["depth", "hit", "xyz"])
    def autograd_sdf(x, lod=None):
        with torch.enable_grad():
            return nef(coords=dev(x), lod_idx=2 if lod is None else lod, channels="sdf").detach().cpu().numpy().reshape(-1, 1)
    ref = OG.sdf_trace(case, num_steps=16, step_size=0.8, min_dis=1e-3, lod_idx=2, field=autograd_sdf, with_normals=False)
    hit = rb.hit.cpu().numpy()
    assert ref["hit"].sum() > 20 and (hit != ref["hit"]).mean() <= 0.002
    both = hit & ref["hit"]
    np.testing.assert_allclose(rb.xyz.cpu().numpy()[both], ref["xyz"][both], atol=1e-4)
    np.testing.assert_allclose(rb.depth.cpu().numpy()[both], ref["depth"][both], atol=1e-4)
