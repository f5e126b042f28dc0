"""GPU parity tests (-m gpu): the CUDA path, called through the product package / C ABI, against
  (1) the golden fixtures produced by the unmodified reference Python, and
  (2) the CPU oracle on seeded inputs.
Tolerances: indices and sample floats bit-exact; fp32 decoders: rgb/alpha 1e-4 abs, depth 5e-4 abs (depth sums
weights times distances up to 10); gradients rtol 1e-3 of the largest entry (atomic summation order)."""
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import oracle as O
from golden_util import load_case

CASES = ["rf_trace_cat", "rf_trace_sum", "rf_trace_noview"]


@pytest.fixture(scope="module")
def W():
    import wisp_b200
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return wisp_b200


def dev(a, dtype=None):
    t = torch.from_numpy(np.ascontiguousarray(a))
    if dtype is not None:
        t = t.to(dtype)
    return t.cuda()


def test_library_is_native_and_device_ok(W):
    assert W._cabi.lib().wb_version() >= 100
    W._cabi.require_device(torch.zeros(1, device="cuda"))
    assert os.path.exists(W._cabi.LIB_PATH)


def test_torch_cuda_contract():
    """The bit-exact contract for sample generation restates what the reference's torch CUDA kernels compute:
    addcmul == fma(dir, t, origin); linspace lower/upper halves FMA-contracted (see wb_common.cuh)."""
    g = torch.Generator().manual_seed(0)
    a, b = torch.randn(1 << 16, generator=g), torch.randn(1 << 16, generator=g)
    c = torch.rand(1 << 16, generator=g) * 10
    t = torch.addcmul(a.cuda(), b.cuda(), c.cuda()).cpu().numpy()
    fma = (a.double() + b.double() * c.double()).float().numpy()          # fused: one rounding
    unf = (a + (b * c)).numpy()
    frac_fma, frac_unf = float((t == fma).mean()), float((t == unf).mean())
    print("addcmul cuda: ==fma", frac_fma, "==unfused", frac_unf)
    n = 2048
    ls = torch.linspace(0, 1, n, device="cuda").cpu().numpy()
    step = np.float32(1.0) / np.float32(n - 1)
    i = np.arange(n)
    lo = (np.float64(step) * i).astype(np.float32)
    hi = (1.0 - np.float64(step) * (n - 1 - i)).astype(np.float32)
    ref = np.where(i < n // 2, lo, hi)
    frac_ls = float((ls == ref).mean())
    print("linspace cuda == contract", frac_ls)
    os.makedirs("gpurun_out", exist_ok=True)
    with open("gpurun_out/contract.txt", "w") as f:
        f.write(f"addcmul_eq_fma {frac_fma}\naddcmul_eq_unfused {frac_unf}\nlinspace_eq_contract {frac_ls}\n")
    assert frac_fma == 1.0
    assert frac_ls == 1.0


def test_query_bit_exact(W):
    rng = np.random.default_rng(0)
    spc = O.octree_to_spc(O.points_to_octree(O.lego_like_points(6), 6))
    coords = rng.uniform(-1.05, 1.05, (200000, 3)).astype(np.float32)
    # exact cell faces and the +/-1 borders
    k = (rng.integers(0, 65, (4096, 3)) / 32.0 - 1.0).astype(np.float32)
    coords = np.concatenate([coords, k, np.nextafter(k, np.float32(-2)), np.nextafter(k, np.float32(2))])
    blas = W.OctreeAS(dev(spc.octree))
    for level in (6, 4):
        got = blas.query(dev(coords), level=level).pidx.cpu().numpy()
        assert np.array_equal(got, O.query(spc, coords, level))
    gp = blas.query(dev(coords), with_parents=True).pidx.cpu().numpy()
    assert np.array_equal(gp, O.query(spc, coords, with_parents=True))
    # the product's own host-side SPC builder agrees with the oracle's
    assert np.array_equal(blas.points.cpu().numpy(), spc.points)
    assert np.array_equal(blas.prefix.cpu().numpy(), spc.prefix)
    assert np.array_equal(blas.pyramid.cpu().numpy(), spc.pyramid)


@pytest.mark.parametrize("name", CASES)
def test_raymarch_golden_bit_exact(W, golden_dir, name):
    g, onef, spc = load_case(os.path.join(golden_dir, name + ".npz"))
    blas = W.OctreeAS(dev(spc.octree))
    rays = W.Rays(dev(g["origins"]), dev(g["dirs"]), dist_min=float(g["near"]), dist_max=float(g["far"]))
    mr = blas.raymarch(rays, 'ray', int(g["n_steps"]), jitter=dev(g["jitter"]))
    assert np.array_equal(mr.ridx.cpu().numpy(), g["mr_ridx"])
    assert np.array_equal(mr.boundary.cpu().numpy(), g["mr_boundary"])
    assert np.array_equal(mr.samples.cpu().numpy(), g["mr_samples"])
    assert np.array_equal(mr.depth_samples.cpu().numpy(), g["mr_depth"])
    assert np.array_equal(mr.deltas.cpu().numpy(), g["mr_deltas"])
    assert mr.ridx.dtype == torch.int64 and mr.boundary.dtype == torch.bool and mr.pack_info is None


@pytest.mark.parametrize("n,level,pernear", [(2048, 7, False), (100, 5, False), (33, 5, True), (1, 4, False)])
def test_raymarch_seeded_vs_oracle(W, n, level, pernear):
    """Counter-based jitter stream, non power-of-two n, per-ray near/far, n == 1; bit-exact vs the oracle."""
    spc = O.octree_to_spc(O.points_to_octree(O.lego_like_points(level), level))
    o, d = O.look_at_rays([-3.0, 0.65, -3.0], [0, 0, 0], 48, 48, 30.0)
    blas = W.OctreeAS(dev(spc.octree))
    if pernear:
        rng = np.random.default_rng(1)
        near = rng.uniform(0.0, 2.0, o.shape[0]).astype(np.float32); far = (near + rng.uniform(3.0, 8.0, o.shape[0])).astype(np.float32)
        rays = W.Rays(dev(o), dev(d), dist_min=dev(near)[:, None], dist_max=dev(far)[:, None])
    else:
        near, far = 0.0, 10.0
        rays = W.Rays(dev(o), dev(d), dist_min=near, dist_max=far)
    mr = blas.raymarch(rays, 'ray', n, seed=1234)
    ref = O.raymarch_ray(spc, o, d, near, far, n, seed=1234)
    assert np.array_equal(mr.ridx.cpu().numpy(), ref["ridx"])
    assert np.array_equal(mr.samples.cpu().numpy(), ref["samples"])
    assert np.array_equal(mr.depth_samples.cpu().numpy(), ref["depth_samples"])
    assert np.array_equal(mr.deltas.cpu().numpy(), ref["deltas"])
    assert np.array_equal(mr.boundary.cpu().numpy(), ref["boundary"])


@pytest.mark.parametrize("level,coarse,n", [(7, 6, 2048), (7, 5, 2048), (7, 3, 512), (6, 2, 100), (5, 3, 33), (5, 4, 64)])
def test_raymarch_word_skipping_is_exact(W, level, coarse, n):
    """The dilated coarse mask only skips 32-candidate words that cannot hold a sample: hit masks are identical with and
    without it, for camera rays, rays starting inside the volume, axis-aligned / grazing rays and unnormalised directions."""
    rng = np.random.default_rng(level * 10 + coarse)
    spc = O.octree_to_spc(O.points_to_octree(O.lego_like_points(level), level))
    o, d = O.look_at_rays([-3.0, 0.65, -3.0], [0, 0, 0], 40, 40, 30.0)
    oi = rng.uniform(-1.2, 1.2, (3000, 3)).astype(np.float32); di = rng.standard_normal((3000, 3)).astype(np.float32)
    di[:500] /= np.linalg.norm(di[:500], axis=1, keepdims=True)
    di[500:700] = np.eye(3, dtype=np.float32)[rng.integers(0, 3, 200)] * rng.choice([-1.0, 1.0], (200, 1)).astype(np.float32)   # axis aligned
    oi[700:900] = np.round(oi[700:900] * 2 ** (level - 1)) / 2 ** (level - 1)                                             # on cell faces
    di[900:1000] *= 7.5                                                                                                   # long directions
    o = np.concatenate([o, oi]); d = np.concatenate([d, di])
    from wisp_b200 import ops
    saved = ops.COARSE_LEVEL
    res = []
    try:
        for cl in (0, coarse):
            ops.COARSE_LEVEL = cl
            blas = W.OctreeAS(dev(spc.octree))
            ms = ops.march_count(blas.tensors(), dev(o), dev(d), 0.0, 6.0, n, level, seed=99)
            assert (blas.tensors().coarse is not None) == (cl > 0)
            res.append((ms.hitmask.cpu().numpy().copy(), ms.counts.cpu().numpy().copy(), ms.total))
    finally:
        ops.COARSE_LEVEL = saved
    assert res[0][2] == res[1][2] > 0
    assert np.array_equal(res[0][0], res[1][0]) and np.array_equal(res[0][1], res[1][1])


def test_raymarch_empty_and_errors(W):
    spc = O.octree_to_spc(O.points_to_octree(np.array([[0, 0, 0]], dtype=np.int16), 4))
    blas = W.OctreeAS(dev(spc.octree))
    o = np.tile(np.array([[5.0, 5.0, 5.0]], np.float32), (7, 1)); d = np.tile(np.array([[1.0, 0, 0]], np.float32), (7, 1))
    mr = blas.raymarch(W.Rays(dev(o), dev(d), 0.0, 1.0), 'ray', 16)
    assert mr.ridx.shape[0] == 0 and mr.samples.shape == (0, 3)
    with pytest.raises(TypeError):
        blas.raymarch(W.Rays(dev(o), dev(d), 0.0, 1.0), 'bogus', 16)          # octree_as.py:427
    mr0 = blas.raymarch(W.Rays(dev(o[:0]), dev(d[:0]), 0.0, 1.0), 'ray', 16)
    assert mr0.ridx.shape[0] == 0


def test_hashgrid_golden_naive(W, golden_dir):
    g = np.load(os.path.join(golden_dir, "hashgrid_naive.npz"))
    res = [int(r) for r in g["resolutions"]]; bw = int(g["codebook_bitwidth"])
    table = dev(g["table"]).requires_grad_(True)
    begin = torch.from_numpy(O.table_layout(res, bw))
    feats = W.ops.HashGridInterpolate.apply(dev(g["coords"]), torch.tensor(res), bw, len(res) - 1, table, begin)
    np.testing.assert_allclose(feats.detach().cpu().numpy(), g["feats"], atol=2e-6, rtol=1e-4)


@pytest.mark.parametrize("bw,F", [(19, 2), (12, 4), (14, 8)])
def test_hashgrid_fwd_bwd_vs_oracle(W, bw, F):
    rng = np.random.default_rng(3)
    res = O.geometric_resolutions(16, 16, 512)
    begin = O.table_layout(res, bw)
    table = rng.standard_normal((int(begin[-1]), F)).astype(np.float32)
    coords = rng.uniform(-1.0, 1.0, (30000, 3)).astype(np.float32)
    coords[:64] = np.sign(coords[:64])                       # corners / faces of the volume: clamp path
    t = dev(table).requires_grad_(True)
    feats = W.ops.HashGridInterpolate.apply(dev(coords), torch.tensor(res), bw, 15, t, torch.from_numpy(begin))
    ref = O.hashgrid_fwd(coords, table, res, bw)
    np.testing.assert_allclose(feats.detach().cpu().numpy(), ref, atol=1e-6, rtol=1e-5)
    go = rng.standard_normal(ref.shape).astype(np.float32)
    feats.backward(dev(go))
    gref = O.hashgrid_bwd(coords, go, table.shape[0], res, bw)
    scale = np.abs(gref).max()
    assert np.abs(t.grad.cpu().numpy() - gref).max() <= 1e-4 * scale


def test_composite_vs_oracle(W):
    rng = np.random.default_rng(5)
    R = 300
    counts = rng.integers(0, 90, R); counts[::7] = 0
    offsets = np.zeros(R + 1, np.int64); offsets[1:] = np.cumsum(counts)
    S = int(offsets[-1])
    shaded = np.concatenate([rng.random((S, 3)), rng.random((S, 1)) * 30], -1).astype(np.float32)
    deltas = (rng.random(S) * 0.01).astype(np.float32)
    depth = np.concatenate([np.sort(rng.random(c) * 10) for c in counts]).astype(np.float32)
    boundary = np.zeros(S, np.uint8); boundary[offsets[:-1][counts > 0]] = 1
    bg = (0.3, 0.6, 0.9)
    sh = dev(shaded).requires_grad_(True)
    rgb, dout, alpha, hit = W.ops.CompositeFn.apply(sh, dev(depth), dev(deltas), dev(offsets), bg)
    tau = shaded[:, 3] * deltas
    cols, w = O.exponential_integration(shaded[:, :3], tau, boundary)
    a = O.sum_reduce(w, boundary); dd = O.sum_reduce(w * depth[:, None], boundary)
    has = counts > 0
    exp_rgb = np.tile(np.array(bg, np.float32), (R, 1)); exp_rgb[has] = np.array(bg, np.float32) * (1 - a) + cols
    exp_a = np.zeros((R, 1), np.float32); exp_a[has] = a
    exp_d = np.zeros((R, 1), np.float32); exp_d[has] = dd
    np.testing.assert_allclose(rgb.detach().cpu().numpy(), exp_rgb, atol=2e-6)
    np.testing.assert_allclose(alpha.detach().cpu().numpy(), exp_a, atol=2e-6)
    np.testing.assert_allclose(dout.detach().cpu().numpy(), exp_d, atol=2e-5)
    assert np.array_equal(hit.cpu().numpy(), exp_a[:, 0] > 0)
    # backward against torch autograd of the twin formulas (CPU)
    from oracle import torch_twin as TW
    g1, g2, g3 = rng.standard_normal((R, 3)).astype(np.float32), rng.standard_normal((R, 1)).astype(np.float32), rng.standard_normal((R, 1)).astype(np.float32)
    (rgb * dev(g1)).sum().add((dout * dev(g2)).sum()).add((alpha * dev(g3)).sum()).backward()
    st = torch.from_numpy(shaded).requires_grad_(True)
    b = torch.from_numpy(boundary.astype(bool))
    c2, w2 = TW.exponential_integration(st[:, :3], st[:, 3:4] * torch.from_numpy(deltas)[:, None], b)
    a2 = TW.sum_reduce(w2, b); d2 = TW.sum_reduce(w2 * torch.from_numpy(depth)[:, None], b)
    rgb2 = torch.tensor(bg) * (1 - a2) + c2
    hs = torch.from_numpy(has)
    ((rgb2 * torch.from_numpy(g1)[hs]).sum() + (d2 * torch.from_numpy(g2)[hs]).sum() + (a2 * torch.from_numpy(g3)[hs]).sum()).backward()
    gref = st.grad.numpy()
    assert np.abs(sh.grad.cpu().numpy() - gref).max() <= 2e-5 * max(1.0, np.abs(gref).max())


def _run_fused(W, g, onef, spc, fused=True, precision=0):
    from gpu_util import nef_from_oracle, packed_grads
    nef, blas = nef_from_oracle(onef, spc)
    tracer = W.PackedRFTracer(raymarch_type='ray', num_steps=int(g["n_steps"]), bg_color=tuple(float(x) for x in g["bg"]))
    tracer.jitter = dev(g["jitter"])
    tracer.precision = precision
    pipe = W.Pipeline(nef, tracer)
    rays = W.Rays(dev(g["origins"]), dev(g["dirs"]), dist_min=float(g["near"]), dist_max=float(g["far"]))
    if not fused:
        nef.fused_spec = lambda lod_idx=None: None           # force the unfused route
    rb = pipe(rays=rays, channels=["rgb", "depth", "alpha", "hit"])
    return nef, tracer, rb


# (fused?, precision): precision 1 = fp16 tensor-core decoders, checked against the fp32 reference outputs with the
# AMP tolerance of BASELINE.md section 3 (2e-3 abs on rgb/alpha; the reference's own fp16 unit-test tolerance is 1e-2)
MODES = [(True, 0), (False, 0), (True, 1)]
TOL = {0: dict(rgb=1e-4, depth=5e-4, grad=1e-3, loss=1e-5), 1: dict(rgb=2e-3, depth=2e-2, grad=3e-2, loss=2e-3)}


@pytest.mark.parametrize("fused,precision", MODES)
@pytest.mark.parametrize("name", CASES)
def test_trace_golden(W, golden_dir, name, fused, precision):
    """Pipeline(nef, PackedRFTracer) forward + backward against what the reference's own classes produced."""
    from gpu_util import packed_grads
    g, onef, spc = load_case(os.path.join(golden_dir, name + ".npz"))
    nef, tracer, rb = _run_fused(W, g, onef, spc, fused, precision)
    tol = TOL[precision]
    assert tracer.get_prev_num_samples() == int(g["num_samples"])
    if precision == 0:
        assert np.array_equal(rb.hit.cpu().numpy(), g["hit"])
    np.testing.assert_allclose(rb.rgb.detach().cpu().numpy(), g["rgb"], atol=tol["rgb"], rtol=0)
    np.testing.assert_allclose(rb.alpha.detach().cpu().numpy(), g["alpha"], atol=tol["rgb"], rtol=0)
    np.testing.assert_allclose(rb.depth.detach().cpu().numpy(), g["depth"], atol=tol["depth"], rtol=0)
    target = dev(g["target"])
    lt = str(g["loss_type"])
    loss = {"huber": lambda: torch.nn.functional.smooth_l1_loss(rb.rgb, target), "l2": lambda: torch.nn.functional.mse_loss(rb.rgb, target),
            "l1": lambda: torch.abs(rb.rgb - target).mean()}[lt]()
    assert abs(float(loss.detach()) - float(g["loss"])) < tol["loss"]
    loss.backward()
    gt, gd, gc = packed_grads(nef)
    for got, ref, nm in ((gt, g["g_table"], "table"), (gd, g["g_dens"], "dens"), (gc, g["g_col"], "col")):
        scale = max(np.abs(ref).max(), 1e-12)
        assert np.abs(got - ref).max() <= tol["grad"] * scale, (nm, np.abs(got - ref).max(), scale)


def test_trace_follows_autocast(W, golden_dir):
    """tracer.precision = None: the fused path runs the tensor-core decoders exactly when torch autocast is on
    (the reference's `enable_amp`), the fp32 decoders otherwise."""
    g, onef, spc = load_case(os.path.join(golden_dir, CASES[0] + ".npz"))
    out = {}
    for key, prec, amp in (("p0", 0, False), ("p1", 1, False), ("auto_off", None, False), ("auto_on", None, True)):
        with torch.autocast("cuda", dtype=torch.float16, enabled=amp):
            _, _, rb = _run_fused(W, g, onef, spc, True, prec)
        out[key] = rb.rgb.detach().cpu().numpy()
    assert np.array_equal(out["auto_off"], out["p0"]) and np.array_equal(out["auto_on"], out["p1"])
    assert not np.array_equal(out["p0"], out["p1"])


def test_premarch_is_the_same_march(W, golden_dir):
    """PackedRFTracer.premarch (side stream, deferred sample count) + trace() == trace() alone, bit for bit; a premarch for other
    rays / another seed is ignored."""
    import copy
    g, onef, spc = load_case(os.path.join(golden_dir, CASES[0] + ".npz"))
    from gpu_util import nef_from_oracle
    nef, blas = nef_from_oracle(onef, spc)
    rays = W.Rays(dev(g["origins"]), dev(g["dirs"]), dist_min=float(g["near"]), dist_max=float(g["far"]))
    other = W.Rays(dev(g["origins"]).clone(), dev(g["dirs"]).clone(), dist_min=float(g["near"]), dist_max=float(g["far"]))
    outs = []
    for mode in ("direct", "premarch", "stale"):
        tracer = W.PackedRFTracer('ray', int(g["n_steps"]), bg_color=(1.0, 1.0, 1.0)); tracer.seed = 77
        if mode == "premarch":
            tracer.premarch(nef, rays, 77)
        if mode == "stale":
            tracer.premarch(nef, other, 77); tracer.premarch(nef, rays, 78)
        rb = W.Pipeline(nef, tracer)(rays=rays, channels=["rgb", "depth"])
        assert (len(tracer._pending) == 0) == (mode != "stale")
        copy.deepcopy(tracer)                                   # streams / pending marches are not part of the state
        outs.append((rb.rgb.detach().cpu().numpy(), rb.depth.detach().cpu().numpy(), tracer.get_prev_num_samples()))
    for o in outs[1:]:
        assert o[2] == outs[0][2] and np.array_equal(o[0], outs[0][0]) and np.array_equal(o[1], outs[0][1])


def test_nef_prune_golden(W, golden_dir):
    """NeuralRadianceField.prune() against what the REFERENCE class did (tests/golden/prune.npz: nerf.py:175-212 run through
    oracle/ref_import.py with a recorded torch.rand draw): same occupancy, same surviving cells, byte-identical rebuilt octree.
    Then properties of the native path: the marcher only samples kept cells; the default counter-based probe stream is
    deterministic per seed (what makes pruning rank-consistent); a second prune keeps decaying."""
    from golden_util import load_case
    from gpu_util import nef_from_oracle
    g, onef, spc = load_case(os.path.join(golden_dir, "prune.npz"))
    level = int(g["level"])

    def fresh():
        nef, blas = nef_from_oracle(onef, spc)
        nef.prune_density_decay, nef.prune_min_density = float(g["decay"]), float(g["min_density"])
        nef.grid.occupancy = torch.from_numpy(g["occupancy0"].copy())
        return nef
    nef = fresh()
    pts = nef.grid.dense_points.cpu().numpy()
    nef.prune(jitter=torch.from_numpy(g["u"]))
    occ = nef.grid.occupancy.cpu().numpy()
    np.testing.assert_allclose(occ, g["occupancy1"], atol=2e-5, rtol=1e-5)
    keep = occ > float(g["min_density"])
    edge = np.abs(g["occupancy1"] - float(g["min_density"])) < 1e-4          # the threshold is the median: a cell may sit on it
    assert np.array_equal(keep[~edge], g["keep"][~edge]) and 0 < keep.sum() < keep.size
    new = nef.grid.blas
    if np.array_equal(keep, g["keep"]):
        assert np.array_equal(new.octree.cpu().numpy(), g["new_octree"]) and new.max_level == int(g["new_max_level"])
    s0, c0 = int(new.pyramid[1, level]), int(new.pyramid[0, level])
    got = set(map(tuple, new.points[s0:s0 + c0].cpu().numpy().tolist()))
    assert got == set(map(tuple, pts[keep].tolist()))
    o, d = O.look_at_rays([-3.0, 0.65, -3.0], [0, 0, 0], 24, 24, 30.0)
    mr = new.raymarch(W.Rays(dev(o), dev(d), dist_min=0.0, dist_max=8.0), 'ray', 128, seed=3)
    cells = torch.floor((mr.samples + 1.0) * 0.5 * 2 ** level).clamp(0, 2 ** level - 1).to(torch.int16).cpu().numpy()
    assert mr.samples.shape[0] > 0 and set(map(tuple, cells.tolist())) <= got
    # counter-based probe stream: same seed -> same result, other seed -> (slightly) different occupancy
    a, b, c = fresh(), fresh(), fresh()
    a.prune(seed=5); b.prune(seed=5); c.prune(seed=6)
    assert torch.equal(a.grid.occupancy, b.grid.occupancy) and np.array_equal(a.grid.blas.octree.cpu().numpy(), b.grid.blas.octree.cpu().numpy())
    assert not torch.equal(a.grid.occupancy, c.grid.occupancy)
    occ_a = a.grid.occupancy.clone()
    a.prune(seed=5)
    assert bool((a.grid.occupancy >= occ_a * float(g["decay"]) - 1e-6).all())


def test_wide_decoders_under_autocast_stay_native(W):
    """Decoders with TWO hidden layers each: the tensor-core backward covers the app/nerf depth only.  precision=None under autocast trains on the
    fp32 kernels (same results as precision 0); an explicit precision=1 with gradients raises at the forward."""
    torch.manual_seed(0)
    blas = W.OctreeAS.make_dense(4, device="cuda")
    grid = W.HashGrid.from_geometric(blas, feature_dim=2, num_lods=8, multiscale_type='cat', feature_std=0.1, codebook_bitwidth=12,
                                     min_grid_res=8, max_grid_res=64)
    nef = W.NeuralRadianceField(grid, view_embedder='positional', view_multires=2, hidden_dim=64, num_layers=2, bias=True).cuda()
    o, d = O.look_at_rays([-3.0, 0.65, -3.0], [0, 0, 0], 16, 16, 30.0)
    rays = W.Rays(dev(o), dev(d), dist_min=0.0, dist_max=8.0)
    outs = []
    for prec, amp in ((0, False), (None, True)):
        tracer = W.PackedRFTracer('ray', 64); tracer.seed = 3; tracer.precision = prec
        nef.zero_grad()
        with torch.autocast("cuda", dtype=torch.float16, enabled=amp):
            rb = W.Pipeline(nef, tracer)(rays=rays, channels=["rgb"])
        rb.rgb.sum().backward()
        outs.append((rb.rgb.detach().clone(), nef.grid.codebook.feats.grad.detach().clone()))
    assert torch.equal(outs[0][0], outs[1][0]) and torch.allclose(outs[0][1], outs[1][1], atol=1e-6, rtol=1e-4)
    tracer = W.PackedRFTracer('ray', 64); tracer.precision = 1
    with pytest.raises(W.WispB200Error):
        W.Pipeline(nef, tracer)(rays=rays, channels=["rgb"])
    tracer.seed = 3
    with torch.no_grad():                                   # inference at precision 1 is fine (forward-only tiles fit)
        rb = W.Pipeline(nef, tracer)(rays=rays, channels=["rgb"])
    assert torch.isfinite(rb.rgb).all() and float((rb.rgb - outs[0][0]).abs().max()) < 2e-2


@pytest.mark.parametrize("precision", [0, 1])
def test_trace_config1_full_frame_vs_oracle(W, precision):
    """BASELINE configs[0] (the reference's CPU-runnable case): HashGrid 8 levels, hidden 32, the WHOLE 256^2 single view
    (65 536 rays x 512 steps) forward + backward against the CPU restatement."""
    from gpu_util import nef_from_oracle, packed_grads
    tol = TOL[precision]
    onef = O.make_nef(feature_std=0.2, seed=5, num_lods=8, hidden_dim=32)
    spc = O.octree_to_spc(O.points_to_octree(O.lego_like_points(7), 7))
    o, d = O.look_at_rays([-3.0, 0.65, -3.0], [0, 0, 0], 256, 256, 30.0)
    nef, blas = nef_from_oracle(onef, spc)
    tracer = W.PackedRFTracer('ray', 512, bg_color=(1.0, 1.0, 1.0)); tracer.seed = 9
    tracer.precision = precision
    rb = W.Pipeline(nef, tracer)(rays=W.Rays(dev(o), dev(d), 0.0, 10.0), channels=["rgb", "depth", "alpha", "hit"])
    f = O.rf_trace_fwd(spc, onef, o, d, 0.0, 10.0, 512, bg=(1, 1, 1), seed=9)
    assert tracer.get_prev_num_samples() == f["num_samples"] > 100000
    np.testing.assert_allclose(rb.rgb.detach().cpu().numpy(), f["rgb"], atol=tol["rgb"])
    np.testing.assert_allclose(rb.alpha.detach().cpu().numpy(), f["alpha"], atol=tol["rgb"])
    if precision == 0:
        assert np.array_equal(rb.hit.cpu().numpy(), f["hit"])
    tgt = torch.sigmoid(torch.randn(o.shape[0], 3, generator=torch.Generator().manual_seed(6)))
    torch.nn.functional.smooth_l1_loss(rb.rgb, tgt.cuda()).backward()
    st = O.rf_step(spc, onef, o, d, 0.0, 10.0, 512, tgt.numpy(), bg=(1, 1, 1), seed=9)
    gt, gd, gc = packed_grads(nef)
    for got, ref, nm in ((gt, st["table"], "table"), (gd, st["dens"], "dens"), (gc, st["col"], "col")):
        scale = np.abs(ref).max()
        assert np.abs(got - ref).max() <= max(2e-3, tol["grad"]) * scale, (nm, np.abs(got - ref).max(), scale)


@pytest.mark.parametrize("precision", [0, 1])
def test_trace_config2_slice_vs_oracle(W, precision):
    """BASELINE config 2 shapes (L=16, F=2, T=2^19, 64-wide decoders, n=2048, level-7 lego-like octree) on a
    32x32-ray slice of the 1024^2 frame; counter-based jitter; fwd + bwd vs the oracle."""
    from gpu_util import nef_from_oracle, packed_grads
    tol = TOL[precision]
    onef = O.make_nef(feature_std=0.2, seed=3)
    spc = O.octree_to_spc(O.points_to_octree(O.lego_like_points(7), 7))
    o, d = O.look_at_rays([-3.0, 0.65, -3.0], [0, 0, 0], 1024, 1024, 30.0)
    sel = (np.arange(496, 528)[:, None] * 1024 + np.arange(500, 532)[None]).reshape(-1)
    o, d = o[sel], d[sel]
    nef, blas = nef_from_oracle(onef, spc)
    tracer = W.PackedRFTracer('ray', 2048, bg_color=(0.0, 0.0, 0.0)); tracer.seed = 77
    tracer.precision = precision
    rays = W.Rays(dev(o), dev(d), 0.0, 10.0)
    rb = W.Pipeline(nef, tracer)(rays=rays, channels=["rgb", "depth", "alpha", "hit"])
    f = O.rf_trace_fwd(spc, onef, o, d, 0.0, 10.0, 2048, bg=(0, 0, 0), seed=77)
    assert tracer.get_prev_num_samples() == f["num_samples"] and f["num_samples"] > 10000
    np.testing.assert_allclose(rb.rgb.detach().cpu().numpy(), f["rgb"], atol=tol["rgb"])
    np.testing.assert_allclose(rb.alpha.detach().cpu().numpy(), f["alpha"], atol=tol["rgb"])
    np.testing.assert_allclose(rb.depth.detach().cpu().numpy(), f["depth"], atol=max(1e-3, tol["depth"]))
    if precision == 0:
        assert np.array_equal(rb.hit.cpu().numpy(), f["hit"])
    tgt = torch.sigmoid(torch.randn(o.shape[0], 3, generator=torch.Generator().manual_seed(2)))
    torch.nn.functional.smooth_l1_loss(rb.rgb, tgt.cuda()).backward()
    st = O.rf_step(spc, onef, o, d, 0.0, 10.0, 2048, tgt.numpy(), bg=(0, 0, 0), seed=77)
    gt, gd, gc = packed_grads(nef)
    for got, ref, nm in ((gt, st["table"], "table"), (gd, st["dens"], "dens"), (gc, st["col"], "col")):
        scale = np.abs(ref).max()
        assert np.abs(got - ref).max() <= max(2e-3, tol["grad"]) * scale, (nm, np.abs(got - ref).max(), scale)


SHAPES = [dict(num_lods=8, feature_dim=4, codebook_bitwidth=14, min_res=8, max_res=128, hidden_dim=32, multiscale="cat", view_freq=4, bias=True),
          dict(num_lods=6, feature_dim=8, codebook_bitwidth=12, min_res=8, max_res=96, hidden_dim=64, multiscale="sum", view_freq=2, bias=False),
          dict(num_lods=12, feature_dim=2, codebook_bitwidth=15, min_res=16, max_res=256, hidden_dim=48, multiscale="cat", view_freq=3, bias=True),
          dict(num_lods=4, feature_dim=2, codebook_bitwidth=10, min_res=4, max_res=32, hidden_dim=16, multiscale="sum", view_freq=1, bias=True),
          # hidden_dim = 128 (the reference's best published app/nerf setting, docs/pages/app_nerf.md:186-192): at precision 1 these train on the
          # one-group tensor-core backward (mixed accumulator orientation), with the fused table scatter (F = 2 'cat') and without it
          dict(num_lods=16, feature_dim=2, codebook_bitwidth=14, min_res=16, max_res=256, hidden_dim=128, multiscale="cat", view_freq=4, bias=True),
          dict(num_lods=8, feature_dim=4, codebook_bitwidth=13, min_res=8, max_res=128, hidden_dim=128, multiscale="cat", view_freq=2, bias=True),
          dict(num_lods=16, feature_dim=2, codebook_bitwidth=14, min_res=16, max_res=256, hidden_dim=128, multiscale="cat", view_freq=4, bias=False),
          # position embeddings (positional + input, identity) and the identity view embedding; F = 2 'cat' with L = 6 puts the position
          # embedding in the same 16-byte slab row as the last grid features
          dict(num_lods=8, feature_dim=2, codebook_bitwidth=13, min_res=8, max_res=128, hidden_dim=64, multiscale="cat", view_freq=4, bias=True,
               pos_mode=3, pos_freq=3),
          dict(num_lods=6, feature_dim=4, codebook_bitwidth=12, min_res=8, max_res=96, hidden_dim=32, multiscale="sum", view_freq=0, bias=True,
               pos_mode=1, view_mode=1),
          dict(num_lods=6, feature_dim=2, codebook_bitwidth=12, min_res=8, max_res=96, hidden_dim=32, multiscale="cat", view_freq=2, bias=True,
               pos_mode=3, pos_freq=2)]


@pytest.mark.parametrize("precision", [0, 1])
@pytest.mark.parametrize("shape", SHAPES, ids=lambda c: f"F{c['feature_dim']}{c['multiscale']}L{c['num_lods']}h{c['hidden_dim']}"
                         + (f"pos{c['pos_mode']}" if c.get('pos_mode') else "") + (f"view{c['view_mode']}" if 'view_mode' in c else ""))
def test_trace_other_shapes_vs_oracle(W, shape, precision):
    """Feature widths 2/4/8, 'cat' and 'sum', decoder widths that are not powers of two, no bias: the generic gather / scatter paths
    of the fused kernels (the app/nerf shape takes the specialised F == 2 'cat' path), forward + backward vs the oracle."""
    from gpu_util import nef_from_oracle, packed_grads
    tol = TOL[precision]
    onef = O.make_nef(feature_std=0.3, seed=11, **shape)
    spc = O.octree_to_spc(O.points_to_octree(O.lego_like_points(5), 5))
    o, d = O.look_at_rays([-3.0, 0.65, -3.0], [0, 0, 0], 24, 24, 30.0)
    nef, blas = nef_from_oracle(onef, spc)
    tracer = W.PackedRFTracer('ray', 256, bg_color=(1.0, 1.0, 1.0)); tracer.seed = 5
    tracer.precision = precision
    rb = W.Pipeline(nef, tracer)(rays=W.Rays(dev(o), dev(d), 0.0, 8.0), channels=["rgb", "depth", "alpha", "hit"])
    f = O.rf_trace_fwd(spc, onef, o, d, 0.0, 8.0, 256, bg=(1, 1, 1), seed=5)
    assert tracer.get_prev_num_samples() == f["num_samples"] > 1000
    np.testing.assert_allclose(rb.rgb.detach().cpu().numpy(), f["rgb"], atol=tol["rgb"])
    np.testing.assert_allclose(rb.alpha.detach().cpu().numpy(), f["alpha"], atol=tol["rgb"])
    tgt = torch.sigmoid(torch.randn(o.shape[0], 3, generator=torch.Generator().manual_seed(4)))
    torch.nn.functional.smooth_l1_loss(rb.rgb, tgt.cuda()).backward()
    st = O.rf_step(spc, onef, o, d, 0.0, 8.0, 256, tgt.numpy(), bg=(1, 1, 1), seed=5)
    gt, gd, gc = packed_grads(nef)
    for got, ref, nm in ((gt, st["table"], "table"), (gd, st["dens"], "dens"), (gc, st["col"], "col")):
        scale = np.abs(ref).max()
        if precision == 1 and nm == "table":
            # fp16 forward vs fp32 forward: a sample whose pre-activation sits at a relu kink takes the other branch, and on this small
            # scene (a table entry collects a handful of samples, |grad| ~ 1e-6) that is 1-9 % of the largest entry for 64- AND 128-wide
            # decoders alike, depending on the seed (the bench-scale parity leg of the real configuration holds 3e-2).  The norm of the
            # whole gradient is the stable figure.
            assert np.linalg.norm((got - ref).ravel()) <= 3e-2 * np.linalg.norm(ref.ravel()), (nm, "L2")
            assert np.abs(got - ref).max() <= 0.15 * scale, (nm, np.abs(got - ref).max(), scale)
            continue
        assert np.abs(got - ref).max() <= max(2e-3, tol["grad"]) * scale, (nm, np.abs(got - ref).max(), scale)


def test_no_rays_and_no_hits(W):
    from gpu_util import nef_from_oracle
    onef = O.make_nef(num_lods=4, codebook_bitwidth=10, min_res=4, max_res=32, hidden_dim=16, feature_std=0.5, seed=1)
    spc = O.octree_to_spc(O.points_to_octree(O.lego_like_points(4), 4))
    nef, blas = nef_from_oracle(onef, spc)
    tracer = W.PackedRFTracer('ray', 32, bg_color=(0.1, 0.2, 0.3))
    o = np.tile(np.array([[5.0, 5.0, 5.0]], np.float32), (5, 1)); d = np.tile(np.array([[1.0, 0, 0]], np.float32), (5, 1))
    rb = tracer(nef, rays=W.Rays(dev(o), dev(d), 0.0, 1.0))
    assert tracer.get_prev_num_samples() == 0
    np.testing.assert_allclose(rb.rgb.detach().cpu().numpy(), np.tile(np.array([[0.1, 0.2, 0.3]], np.float32), (5, 1)))
    assert not rb.hit.any() and float(rb.alpha.detach().abs().sum()) == 0.0
    rb0 = tracer(nef, rays=W.Rays(dev(o[:0]), dev(d[:0]), 0.0, 1.0))
    assert rb0.rgb.shape == (0, 3)


# ---------------------------------------------------------------------------------------------------------------
# tensor-core operand layouts (csrc/wb_tc.cuh)
# ---------------------------------------------------------------------------------------------------------------
def slab_image(X):
    """[R, C] -> byte image: element (s, f) at (f/8)*(R*16) + s*16 + (f%8)*2."""
    S, Cc = X.shape
    assert S in (64, 128) and Cc % 8 == 0
    return np.ascontiguousarray(X.astype(np.float16).reshape(S, Cc // 8, 8).transpose(1, 0, 2)).view(np.uint8).reshape(-1)


def weight_image(Wm):
    """W [N, K] -> byte image: element (n, k) at (k/8)*(N*16) + n*16 + (k%8)*2."""
    N, K = Wm.shape
    return np.ascontiguousarray(Wm.astype(np.float16).reshape(N, K // 8, 8).transpose(1, 0, 2)).view(np.uint8).reshape(-1)


def _selftest(W, mode, rows, N, K, a, b):
    import ctypes as C
    D = torch.zeros((128 if mode == 2 else rows, N), dtype=torch.float32, device="cuda")
    ta, tb = dev(a), dev(b)
    A = W._cabi
    m = mode | (4 if rows == 64 else 0)
    A.check(A.lib().wb_tc_selftest(A.ptr(ta), C.c_int(a.size), A.ptr(tb), C.c_int(b.size), A.ptr(D), C.c_int(N), C.c_int(K), C.c_int(m), A.stream()))
    torch.cuda.synchronize()
    return D.cpu().numpy()


def _operand_case(W, mode, N, K, rows, seed):
    rng = np.random.default_rng(seed)
    q = lambda a: a.astype(np.float16).astype(np.float32)
    if mode == 0:
        X, Wm = q(rng.standard_normal((rows, K))), q(rng.standard_normal((N, K)))
        a, b, ref = slab_image(X), weight_image(Wm), X.astype(np.float64) @ Wm.T
    elif mode == 1:
        dY, Wm = q(rng.standard_normal((rows, K))), q(rng.standard_normal((K, N)))      # W: out=K rows, in=N cols
        a, b, ref = slab_image(dY), weight_image(Wm), dY.astype(np.float64) @ Wm
    else:
        X, dY = q(rng.standard_normal((rows, 128))), q(rng.standard_normal((rows, N)))
        if N == 8:                                              # the constant-one slab: feature 0 = 1, features 1..7 = 0
            dY[:] = 0.0; dY[:, 0] = 1.0
        a, b, ref = slab_image(X), slab_image(dY), X.T.astype(np.float64) @ dY
    np.testing.assert_allclose(_selftest(W, mode, rows, N, K, a, b), ref, atol=2e-3, rtol=1e-3)


@pytest.mark.parametrize("mode,N,K", [(0, 64, 32), (0, 16, 64), (0, 64, 48), (1, 48, 64), (1, 32, 64), (1, 64, 16), (2, 64, 128), (2, 16, 128)])
def test_tcgen05_operand_layouts(W, mode, N, K):
    """128-row tiles (slab = 2048 bytes, two warpgroups).  The name predates the Hopper port: the self-test runs wgmma."""
    _operand_case(W, mode, N, K, 128, mode * 100 + N)


# the decoder kernels' 64-row tile (slab = 1024 bytes, one warpgroup for modes 0 / 1); N = 80 / 96 / 112: the tc_chain_n instances of
# 80..112-wide layers; N = 8 (mode 2): the bias-gradient chain
@pytest.mark.parametrize("mode,N,K", [(0, 80, 96), (0, 96, 128), (0, 112, 32), (0, 128, 112), (0, 16, 16), (0, 64, 48),
                                      (1, 80, 112), (1, 96, 64), (1, 112, 128), (1, 16, 96), (1, 64, 16),
                                      (2, 8, 64), (2, 80, 64), (2, 96, 64), (2, 112, 64), (2, 128, 64), (2, 16, 64), (2, 64, 64)])
def test_wgmma_operand_layouts(W, mode, N, K):
    _operand_case(W, mode, N, K, 64, mode * 100 + N + 64)


def test_wgmma_accumulation_precision(W):
    """Measured fp32 accumulation error of wgmma.mma_async .f32.f16.f16 on random fp16 operands with a wide exponent range, K up to
    128: max |D - exact| / sum |a b| must not exceed the gamma(K) the interval reference of the decoders (oracle/tc_decoders.py) uses."""
    from oracle import tc_decoders as T
    rng = np.random.default_rng(42)
    worst = {}
    for K in (16, 64, 128):
        for rep in range(4):
            X = rng.standard_normal((64, K)) * 2.0 ** rng.integers(-8, 8, (64, K))
            Wm = rng.standard_normal((128, K)) * 2.0 ** rng.integers(-8, 8, (128, K))
            if rep % 2:                                         # cancellation: sums much smaller than sum |terms|
                X[:, K // 2:] = X[:, :K // 2]
                Wm[:, K // 2:] = -Wm[:, :K // 2] * (1.0 + 2.0 ** -9 * rng.standard_normal((128, K // 2)))
            X, Wm = X.astype(np.float16).astype(np.float64), Wm.astype(np.float16).astype(np.float64)
            assert np.isfinite(X).all() and np.isfinite(Wm).all()
            D = _selftest(W, 0, 64, 128, K, slab_image(X), weight_image(Wm))
            exact, mag = X @ Wm.T, np.abs(X) @ np.abs(Wm).T
            ratio = float((np.abs(D - exact) / mag).max())
            worst[K] = max(worst.get(K, 0.0), ratio)
    print("wgmma accumulation max|err|/sum|terms|:", {k: f"{v:.3e} (gamma {T.gamma(k):.3e}, {v / 2.0 ** -24:.2f} units of 2^-24)" for k, v in worst.items()})
    for K, v in worst.items():
        assert v <= T.gamma(K), (K, v, T.gamma(K))


# ---------------------------------------------------------------------------------------------------------------
# raytrace + 'voxel' / 'uniform' samplers
# ---------------------------------------------------------------------------------------------------------------
def test_raytrace_voxel_uniform_golden(W, golden_dir):
    """Kernels vs what the reference's own _raymarch_voxel / _raymarch_uniform produced (bit-exact)."""
    g = np.load(os.path.join(golden_dir, "raymarch_nuggets.npz"))
    blas = W.OctreeAS(dev(g["octree"]))
    rays = W.Rays(dev(g["origins"]), dev(g["dirs"]), 0.0, 10.0)
    level = int(g["level"])
    rt = blas.raytrace(rays, level, with_exit=True)
    assert rt.ridx.dtype == torch.int32 and rt.depth.shape[1] == 2
    assert np.array_equal(rt.ridx.cpu().numpy(), g["nug_ridx"]) and np.array_equal(rt.pidx.cpu().numpy(), g["nug_pidx"])
    assert np.array_equal(rt.depth.cpu().numpy(), g["nug_depth"])
    assert blas.raytrace(rays, level, with_exit=False).depth.shape[1] == 1
    mv = blas.raymarch(rays, 'voxel', int(g["n_voxel"]), level, jitter=dev(g["jitter"]))
    mu = blas.raymarch(rays, 'uniform', int(g["n_uniform"]), level)
    for m, pre in ((mv, "v_"), (mu, "u_")):
        assert np.array_equal(m.ridx.cpu().numpy(), g[pre + "ridx"])
        assert np.array_equal(m.samples.cpu().numpy(), g[pre + "samples"])
        assert np.array_equal(m.depth_samples.cpu().numpy(), g[pre + "depth"])
        assert np.array_equal(m.deltas.cpu().numpy(), g[pre + "deltas"])
        assert np.array_equal(m.boundary.cpu().numpy(), g[pre + "boundary"])
        assert m.ridx.dtype == torch.int64 and m.boundary.dtype == torch.bool


@pytest.mark.parametrize("level,lvl_trace", [(7, 7), (7, 4), (5, 0)])
def test_raytrace_seeded_vs_oracle(W, level, lvl_trace):
    spc = O.octree_to_spc(O.points_to_octree(O.lego_like_points(level), level))
    o, d = O.look_at_rays([-3.0, 0.65, -3.0], [0, 0, 0], 64, 64, 30.0)
    o = np.concatenate([o, np.array([[0.05, 0.02, -0.03]], np.float32)]); d = np.concatenate([d, np.array([[0.0, 0.0, 1.0]], np.float32)])
    blas = W.OctreeAS(dev(spc.octree))
    rt = blas.raytrace(W.Rays(dev(o), dev(d)), lvl_trace, with_exit=True)
    ref = O.raytrace(spc, o, d, lvl_trace)
    assert np.array_equal(rt.ridx.cpu().numpy(), ref["ridx"]) and np.array_equal(rt.pidx.cpu().numpy(), ref["pidx"])
    assert np.array_equal(rt.depth.cpu().numpy(), ref["depth"])
    mv = blas.raymarch(W.Rays(dev(o), dev(d)), 'voxel', 5, lvl_trace, seed=9)
    rv = O.raymarch_voxel(spc, o, d, 5, lvl_trace, seed=9)
    assert np.array_equal(mv.depth_samples.cpu().numpy(), rv["depth_samples"]) and np.array_equal(mv.deltas.cpu().numpy(), rv["deltas"])
    assert np.array_equal(mv.boundary.cpu().numpy(), rv["boundary"]) and np.array_equal(mv.samples.cpu().numpy(), rv["samples"])


@pytest.mark.parametrize("kind,n", [("voxel", 3), ("uniform", 160)])
def test_fused_trace_with_nugget_samplers(W, kind, n):
    """PackedRFTracer(raymarch_type='voxel'|'uniform'): fused route == unfused route == oracle nef + compositing."""
    from gpu_util import nef_from_oracle
    onef = O.make_nef(num_lods=6, codebook_bitwidth=12, min_res=4, max_res=64, hidden_dim=32, feature_std=0.5, seed=4)
    spc = O.octree_to_spc(O.points_to_octree(O.lego_like_points(5), 5))
    o, d = O.look_at_rays([-3.0, 0.65, -3.0], [0, 0, 0], 24, 24, 30.0)
    outs = []
    for fused in (True, False):
        nef, blas = nef_from_oracle(onef, spc)
        if not fused:
            nef.fused_spec = lambda lod_idx=None: None
        tr = W.PackedRFTracer(kind, n, bg_color=(1.0, 1.0, 1.0)); tr.seed = 21
        rb = tr(nef, rays=W.Rays(dev(o), dev(d), 0.0, 10.0), channels=["rgb", "depth", "alpha", "hit"])
        outs.append((rb, tr.get_prev_num_samples()))
    (a, sa), (b, sb) = outs
    assert sa == sb > 0
    np.testing.assert_allclose(a.rgb.detach().cpu().numpy(), b.rgb.detach().cpu().numpy(), atol=2e-5)
    np.testing.assert_allclose(a.depth.detach().cpu().numpy(), b.depth.detach().cpu().numpy(), atol=2e-4)
    # oracle: samples from the oracle marcher, field + compositing from the oracle
    mr = O.raymarch_voxel(spc, o, d, n, seed=21) if kind == "voxel" else O.raymarch_uniform(spc, o, d, n)
    assert mr["ridx"].shape[0] == sa
    rgb_s, dens_s = O.nef_rgba(onef, mr["samples"], d[mr["ridx"]])
    cols, w = O.exponential_integration(rgb_s, dens_s[:, 0] * mr["deltas"][:, 0], mr["boundary"])
    alpha = O.sum_reduce(w, mr["boundary"])
    exp_rgb = np.ones((o.shape[0], 3), np.float32)
    hit_rays = mr["ridx"][mr["boundary"]]
    exp_rgb[hit_rays] = (1.0 - alpha) + cols
    np.testing.assert_allclose(a.rgb.detach().cpu().numpy(), exp_rgb, atol=1e-4)


def test_raytrace_single_traversal_matches_two_pass(W):
    """OctreeAS.raytrace with the nugget cache (one depth-first traversal: count + cache, then copy; rays that overflow the cache are
    traversed again) gives exactly the nuggets of the two-traversal form, for a cache that holds everything, almost nothing, and nothing."""
    blas = W.OctreeAS.from_quantized_points(torch.from_numpy(O.lego_like_points(6)).cuda(), 6)
    o, d = O.look_at_rays([-3.0, 0.65, -3.0], [0, 0, 0], 64, 64, 30.0)
    outs = []
    old = W.ops.RAYTRACE_CACHE_K
    try:
        for K in (0, 24, 2, 1):
            W.ops.RAYTRACE_CACHE_K = K
            outs.append(W.ops.raytrace(blas.tensors(), dev(o), dev(d), 6))
    finally:
        W.ops.RAYTRACE_CACHE_K = old
    assert outs[0][0].shape[0] > 2000 and int((outs[0][3][1:] - outs[0][3][:-1]).max()) > 2        # some rays overflow K = 2
    for other in outs[1:]:
        for a, b in zip(outs[0], other):
            assert torch.equal(a, b)


def test_raygen_kernels(W, golden_dir):
    """wb_raygen_lookat vs the reference's _look_at (golden from the unmodified source, persp + ortho, wide / tall aspect), and
    wb_raygen_pinhole vs a torch restatement of generate_pinhole_rays (raygen.py:40-85; Kaolin's Camera is absent: unpinned)."""
    g = np.load(os.path.join(golden_dir, "raygen.npz"))
    for n in ("square", "wide", "tall", "ortho"):
        a = g[n + "_args"]
        rays = W.raygen.look_at_rays(list(a[:3]), list(a[3:6]), int(a[6]), int(a[7]), mode=str(g[n + "_mode"]), fov=float(a[8]))
        np.testing.assert_allclose(rays.origins.cpu().numpy(), g[n + "_origins"], atol=1e-6)
        np.testing.assert_allclose(rays.dirs.cpu().numpy(), g[n + "_dirs"], atol=1e-6)
    H, Wd, ry, rx = 24, 40, 12, 20
    ang = 0.7
    Rm = np.array([[np.cos(ang), 0, np.sin(ang)], [0, 1, 0], [-np.sin(ang), 0, np.cos(ang)]], np.float32)
    pos = np.array([1.0, 0.5, -2.0], np.float32)
    rays = W.raygen.pinhole_rays(pos, Rm, 50.0, H, Wd, res_y=ry, res_x=rx, x0=1.5, y0=-0.5)
    py, px = torch.meshgrid(torch.arange(ry, dtype=torch.float), torch.arange(rx, dtype=torch.float), indexing="ij")
    px = px * (float(Wd) / rx) + 0.5 - 1.5; py = py * (float(H) / ry) + 0.5 + (-0.5)
    px = 2 * (px / Wd) - 1.0; py = 2 * (py / H) - 1.0
    th = float(np.tan(np.radians(50.0) / 2)); tv = th * H / Wd
    dc = torch.stack((px * th, -py * tv, -torch.ones_like(px)), -1).reshape(-1, 3)
    dw = dc @ torch.from_numpy(Rm).t()
    dw = dw / torch.linalg.norm(dw, dim=-1, keepdim=True)
    np.testing.assert_allclose(rays.dirs.cpu().numpy(), dw.numpy(), atol=2e-6)
    np.testing.assert_allclose(rays.origins.cpu().numpy(), np.broadcast_to(pos, (ry * rx, 3)), atol=0)


# ---------------------------------------------------------------------------------------------------------------
# TriplanarGrid
# ---------------------------------------------------------------------------------------------------------------
def _triplanar_from_golden(W, g, ms):
    grid = W.TriplanarGrid(None, feature_dim=4, log_base_resolution=2, num_lods=3, multiscale_type=ms, feature_std=0.0).cuda()
    planes = [getattr(f, n) for f in grid.features for n in ("fmx", "fmy", "fmz")]
    with torch.no_grad():
        for i, p in enumerate(planes):
            p.copy_(dev(g[f"{ms}_plane{i}"]))
    return grid, planes


@pytest.mark.parametrize("ms", ["sum", "cat"])
def test_triplanar_golden(W, golden_dir, ms):
    """One-launch triplane kernel vs the reference TriplanarGrid (3 F.grid_sample per LOD, reflection padding), fwd + bwd.
    Tolerance: the reference's fp32 interpolation test tolerance (tests/core/test_grid_interpolation.py:50-53)."""
    g = np.load(os.path.join(golden_dir, "triplanar.npz"))
    grid, planes = _triplanar_from_golden(W, g, ms)
    coords = dev(g[f"{ms}_coords"])
    feats = grid.interpolate(coords, 2)
    np.testing.assert_allclose(feats.detach().cpu().numpy(), g[f"{ms}_feats"], atol=2e-6, rtol=1e-4)
    np.testing.assert_allclose(grid.interpolate(coords, 0).detach().cpu().numpy(), g[f"{ms}_feats_lod0"], atol=2e-6, rtol=1e-4)
    feats.backward(dev(g[f"{ms}_go"]))
    for i, p in enumerate(planes):
        np.testing.assert_allclose(p.grad.cpu().numpy(), g[f"{ms}_gplane{i}"], atol=2e-5, rtol=1e-4)
    assert grid.interpolate(coords.reshape(7, 43, 3), 2).shape[:2] == (7, 43)


def test_triplanar_config4_shapes_vs_torch(W):
    """BASELINE config 4 shapes: 4 LODs 65^2..513^2 x 4 channels x 3 planes; kernel vs torch's own F.grid_sample on the GPU."""
    import torch.nn.functional as Fn
    torch.manual_seed(0)
    grid = W.TriplanarGrid(None, feature_dim=4, log_base_resolution=6, num_lods=4, multiscale_type='sum', feature_std=1.0).cuda()
    coords = torch.rand(200000, 3, device="cuda") * 2 - 1
    feats = grid.interpolate(coords, 3)
    ref = 0
    sc = coords.reshape(1, -1, 1, 3)
    for f in grid.features:
        sx = Fn.grid_sample(f.fmx, sc[..., [1, 2]], align_corners=True, padding_mode='reflection')[0, :, :, 0].t()
        sy = Fn.grid_sample(f.fmy, sc[..., [0, 2]], align_corners=True, padding_mode='reflection')[0, :, :, 0].t()
        sz = Fn.grid_sample(f.fmz, sc[..., [0, 1]], align_corners=True, padding_mode='reflection')[0, :, :, 0].t()
        ref = ref + torch.cat([sx, sy, sz], -1)
    assert feats.shape == (200000, 12)
    assert float((feats - ref).abs().max()) < 2e-5


def test_triplanar_nerf_voxel_trace(W):
    """Config 4 pipeline in miniature: NeuralRadianceField(TriplanarGrid over an AABB) traced with 'voxel' sampling at the root
    level (triplanar_grid.py:145-150), forward + backward through the unfused route; checked against a torch-CPU evaluation."""
    import torch.nn.functional as Fn
    torch.manual_seed(1)
    blas = W.AxisAlignedBBoxAS(device="cuda")
    grid = W.TriplanarGrid(blas, feature_dim=4, log_base_resolution=3, num_lods=2, multiscale_type='sum', feature_std=0.5)
    nef = W.NeuralRadianceField(grid, view_embedder='positional', view_multires=4, hidden_dim=32, num_layers=1, bias=True).cuda()
    tracer = W.PackedRFTracer('voxel', 24, bg_color=(0.0, 0.0, 0.0)); tracer.seed = 3
    o, d = O.look_at_rays([-3.0, 0.65, -3.0], [0, 0, 0], 16, 16, 30.0)
    rb = tracer(nef, rays=W.Rays(dev(o), dev(d), 0.0, 10.0), channels=["rgb", "alpha", "depth", "hit"])
    S = tracer.get_prev_num_samples()
    assert S == int(rb.hit.sum()) * 24 or S >= int(rb.hit.sum()) * 24          # one root nugget per ray that meets the cube
    rb.rgb.sum().backward()
    assert grid.features[0].fmx.grad is not None and float(grid.features[0].fmx.grad.abs().sum()) > 0
    assert nef.decoder_color.lout.weight.grad is not None
    # CPU evaluation of the same samples with torch ops only
    spc1 = O.octree_to_spc(O.dense_octree(1))
    mr = O.raymarch_voxel(spc1, o, d, 24, level=0, seed=3)
    assert mr["ridx"].shape[0] == S
    nef_cpu = nef.cpu()
    with torch.no_grad():
        c = torch.from_numpy(mr["samples"]); feats = 0
        sc = c.reshape(1, -1, 1, 3)
        for f in nef_cpu.grid.features:
            feats = feats + torch.cat([Fn.grid_sample(f.fmx, sc[..., [1, 2]], align_corners=True, padding_mode='reflection')[0, :, :, 0].t(),
                                       Fn.grid_sample(f.fmy, sc[..., [0, 2]], align_corners=True, padding_mode='reflection')[0, :, :, 0].t(),
                                       Fn.grid_sample(f.fmz, sc[..., [0, 1]], align_corners=True, padding_mode='reflection')[0, :, :, 0].t()], -1)
        df = nef_cpu.decoder_density(feats)
        fdir = torch.cat([df, nef_cpu.view_embedder(torch.from_numpy(d[mr["ridx"]]))], -1)
        rgb_s = torch.sigmoid(nef_cpu.decoder_color(fdir[..., 1:])).numpy(); sig = torch.relu(df[..., 0]).numpy()
    cols, w = O.exponential_integration(rgb_s, sig * mr["deltas"][:, 0], mr["boundary"])
    exp = np.zeros((o.shape[0], 3), np.float32); exp[mr["ridx"][mr["boundary"]]] = cols
    np.testing.assert_allclose(rb.rgb.detach().cpu().numpy(), exp, atol=2e-4)


def _trace_with_grads(W, nef, tracer, rays, fused, precision):
    """One forward + backward of the tracer; fused=False forces the unfused route (native grid kernel + torch nn.Linear decoders:
    autograd gives the reference gradients).  -> rgb, depth, alpha, {param name: grad}."""
    for p_ in nef.parameters():
        p_.grad = None
    tracer.precision = precision
    if not fused:
        nef.fused_spec = lambda lod_idx=None: None
    try:
        assert (nef.fused_spec() is not None) == fused
        rb = tracer(nef, rays=rays, channels=["rgb", "depth", "alpha", "hit"])
        tgt = torch.sigmoid(torch.randn(rays.origins.shape[0], 3, generator=torch.Generator().manual_seed(4))).cuda()
        (torch.nn.functional.smooth_l1_loss(rb.rgb, tgt) + 0.1 * rb.alpha.mean() + 0.01 * rb.depth.mean()).backward()
    finally:
        if not fused:
            del nef.fused_spec
    grads = {n: p_.grad.detach().clone() for n, p_ in nef.named_parameters() if p_.grad is not None}
    return rb.rgb.detach(), rb.depth.detach(), rb.alpha.detach(), grads


@pytest.mark.parametrize("kind", ["triplanar_sum", "triplanar_cat", "octree_sum", "octree_cat"])
def test_fused_triplanar_octree_nerf(W, kind):
    """NeuralRadianceField over TriplanarGrid / OctreeGrid through the FUSED pipeline (gather inside the shade kernels, decoders on
    the fp32 SIMT kernels or the tensor cores -- no nn.Linear) against the unfused route, whose grid kernels are pinned to the
    reference classes' goldens and whose decoders are torch's.  Config-4 shapes for the triplanar grid (4 LODs 65^2..513^2 x 4
    channels, 'voxel' marching of the AABB, 64-wide decoders); nerf_octree.yaml shapes in miniature for the octree grid."""
    torch.manual_seed(2)
    o, d = O.look_at_rays([-3.0, 0.65, -3.0], [0, 0, 0], 40, 40, 30.0)
    rays = W.Rays(dev(o), dev(d), 0.0, 10.0)
    ms = kind.split("_")[1]
    if kind.startswith("triplanar"):
        blas = W.AxisAlignedBBoxAS(device="cuda")
        grid = W.TriplanarGrid(blas, feature_dim=4, log_base_resolution=6, num_lods=4, multiscale_type=ms, feature_std=0.3)
        tracer = W.PackedRFTracer('voxel', 48, bg_color=(1.0, 1.0, 1.0))
    else:
        blas = W.OctreeAS.from_quantized_points(torch.from_numpy(O.lego_like_points(6)).cuda(), 6)
        grid = W.OctreeGrid(blas, feature_dim=8, num_lods=4, multiscale_type=ms, feature_std=0.3)
        tracer = W.PackedRFTracer('ray', 192, bg_color=(1.0, 1.0, 1.0))
    nef = W.NeuralRadianceField(grid, view_embedder='positional', view_multires=4, hidden_dim=64, num_layers=1, bias=True).cuda()
    spec = nef.fused_spec()
    assert spec is not None and spec.kind == kind.split("_")[0]
    tracer.seed = 11
    ref = _trace_with_grads(W, nef, tracer, rays, fused=False, precision=0)
    n_ref = tracer.get_prev_num_samples()
    assert n_ref > 5000 and float(ref[2].max()) > 0.2
    # precision 1 gradient tolerance: 3e-2 of max (as for the hash grid) only for the octree 'cat' grid; 0.2 of max for the triplanar
    # grids and the 'sum' octree grid: fp16 rounding of the gathered features dominates there, and torch's own autocast(fp16) of the
    # unfused route (the reference's AMP arithmetic without GradScaler) is further off still; the worst entry moves with the reduction
    # order (fine-LOD texels that only a handful of samples touch: one relu mask that flips under fp16 rounding changes such an entry by several per cent of the plane's maximum).
    # The fp32 path (precision 0) of the same kernels is held to 2e-3 just above.
    tol_g1 = 3e-2 if kind == "octree_cat" else 0.2
    for precision, (tol_rgb, tol_depth, tol_g) in ((0, (1e-4, 5e-4, 2e-3)), (1, (2e-3, 2e-2, tol_g1))):
        tracer.seed = 11
        got = _trace_with_grads(W, nef, tracer, rays, fused=True, precision=precision)
        assert tracer.get_prev_num_samples() == n_ref
        assert float((got[0] - ref[0]).abs().max()) <= tol_rgb, (precision, "rgb")
        assert float((got[1] - ref[1]).abs().max()) <= tol_depth, (precision, "depth")
        assert float((got[2] - ref[2]).abs().max()) <= tol_rgb, (precision, "alpha")
        assert set(got[3]) == set(ref[3])
        for n, gr in ref[3].items():
            scale = float(gr.abs().max())
            assert scale > 0, n
            assert float((got[3][n] - gr).abs().max()) <= tol_g * scale, (precision, n)


# ---------------------------------------------------------------------------------------------------------------
# OctreeGrid / NeuralSDF / PackedSDFTracer (BASELINE config 3 path)
# ---------------------------------------------------------------------------------------------------------------
def _sdf_from_golden(W, g, ms):
    blas = W.OctreeAS(dev(g["octree"]))
    grid = W.OctreeGrid(blas, feature_dim=8, num_lods=3, multiscale_type=ms, feature_std=0.0)
    nef = W.NeuralSDF(grid, pos_embedder='none', position_input=True, hidden_dim=16, num_layers=1).cuda()
    assert np.array_equal(grid.trinkets.cpu().numpy(), g[f"{ms}_trinkets"]) and np.array_equal(grid.pyramid_dual.numpy(), g[f"{ms}_pyramid_dual"])
    with torch.no_grad():
        for i, f in enumerate(grid.features):
            f.copy_(dev(g[f"{ms}_feat{i}"]))
        nef.decoder.layers[0].weight.copy_(dev(g[f"{ms}_W0"])); nef.decoder.layers[0].bias.copy_(dev(g[f"{ms}_b0"]))
        nef.decoder.lout.weight.copy_(dev(g[f"{ms}_W1"])); nef.decoder.lout.bias.copy_(dev(g[f"{ms}_b1"]))
    return nef, grid, blas


@pytest.mark.parametrize("ms", ["sum", "cat"])
def test_octree_grid_golden(W, golden_dir, ms):
    """OctreeGrid.interpolate + NeuralSDF.sdf forward/backward vs the reference classes (fp16-feature semantics of the call site;
    tolerance = the reference's fp16 interpolation tolerance 1e-2, tests/core/test_grid_interpolation.py:56-59, tightened to 2e-3)."""
    g = np.load(os.path.join(golden_dir, "sdf_octree.npz"))
    nef, grid, blas = _sdf_from_golden(W, g, ms)
    coords = dev(g[f"{ms}_coords"])
    np.testing.assert_allclose(grid.interpolate(coords, 2).detach().cpu().numpy(), g[f"{ms}_feats"], atol=2e-3)
    np.testing.assert_allclose(grid.interpolate(coords, 0).detach().cpu().numpy(), g[f"{ms}_feats_lod0"], atol=2e-3)
    sdf = nef(coords=coords, lod_idx=2, channels="sdf")
    np.testing.assert_allclose(sdf.detach().cpu().numpy(), g[f"{ms}_sdf"], atol=2e-3)
    sdf.abs().sum().backward()
    for i, f in enumerate(grid.features):
        ref = g[f"{ms}_gfeat{i}"]
        assert np.abs(f.grad.cpu().numpy() - ref).max() <= 2e-2 * max(np.abs(ref).max(), 1e-6), i
    refw = g[f"{ms}_gW0"]
    assert np.abs(nef.decoder.layers[0].weight.grad.cpu().numpy() - refw).max() <= 2e-2 * np.abs(refw).max()


def test_octree_grid_fp32_vs_oracle(W):
    """Same kernel without the fp16 rounding (half_features=False) against the numpy oracle at fp32 tolerance, larger tree."""
    from oracle import octree_grid as OG
    rng = np.random.default_rng(2)
    spc = O.octree_to_spc(O.points_to_octree(O.lego_like_points(6), 6))
    _, pyr, tr, _ = OG.make_trilinear_spc(spc)
    blas = W.OctreeAS(dev(spc.octree))
    grid = W.OctreeGrid(blas, feature_dim=16, num_lods=4, multiscale_type='sum', feature_std=1.0).cuda()
    grid.half_features = False
    coords = rng.uniform(-0.9, 0.9, (20000, 3)).astype(np.float32)
    out = grid.interpolate(dev(coords), 3).detach().cpu().numpy()
    ref = OG.octree_grid_interpolate(spc, tr, [f.detach().cpu().numpy() for f in grid.features], grid.active_lods, coords, 3, "sum", half=False)
    np.testing.assert_allclose(out, ref, atol=2e-5, rtol=1e-5)
    assert np.abs(ref).max() > 0.1


def test_find_depth_bound_vs_oracle(W):
    from oracle import octree_grid as OG
    rng = np.random.default_rng(3)
    P = 300
    counts = rng.integers(1, 6, P); offs = np.concatenate([[0], np.cumsum(counts)]).astype(np.int32)
    Ng = int(offs[-1])
    en = np.sort(rng.random(Ng) * 5).astype(np.float32); depth = np.stack([en, en + 0.01 + rng.random(Ng).astype(np.float32) * 0.05], -1).astype(np.float32)
    curr = offs[:-1].copy(); curr[::13] = -1
    q = (rng.random(P) * 5).astype(np.float32)
    got = W.ops.find_depth_bound(dev(q)[:, None], dev(depth), curr_idxes=dev(curr)).cpu().numpy()
    assert np.array_equal(got, OG.find_depth_bound(q, curr, depth))


def test_sdf_tracer_golden(W, golden_dir):
    """PackedSDFTracer.trace (persistent kernel: sphere tracing + nugget cursor + finite-difference normals) vs the reference
    tracer run by the reference's own classes.  The decoder sums in a different order than torch's CPU GEMM, so a ray whose
    |sdf| lands within fp32 round-off of a threshold may flip: at most 1 of the 400 rays, everything else must agree."""
    g = np.load(os.path.join(golden_dir, "sdf_octree.npz"))
    nef, grid, blas = _sdf_from_golden(W, g, "sum")
    tracer = W.PackedSDFTracer(num_steps=24, step_size=0.8, min_dis=1e-3)
    rb = tracer(nef, rays=W.Rays(dev(g["origins"]), dev(g["dirs"]), dist_min=0.0, dist_max=6.0), lod_idx=2,
                channels=["rgb", "depth", "hit", "normal", "alpha", "xyz"])
    hit, ref_hit = rb.hit.cpu().numpy(), g["t_hit"]
    assert (hit != ref_hit).sum() <= 1 and ref_hit.sum() > 20
    both = hit & ref_hit
    np.testing.assert_allclose(rb.depth.cpu().numpy()[both], g["t_depth"][both], atol=2e-4)
    np.testing.assert_allclose(rb.xyz.cpu().numpy()[both], g["t_xyz"][both], atol=2e-4)
    np.testing.assert_allclose(rb.alpha.cpu().numpy(), np.where(hit[:, None], 1.0, 0.0))
    np.testing.assert_allclose(rb.normal.detach().cpu().numpy()[both], g["t_normal"][both], atol=2e-2)
    miss = ~hit & ~ref_hit
    np.testing.assert_allclose(rb.rgb.cpu().numpy()[miss], g["t_rgb"][miss])            # rgb = (0 + 1) / 2 where nothing was hit


@pytest.mark.parametrize("ms", ["sum", "cat"])
def test_codebook_octree_grid_golden(W, golden_dir, ms):
    """CodebookOctreeGrid.interpolate (VQAD): row-wise selection + native trilinear blend vs the reference class run on CPU
    (tests/golden/codebook.npz): training mode (straight-through softmax: features, gradients of logits and dictionary) and eval
    mode (argmax selection), finest LOD and LOD 0."""
    g = np.load(os.path.join(golden_dir, "codebook.npz"))
    blas = W.OctreeAS(dev(g["octree"]))
    grid = W.CodebookOctreeGrid(blas, feature_dim=4, num_lods=3, multiscale_type=ms, feature_std=1.0, codebook_bitwidth=4).cuda()
    with torch.no_grad():
        for i in range(3):
            assert grid.features[i].shape == g[f"{ms}_logits{i}"].shape and grid.dictionary[i].shape == g[f"{ms}_dict{i}"].shape
            grid.features[i].copy_(dev(g[f"{ms}_logits{i}"])); grid.dictionary[i].copy_(dev(g[f"{ms}_dict{i}"]))
    coords = dev(g[f"{ms}_coords"])
    grid.train()
    feats = grid.interpolate(coords, 2)
    np.testing.assert_allclose(feats.detach().cpu().numpy(), g[f"{ms}_feats_train"], atol=2e-5, rtol=1e-5)
    feats.backward(dev(g[f"{ms}_go"]))
    for i in range(3):
        for got, ref in ((grid.features[i].grad, g[f"{ms}_glogits{i}"]), (grid.dictionary[i].grad, g[f"{ms}_gdict{i}"])):
            assert np.abs(got.cpu().numpy() - ref).max() <= 2e-4 * max(np.abs(ref).max(), 1e-6), i
    grid.eval()
    with torch.no_grad():
        np.testing.assert_allclose(grid.interpolate(coords, 2).cpu().numpy(), g[f"{ms}_feats_eval"], atol=2e-5, rtol=1e-5)
        np.testing.assert_allclose(grid.interpolate(coords, 0).cpu().numpy(), g[f"{ms}_feats_eval_lod0"], atol=2e-5, rtol=1e-5)
    # the grid plugs into the radiance-field tracer like any other (unfused route: native grid kernels + decoders)
    nef = W.NeuralRadianceField(grid, view_embedder='positional', view_multires=2, hidden_dim=16, num_layers=1, bias=True).cuda()
    assert nef.fused_spec() is None
    o, d = O.look_at_rays([-3.0, 0.65, -3.0], [0, 0, 0], 12, 12, 30.0)
    rb = W.PackedRFTracer('ray', 64, bg_color=(1.0, 1.0, 1.0))(nef, rays=W.Rays(dev(o), dev(d), 0.0, 10.0), channels=["rgb", "alpha"])
    assert torch.isfinite(rb.rgb).all() and float(rb.alpha.max()) > 0.0


def _config3_case():
    from oracle import octree_grid as OG
    # BASELINE config 3 shapes (nglod_octree.yaml): level-7 octree, OctreeGrid(F=16, 6 LODs, 'sum'), NeuralSDF(128 wide, 1 layer)
    return OG, OG.make_sdf_case(level=7, num_lods=6, feature_dim=16, hidden_dim=128, multiscale="sum", res=64, seed=11, feature_std=0.02)


def test_sdf_eval_config3_vs_oracle(W):
    """wb_sdf_eval (descent + 6 LODs x 8 corners x 16 features + position input + 19-128-1 decoder in one launch) vs numpy."""
    from gpu_util import sdf_nef_from_case
    OG, case = _config3_case()
    nef = sdf_nef_from_case(case)
    rng = np.random.default_rng(5)
    pts = case["spc"].points[case["spc"].pyramid[1, 7]: case["spc"].pyramid[1, 7] + case["spc"].pyramid[0, 7]].astype(np.float32)
    near = ((pts[rng.integers(0, pts.shape[0], 6000)] + rng.random((6000, 3)).astype(np.float32)) / 64.0 - 1.0).astype(np.float32)
    coords = np.concatenate([near, rng.uniform(-1.05, 1.05, (2000, 3)).astype(np.float32)])
    with torch.no_grad():
        for lod in (5, 2, 0):
            got = nef(coords=dev(coords), lod_idx=lod, channels="sdf").cpu().numpy()
            ref = OG.neural_sdf(case, coords, lod)
            np.testing.assert_allclose(got, ref, atol=2e-5, rtol=1e-5)
        # the no-grad fast path and the autograd route (grid kernel + torch decoder) are the same function
        with torch.enable_grad():
            slow = nef(coords=dev(coords), lod_idx=5, channels="sdf").detach().cpu().numpy()
        np.testing.assert_allclose(nef(coords=dev(coords), lod_idx=5, channels="sdf").cpu().numpy(), slow, atol=2e-5)


def test_sdf_trace_config3_vs_oracle(W):
    """Sphere tracing at BASELINE config-3 shapes (64^2-ray slice of the 512^2 frame, 32 steps, step 0.8): every quirk of the
    reference loop is observable here -- terminated packs keep drifting by `dist` until the LAST pack terminates, so depth != |xyz - o|."""
    from gpu_util import sdf_nef_from_case
    OG, case = _config3_case()
    nef = sdf_nef_from_case(case)
    ref = OG.sdf_trace(case, num_steps=32, step_size=0.8, min_dis=3e-3, dist_max=6.0, return_debug=True)
    tracer = W.PackedSDFTracer(num_steps=32, step_size=0.8, min_dis=3e-3)
    rays = W.Rays(dev(case["origins"]), dev(case["dirs"]), dist_min=0.0, dist_max=6.0)
    rb = tracer(nef, rays=rays, channels=["rgb", "depth", "hit", "normal", "alpha", "xyz"])
    hit = rb.hit.cpu().numpy()
    flips = int((hit != ref["hit"]).sum())
    assert ref["hit"].sum() > 500 and flips <= max(1, hit.size // 500), (flips, int(ref["hit"].sum()))    # <= 0.2 %
    both = hit & ref["hit"]
    np.testing.assert_allclose(rb.depth.cpu().numpy()[both], ref["depth"][both], atol=1e-4)
    np.testing.assert_allclose(rb.xyz.cpu().numpy()[both], ref["xyz"][both], atol=1e-4)
    dotn = (rb.normal.cpu().numpy()[both] * ref["normal"][both]).sum(-1)
    assert np.quantile(dotn, 0.01) > 0.999
    # the phase-by-phase route (fields the library cannot evaluate itself) is the same state machine
    orig = W.ops.sdf_field
    try:
        W.ops.sdf_field = lambda nef_: None
        rb2 = tracer(nef, rays=rays, channels=["rgb", "depth", "hit", "normal", "alpha", "xyz"])
    finally:
        W.ops.sdf_field = orig
    h2 = rb2.hit.cpu().numpy()
    assert int((h2 != hit).sum()) <= max(1, hit.size // 500)
    b2 = h2 & hit
    np.testing.assert_allclose(rb2.depth.detach().cpu().numpy()[b2], rb.depth.cpu().numpy()[b2], atol=1e-4)
    np.testing.assert_allclose(rb2.normal.detach().cpu().numpy()[b2], rb.normal.cpu().numpy()[b2], atol=2e-2)


# ---------------------------------------------------------------------------------------------------------------
# full BASELINE config-2 size: size-independent properties (the oracle cannot finish 2.1e9 candidates in seconds)
# ---------------------------------------------------------------------------------------------------------------
def test_full_frame_properties(W):
    """1024^2 rays x 2048 steps, lego-like level-7 octree, L=16/F=2/T=2^19, 64-wide decoders, tensor-core precision.
    Checks: packed sample list is consistent (offsets == scan of counts == popcount of the hit masks, ray-sorted records);
    a strided subset of rays reproduces the oracle's per-ray sample counts bit-exactly; outputs are in range and idempotent;
    the backward is linear in the upstream gradient; rays that miss the occupied box get the background."""
    torch.manual_seed(0)
    pts = torch.from_numpy(O.lego_like_points(7)).cuda()
    blas = W.OctreeAS.from_quantized_points(pts, 7)
    grid = W.HashGrid.from_geometric(blas, feature_dim=2, num_lods=16, multiscale_type='cat', feature_std=0.05, codebook_bitwidth=19,
                                     min_grid_res=16, max_grid_res=512)
    nef = W.NeuralRadianceField(grid, view_embedder='positional', view_multires=4, hidden_dim=64, num_layers=1, bias=True).cuda()
    o, d = O.look_at_rays([-3.0, 0.65, -3.0], [0, 0, 0], 1024, 1024, 30.0)
    R = o.shape[0]
    od, dd = dev(o), dev(d)
    ms = W.ops.march_count(blas.tensors(), od, dd, 0.0, 10.0, 2048, 7, seed=5)
    counts = ms.counts.long()
    assert int(counts.sum()) == ms.total and int(ms.offsets[-1]) == ms.total
    assert torch.equal(ms.offsets[1:] - ms.offsets[:-1], counts)
    pop = torch.zeros(R, dtype=torch.int64, device="cuda")
    hm = ms.hitmask.view(torch.int32)
    for b in range(32):
        pop += ((hm >> b) & 1).long().sum(1)
    assert torch.equal(pop, counts)
    rec_t, rec_delta, rec_ray = W.ops.march_fill_records(ms, od.device)
    assert bool((rec_ray[1:] >= rec_ray[:-1]).all())                                # ray-sorted
    same = rec_ray[1:] == rec_ray[:-1]
    assert bool((rec_t[1:][same] > rec_t[:-1][same]).all())                         # front to back inside a ray
    assert bool((rec_delta > 0).all()) and float(rec_t.min()) >= 0.0 and float(rec_t.max()) <= 10.0
    sel = np.arange(0, R, 2731)
    spc = O.octree_to_spc(O.points_to_octree(O.lego_like_points(7), 7))
    # oracle on a strided subset: the counter-based jitter is keyed by the GLOBAL ray index, so re-march those rays on the GPU as their own batch
    sub = W.ops.march_count(blas.tensors(), od[sel], dd[sel], 0.0, 10.0, 2048, 7, seed=5)
    ref = O.raymarch_ray(spc, o[sel], d[sel], 0.0, 10.0, 2048, seed=5)
    assert np.array_equal(sub.counts.cpu().numpy(), ref["counts"])
    tracer = W.PackedRFTracer('ray', 2048, bg_color=(0.25, 0.5, 0.75)); tracer.precision = 1; tracer.seed = 5
    rays = W.Rays(od, dd, 0.0, 10.0)
    rb = tracer(nef, rays=rays, channels=["rgb", "alpha", "depth", "hit"])
    assert tracer.get_prev_num_samples() == ms.total
    rgb = rb.rgb.detach(); alpha = rb.alpha.detach()
    assert float(rgb.min()) >= 0.0 and float(rgb.max()) <= 1.0 + 1e-5 and float(alpha.max()) <= 1.0 + 1e-5 and float(alpha.min()) >= 0.0
    miss = counts == 0
    assert bool(miss.any()) and torch.allclose(rgb[miss], torch.tensor([0.25, 0.5, 0.75], device="cuda").expand(int(miss.sum()), 3))
    assert float(alpha[miss].abs().sum()) == 0.0 and not bool(rb.hit[miss].any())
    tracer.seed = 5
    rb2 = tracer(nef, rays=rays, channels=["rgb"])
    assert torch.equal(rb2.rgb.detach(), rgb)                                       # idempotent / deterministic forward
    # backward linearity: grad(2*g) == 2*grad(g) up to atomic-order noise
    g1 = torch.randn(R, 3, device="cuda", generator=torch.Generator(device="cuda").manual_seed(1)) / R
    grads = []
    for k in (1.0, 2.0):
        nef.zero_grad(set_to_none=True)
        tracer.seed = 5
        out = tracer(nef, rays=rays, channels=["rgb"]).rgb
        out.backward(g1 * k)
        grads.append((grid.codebook.feats.grad.clone(), nef.decoder_color.layers[0].weight.grad.clone()))
    for a, b in zip(grads[0], grads[1]):
        assert float((2 * a - b).abs().max()) <= 2e-2 * float(b.abs().max()) + 1e-12
    assert float(grads[0][0][int(grid.codebook.begin_idxes[15]):].abs().sum()) == 0.0      # the zeroed last LOD receives no gradient


def test_triplane_relayout_roundtrip(W):
    """wb_triplane_relayout: [1, C, H, W] -> [H, W, C] is torch's permute, and back is the identity (C = 4 vector path and C = 3 scalar path)."""
    for Cc in (4, 3):
        planes = [torch.randn(1, Cc, n, n, device="cuda") for n in (5, 17, 33, 65, 9, 129)]
        cl = W.ops.triplane_relayout(planes, True)
        for p, q in zip(planes, cl):
            assert q.shape == (p.shape[2], p.shape[3], Cc) and torch.equal(q, p[0].permute(1, 2, 0).contiguous())
        back = W.ops.triplane_relayout(cl, False)
        for p, q in zip(planes, back):
            assert torch.equal(p, q)
