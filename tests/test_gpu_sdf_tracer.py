"""PackedSDFTracer's two native routes against tests/sdf_trace_reference.py (the tracer's loop restated in numpy, exactly rounded):
  * the phase route (wb_sdf_phase, the field through its own forward between the launches) over an analytic fp32 field -- bit for
    bit, through every edge of the state machine -- and over the fields it exists for: NeuralSDF over a hash grid (app/nglod hash),
    over a triplanar grid (app/nglod triplanar) and over a 'cat' octree grid below its finest LOD;
  * the persistent kernel (wb_sdf_trace) with several packs per thread: the bench's 512^2 frame and a frame of more packs than
    SMs x 2048 threads, on both compiled instances, its evaluation counter included.
The restatement is fed the same nuggets (the native raytrace, pinned by test_gpu_octree_traversal.py) and the same field evaluated on
the device, so what is compared is the state machine."""
import numpy as np
import pytest
import torch

from oracle import octree_grid as OG
from oracle import oracle as O

import sdf_trace_reference as TR

pytestmark = pytest.mark.gpu

C3 = float(np.float32(1.0 / np.sqrt(3.0)))
CAM_ORIGIN, CAM_LOOKAT, CAM_FOV = [-3.0, 0.65, -3.0], [0.0, 0.0, 0.0], 30.0          # bench.py's camera (config 3: origin x 0.75)


@pytest.fixture(scope="module")
def W():
    import wisp_b200
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return wisp_b200


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _pack_bound():
    """Threads of one wave of either tracer kernel, whatever its occupancy: SMs x 2048 (the phase kernel launches at most SMs x 8 CTAs
    of 256 threads, the persistent kernel at most SMs x blocks_per_SM <= SMs x 8)."""
    return _sms() * 2048


_CASE = {}


def _case():
    if not _CASE:
        _CASE.update(OG.make_sdf_case(level=5, num_lods=3, feature_dim=4, hidden_dim=8, res=32, seed=5))
    return _CASE


def _frame(res, scale):
    o, d = O.look_at_rays(CAM_ORIGIN, CAM_LOOKAT, res, res, CAM_FOV)
    return o * np.float32(scale), d


def _nuggets(W, grid, o, d, lod):
    ridx, _, depth, _ = W.ops.raytrace(W.ops.octree_tensors(grid.blas), dev(o), dev(d), W.ops.raytrace_level(grid, lod))
    return ridx.cpu().numpy(), depth.cpu().numpy()


def _trace(W, nef, o, d, lod, steps, step_size, min_dis, dist_max, normals=True):
    tracer = W.PackedSDFTracer(num_steps=steps, step_size=step_size, min_dis=min_dis)
    chans = ["depth", "hit", "xyz", "normal", "rgb", "alpha"] if normals else ["depth", "hit", "xyz", "alpha"]
    rb = tracer(nef, rays=W.Rays(dev(o), dev(d), dist_min=0.0, dist_max=dist_max), lod_idx=lod, channels=chans)
    torch.cuda.synchronize()
    out = {k: getattr(rb, k).detach().cpu().numpy() for k in chans}
    return out, tracer


def _device_field(fn):
    """field(x, lod) of the restatement evaluated on the device."""
    def f(x, lod=None):
        if x.shape[0] == 0:
            return np.zeros((0, 1), np.float32)
        with torch.no_grad():
            return fn(dev(x.astype(np.float32)), lod).reshape(-1, 1).float().cpu().numpy()
    return f


def _report(what, got, ref):
    hit, rh = got["hit"], ref["hit"]
    both = hit & rh
    dx = float(np.abs(got["xyz"][both] - ref["xyz"][both]).max()) if both.any() else 0.0
    dd = float(np.abs(got["depth"][both] - ref["depth"][both]).max()) if both.any() else 0.0
    dn = float(np.abs(got["normal"][both] - ref["normal"][both]).max()) if both.any() and "normal" in got else 0.0
    print(f"{what}: rays {hit.size} packs {ref['packs']} hits {int(rh.sum())} flips {int((hit != rh).sum())} max|dxyz| {dx:.3g} "
          f"max|ddepth| {dd:.3g} max|dnormal| {dn:.3g} iters {ref['iters']} exit {ref['exit']} bound_stops {ref['bound_stops']} "
          f"evals {ref['evals']}")
    return both


def _exact(what, got, ref, normals=True):
    _report(what, got, ref)
    assert np.array_equal(got["hit"], ref["hit"]), what
    assert np.array_equal(got["xyz"].view(np.int32), ref["xyz"].view(np.int32)), what
    assert np.array_equal(got["depth"].view(np.int32), ref["depth"].view(np.int32)), what
    assert np.array_equal(got["alpha"], ref["alpha"]), what
    if normals:
        assert np.abs(got["normal"] - ref["normal"]).max() <= 2e-6, what
        assert np.abs(got["rgb"] - ref["rgb"]).max() <= 1e-6, what


def _close(what, got, ref, normals=True):
    """The bounds of the tracer checks that compare fp32 fields evaluated in different batches."""
    both = _report(what, got, ref)
    hit, rh = got["hit"], ref["hit"]
    assert rh.sum() > 20 and (hit != rh).sum() <= max(1, 0.002 * hit.size), what
    np.testing.assert_allclose(got["xyz"][both], ref["xyz"][both], atol=1e-4)
    np.testing.assert_allclose(got["depth"][both], ref["depth"][both], atol=1e-4)
    if normals:
        assert np.quantile((got["normal"][both] * ref["normal"][both]).sum(-1), 0.01) > 0.999, what


# ---------------------------------------------------------------------------------------------------------------
# phase route, analytic field: bit for bit
# ---------------------------------------------------------------------------------------------------------------
def _analytic_np(scale, r, const=None):
    def f(x, lod=None):
        if const is not None:
            return np.full((x.shape[0], 1), np.float32(const), np.float32)
        a = np.abs(x.astype(np.float32))
        s = (a[:, 0] + a[:, 1]) + a[:, 2]
        return (((s - np.float32(r)) * np.float32(C3)) * np.float32(scale)).astype(np.float32)[:, None]
    return f


def _analytic_nef(W, case, scale, r, const=None):
    """A NeuralSDF on the case's OctreeGrid whose sdf() is an elementwise fp32 expression (the numpy side writes the same ops in the
    same order): ((|x| + |y| + |z| - r) * fp32(1/sqrt 3)) * scale, or a constant."""
    r32, s32 = float(np.float32(r)), float(np.float32(scale))

    class AnalyticSDF(W.NeuralSDF):
        def sdf(self, coords, lod_idx=None):
            if const is not None:
                return dict(sdf=torch.full((*coords.shape[:-1], 1), float(np.float32(const)), device=coords.device))
            a = coords.reshape(-1, 3).abs()
            s = a[:, 0] + a[:, 1] + a[:, 2]
            return dict(sdf=(((s - r32) * C3) * s32).reshape(*coords.shape[:-1], 1))

    blas = W.OctreeAS(dev(case["octree"]))
    grid = W.OctreeGrid(blas, feature_dim=4, num_lods=len(case["active_lods"]), multiscale_type="sum", feature_std=0.0)
    return AnalyticSDF(grid, hidden_dim=8).cuda()


_BASE = dict(steps=32, step_size=0.8, min_dis=1e-3, dist_max=6.0, scale=1.0, r=0.52, lod=2, frame=None)
# name: overrides, and what the case must exercise (checked on the restatement's counters)
ANALYTIC = {
    "steps0": (dict(steps=0), lambda s: s["iters"] == 0 and s["evals"] == s["packs"]),
    "steps1": (dict(steps=1), lambda s: s["iters"] == 1 and s["exit"] == "steps"),
    "steps2": (dict(steps=2), lambda s: s["iters"] == 2 and s["exit"] == "steps"),
    "steps64": (dict(steps=64), lambda s: s["iters"] > 32 and s["hits"] > 50),
    "min_dis_large": (dict(min_dis=0.5, steps=16), lambda s: s["iters"] == 1 and s["exit"] == "march" and s["hits"] == s["packs"]),
    "min_dis_tiny": (dict(min_dis=1e-12, steps=24), lambda s: s["iters"] == 24 and s["exit"] == "steps"),
    "dist_max": (dict(dist_max=2.45), lambda s: s["dist_max_kills"] > 20 and s["hits"] > 20 and s["iters"] > 2 and s["exit"] == "march"),
    "start_inside": (dict(r=0.75), lambda s: (s["dist0"] < 0).mean() > 0.9 and s["hits"] > 50),
    "overestimate3": (dict(scale=3.0), lambda s: s["bound_stops"] > 0 and s["hits"] > 20),
    "exit_after_jump": (dict(r=0.3, steps=64), lambda s: s["exit"] == "jump" and s["hits"] == 0),
    "interleaved": (dict(frame="interleaved"), lambda s: s["hits"] > 50),
    "one_ray": (dict(frame="one"), lambda s: s["packs"] == 1 and s["exit"] == "jump"),       # R = 1: the last pack is bounded by P = 1
    "all_miss": (dict(frame="away"), lambda s: s["nuggets"] == 0),
    "lod0": (dict(lod=0), lambda s: s["hits"] > 50),
    "lod1": (dict(lod=1, steps=64), lambda s: s["hits"] > 50),
    "many_packs": (dict(frame="large"), lambda s: s["packs"] > _pack_bound() and s["hits"] > 1000),
}


def _analytic_rays(case, frame):
    o, d = case["origins"], case["dirs"]
    if frame == "interleaved":           # every other ray points away from the scene: packs with rays without nuggets between them
        o2, d2 = np.empty((2 * o.shape[0], 3), np.float32), np.empty((2 * o.shape[0], 3), np.float32)
        o2[0::2], d2[0::2], o2[1::2], d2[1::2] = o, d, o, -d
        return o2, d2
    if frame == "one":                     # the hitting ray nearest the middle of the frame
        rt = O.raytrace(case["spc"], o, d, case["active_lods"][-1])
        full = TR.trace(o, d, rt["ridx"], rt["depth"], _analytic_np(1.0, 0.52), 2, 32, 0.8, 1e-3, 6.0, with_normals=False)
        hits = np.nonzero(full["hit"])[0]
        k = int(hits[np.argmin(np.abs(hits - o.shape[0] // 2))])
        return o[k:k + 1].copy(), d[k:k + 1].copy()
    if frame == "away":
        return o, -d
    if frame == "large":
        return _frame(768, 0.4)
    return o, d


@pytest.mark.parametrize("name", list(ANALYTIC))
def test_phase_route_analytic_field_exact(W, monkeypatch, name):
    over, exercised = ANALYTIC[name]
    p = dict(_BASE, **over)
    case = _case()
    nef = _analytic_nef(W, case, p["scale"], p["r"])
    monkeypatch.setattr(W.ops, "sdf_field", lambda nef: None)                # else the octree NeuralSDF goes to wb_sdf_trace
    o, d = _analytic_rays(case, p["frame"])
    ridx, depth = _nuggets(W, nef.grid, o, d, p["lod"])
    ref = TR.trace(o, d, ridx, depth, _analytic_np(p["scale"], p["r"]), p["lod"], p["steps"], p["step_size"], p["min_dis"], p["dist_max"])
    ref["hits"] = int(ref["hit"].sum())
    assert exercised(ref), (name, {k: ref[k] for k in ("packs", "nuggets", "iters", "exit", "bound_stops", "dist_max_kills", "evals", "hits")})
    if name == "interleaved":
        has = np.zeros(o.shape[0], bool); has[ridx] = True
        assert not has[1::2].any() and ref["hit"][0::2].sum() > 50
    got, _ = _trace(W, nef, o, d, p["lod"], p["steps"], p["step_size"], p["min_dis"], p["dist_max"])
    if name == "all_miss":                                                       # the buffers as _sdf_buffers initialises them
        assert not got["hit"].any() and not got["xyz"].any() and not got["depth"].any() and not got["normal"].any()
        assert np.all(got["rgb"] == 0.5) and not got["alpha"].any()
    _exact(name, got, ref)


def test_min_dis_thresholds_round_once(W, monkeypatch):
    """The tracer compares |dist| with fp32(min_dis) and (|dist + dist_prev| / 2) with fp32(min_dis * 5), each product a Python double
    rounded once.  For min_dis = 1e-3, fp32(fp32(1e-3) * 5) is one ulp above fp32(5e-3): a constant field of exactly fp32(5e-3) must
    not hit, on either route (a zero decoder with output bias c is exactly c on wb_sdf_trace)."""
    c = np.float32(5e-3)
    assert np.float32(np.float32(1e-3) * np.float64(5.0)) > c and np.float32(1e-3 * 5) == c
    case = _case()
    o, d = case["origins"], case["dirs"]
    ref = None
    for route in ("phase", "persistent"):
        if route == "phase":
            nef = _analytic_nef(W, case, 1.0, 0.52, const=c)
            monkeypatch.setattr(W.ops, "sdf_field", lambda nef: None)
        else:
            monkeypatch.undo()
            from gpu_util import sdf_nef_from_case
            z = dict(case, W=[np.zeros_like(w) for w in case["W"]], b=[np.zeros_like(case["b"][0]), np.full(1, c, np.float32)])
            nef = sdf_nef_from_case(z)
            assert W.ops.sdf_field(nef) is not None
        ridx, depth = _nuggets(W, nef.grid, o, d, 2)
        ref = TR.trace(o, d, ridx, depth, _analytic_np(1.0, 0.52, const=c), 2, 4, 1.0, 1e-3, 6.0)
        assert ref["packs"] > 50 and not ref["hit"].any()
        got, _ = _trace(W, nef, o, d, 2, 4, 1.0, 1e-3, 6.0)
        _exact(f"min_dis threshold ({route})", got, ref)


# ---------------------------------------------------------------------------------------------------------------
# phase route, the fields it exists for
# ---------------------------------------------------------------------------------------------------------------
def _sdf_like(nef, H):
    """(|x|+|y|+|z| - 0.52)/sqrt(3) through the first six hidden units plus a small grid part: the case's octree surface."""
    with torch.no_grad():
        l0 = nef.decoder.layers[0]
        l0.weight.mul_(0.05)
        l0.weight[:6, :3] = torch.tensor([[1, 0, 0], [-1, 0, 0], [0, 1, 0], [0, -1, 0], [0, 0, 1], [0, 0, -1.0]])
        l0.bias.zero_()
        nef.decoder.lout.weight.mul_(0.01); nef.decoder.lout.weight[0, :6] = 1.0 / np.sqrt(3.0)
        nef.decoder.lout.bias.fill_(-0.52 / np.sqrt(3.0))
    return nef


def test_phase_route_hash_field_exact(W):
    """NeuralSDF(HashGrid) at the nglod_hash shape: its sdf is wb_sdf_eval, one thread per point, so a point's value does not depend
    on its batch and the trace is exact."""
    case = _case()
    torch.manual_seed(0)
    blas = W.OctreeAS(dev(case["octree"]))
    grid = W.HashGrid.from_geometric(blas, feature_dim=8, num_lods=4, multiscale_type="cat", feature_std=0.01, codebook_bitwidth=19,
                                     min_grid_res=16, max_grid_res=2048)
    nef = _sdf_like(W.NeuralSDF(grid, pos_embedder="none", position_input=True, hidden_dim=128, num_layers=1).cuda(), 128)
    fd = W.ops.sdf_field(nef)
    assert fd is not None and fd[1] is None                                     # a hash field: wb_sdf_eval, the phase route
    lod = 3
    o, d = case["origins"], case["dirs"]
    ridx, depth = _nuggets(W, grid, o, d, lod)
    ref = TR.trace(o, d, ridx, depth, _device_field(lambda x, l: W.ops.sdf_eval(nef, x, l)), lod, 64, 0.8, 1e-3, 6.0)
    assert ref["hit"].sum() > 50
    got, tracer = _trace(W, nef, o, d, lod, 64, 0.8, 1e-3, 6.0)
    assert tracer.prev_num_evals is None
    _exact("nglod_hash", got, ref, normals=False)
    # the tracer's finite differences run with autograd enabled, where NeuralSDF.sdf takes the torch decoder (cuBLAS), not wb_sdf_eval
    both = got["hit"] & ref["hit"]
    assert np.quantile((got["normal"][both] * ref["normal"][both]).sum(-1), 0.01) > 0.999


def test_phase_route_triplanar_field(W):
    """NeuralSDF(TriplanarGrid) at the nglod_triplanar shape, scaled down (log_base_resolution 4, 32 wide): traced over its AABB
    (level 0 of the blas, triplanar_grid.py:152-157); torch Linear layers, whose rounding may depend on the batch."""
    case = _case()
    torch.manual_seed(1)
    grid = W.TriplanarGrid(W.AxisAlignedBBoxAS(), feature_dim=4, log_base_resolution=4, num_lods=1, multiscale_type="sum", feature_std=0.01)
    nef = _sdf_like(W.NeuralSDF(grid, pos_embedder="none", position_input=True, hidden_dim=32, num_layers=1).cuda(), 32)
    assert W.ops.sdf_field(nef) is None
    o, d = case["origins"], case["dirs"]
    ridx, depth = _nuggets(W, grid, o, d, 0)
    assert ridx.shape[0] == np.unique(ridx).shape[0] > 100                     # one AABB nugget per ray that meets the box
    ref = TR.trace(o, d, ridx, depth, _device_field(lambda x, l: nef(coords=x, lod_idx=0 if l is None else l, channels="sdf")), 0, 64, 0.8, 1e-3, 6.0)
    got, _ = _trace(W, nef, o, d, 0, 64, 0.8, 1e-3, 6.0)
    _close("nglod_triplanar (scaled)", got, ref)


def test_phase_route_cat_octree_below_finest(W):
    """A 'cat' NeuralSDF(OctreeGrid) traced at lod_idx 1 of 3 (its decoder takes the two LODs' features): the phase route with the
    torch field.  No normals: the finite differences evaluate the finest LOD, which this decoder cannot take."""
    from gpu_util import sdf_nef_from_case
    case = OG.make_sdf_case(level=5, num_lods=3, feature_dim=8, hidden_dim=16, multiscale="cat", res=32, seed=9)
    nef = sdf_nef_from_case(case)
    lod, F = 1, case["feature_dim"]
    dec = W.BasicDecoder(3 + F * (lod + 1), 1, torch.relu, True, torch.nn.Linear, 1, case["hidden_dim"]).cuda()
    with torch.no_grad():
        dec.layers[0].weight.copy_(dev(case["W"][0][:, :3 + F * (lod + 1)])); dec.layers[0].bias.copy_(dev(case["b"][0]))
        dec.lout.weight.copy_(dev(case["W"][1])); dec.lout.bias.copy_(dev(case["b"][1]))
    nef.decoder = dec
    assert W.ops.sdf_field(nef) is None
    o, d = case["origins"], case["dirs"]
    ridx, depth = _nuggets(W, nef.grid, o, d, lod)
    ref = TR.trace(o, d, ridx, depth, _device_field(lambda x, l: nef(coords=x, lod_idx=l, channels="sdf")), lod, 32, 0.8, 1e-3, 6.0,
                   with_normals=False)
    got, _ = _trace(W, nef, o, d, lod, 32, 0.8, 1e-3, 6.0, normals=False)
    _close("'cat' octree at lod 1 of 3", got, ref, normals=False)


# ---------------------------------------------------------------------------------------------------------------
# persistent kernel, several packs per thread
# ---------------------------------------------------------------------------------------------------------------
def _config3():
    from gpu_util import sdf_nef_from_case
    case = OG.make_sdf_case(level=7, num_lods=6, feature_dim=16, hidden_dim=128, multiscale="sum", res=8, seed=11, feature_std=0.02)
    return case, sdf_nef_from_case(case)


def _l3_h128(W):
    from sdf_shapes import make_field
    field, case = make_field("l3_h128")
    field.Ws[-1][:, 6:] *= 0.1                      # |grad| ~ 1, as test_gpu_sdf_kernels.py's trace check
    blas = W.OctreeAS(dev(case["octree"]))
    grid = W.OctreeGrid(blas, feature_dim=field.F, num_lods=field.num_lods, multiscale_type=field.multiscale, feature_std=0.0)
    grid.half_features = field.half
    pos = {0: ("none", False), 1: ("none", True), 2: ("positional", False), 3: ("positional", True)}[field.pos_mode]
    nef = W.NeuralSDF(grid, pos_embedder=pos[0], pos_multires=max(field.pos_freq, 1), position_input=pos[1], hidden_dim=field.Ws[0].shape[0],
                      num_layers=len(field.Ws) - 1).cuda()
    with torch.no_grad():
        for f, r in zip(grid.features, field.feats):
            f.copy_(dev(r))
        for l, Wm, b in zip(list(nef.decoder.layers) + [nef.decoder.lout], field.Ws, field.bs):
            l.weight.copy_(dev(Wm)); l.bias.copy_(dev(b))
    return nef


@pytest.mark.parametrize("model,frame", [("config3", "bench512"), ("config3", "large"), ("l3_h128", "large")])
def test_persistent_kernel_many_packs_per_thread(W, model, frame):
    """wb_sdf_trace against the restatement fed by wb_sdf_eval of the same field (the same sdf_eval<FT,PT> device function): hits,
    points and depths bit for bit, and its evaluation counter (PackedSDFTracer.prev_num_evals) equal to the restatement's count."""
    if model == "config3":
        case, nef = _config3()
        steps, step_size, min_dis = 32, 0.8, 3e-4                               # bench.py --config 3
    else:
        nef = _l3_h128(W)
        steps, step_size, min_dis = 32, 0.8, 1e-3
    fd = W.ops.sdf_field(nef)
    assert fd is not None and fd[1] is not None
    lod = nef.grid.num_lods - 1
    o, d = _frame(512, 0.75) if frame == "bench512" else _frame(768, 0.4)
    ridx, depth = _nuggets(W, nef.grid, o, d, lod)
    ref = TR.trace(o, d, ridx, depth, _device_field(lambda x, l: W.ops.sdf_eval(nef, x, l)), lod, steps, step_size, min_dis, 6.0)
    if frame == "large":
        assert ref["packs"] > _pack_bound(), (ref["packs"], _pack_bound())
    got, tracer = _trace(W, nef, o, d, lod, steps, step_size, min_dis, 6.0)
    evals = int(tracer.prev_num_evals.item())
    print(f"{model} {frame}: device evaluations {evals}, restatement {ref['evals']}")
    _close(f"{model} {frame}", got, ref)
    _exact(f"{model} {frame}", got, ref, normals=False)
    both = got["hit"] & ref["hit"]
    assert np.quantile((got["normal"][both] * ref["normal"][both]).sum(-1), 0.01) > 0.999
    assert evals == ref["evals"]
