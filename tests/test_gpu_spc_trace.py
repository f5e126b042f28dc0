"""GPU tests (-m gpu) of the SPC render path: wb_spc_trace behind ops.spc_trace, SPCField and PackedSPCTracer.

  - golden: the reference's own SPCField + PackedSPCTracer (tests/golden/spc_trace.npz, tools/make_spc_golden.py): hit, rgb and alpha
    equal, depth within 1e-6, for the three colour sources; lod_idx below the finest level runs the reference body (torch +
    OctreeAS.raytrace) and equals the reference's output, negative colour rows included;
  - bit for bit against the existing traversal: with the point index in colors[:, 0] (exact below 2^24) the kernel's point and depth
    are the first nugget of every ray of ops.raytrace, on the adversarial octrees of tests/octree_reference.py up to random10 at
    several levels; its hit set lies between the unambiguous exact nuggets and the exact-or-ambiguous ones;
  - edge cases: origins inside occupied cells (entry 0), rays that miss or start past the cube, R = 0 (no launch), 1 and 2^20 + 3;
  - one library launch per native trace, and install() routes wisp's PackedSPCTracer through it."""
import os
import sys
import types

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import oracle as O

import octree_reference as OR

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "spc_trace.npz")
f32 = np.float32


@pytest.fixture(scope="module")
def W():
    import wisp_b200
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return wisp_b200


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def bits(a):
    return np.ascontiguousarray(a, f32).view(np.uint32)


def golden_field(W, z, name, src):
    feats = {"rgba": {"colors": dev(z[f"{name}_colors"])}, "normals": {"normals": dev(z[f"{name}_normals"])}, "coords": None}[src]
    return W.SPCField(dev(z[f"{name}_octree"]), features_dict=feats), W.Rays(dev(z[f"{name}_origins"]), dev(z[f"{name}_dirs"]))


def colour_ulps(src):
    """RGBA / 255.0 on the device is torch's multiply by the reciprocal, which can round one ulp away from the reference's CPU
    division; the normal and coordinate colours (add, multiply, division by 2^level) are exact on both."""
    return 1 if src == "rgba" else 0


def check_golden(rb, z, key, maxulp=0):
    hit = rb.hit.cpu().numpy()
    assert rb.hit.dtype == torch.bool and np.array_equal(hit, z[f"{key}_hit"])
    if maxulp:
        np.testing.assert_array_max_ulp(rb.rgb.cpu().numpy(), z[f"{key}_rgb"], maxulp=maxulp)
    else:
        assert np.array_equal(rb.rgb.cpu().numpy(), z[f"{key}_rgb"])
    assert np.array_equal(rb.alpha.cpu().numpy(), z[f"{key}_alpha"])
    assert rb.depth.shape == z[f"{key}_depth"].shape and np.abs(rb.depth.cpu().numpy() - z[f"{key}_depth"]).max() <= 1e-6
    return int(hit.sum())


# ---- the reference's own classes --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["octa5", "rand7"])
@pytest.mark.parametrize("src", ["rgba", "normals", "coords"])
def test_golden_native_route(W, name, src):
    z = np.load(GOLDEN)
    nef, rays = golden_field(W, z, name, src)
    np.testing.assert_array_max_ulp(nef.colors.cpu().numpy(), z[f"{name}_{src}_field_colors"], maxulp=colour_ulps(src))
    tracer = W.PackedSPCTracer()
    tracer(nef, rays)                                               # first call: colour view and octree handle
    n0 = W._cabi.launch_count()
    rb = tracer(nef, rays)
    assert W._cabi.launch_count() - n0 == 1                         # one library launch per native trace
    hits = check_golden(rb, z, f"{name}_{src}", colour_ulps(src))
    assert 0 < hits < rays.origins.shape[0]
    rb2 = tracer(nef, rays, lod_idx=nef.grid.blas.max_level)
    assert all(torch.equal(getattr(rb, c), getattr(rb2, c)) for c in ("depth", "hit", "rgb", "alpha"))


@pytest.mark.parametrize("src", ["rgba", "normals", "coords"])
def test_golden_coarser_level_runs_the_reference_body(W, src, monkeypatch):
    """lod_idx 3 of a level-5 SPC: the reference body over OctreeAS.raytrace, colours indexed with negative rows (packed_spc_tracer.py
    :56-90 + spc_field.py:130-147); wb_spc_trace is not called."""
    z = np.load(GOLDEN)
    nef, rays = golden_field(W, z, "octa5", src)
    monkeypatch.setattr(W.ops, "spc_trace", lambda *a, **k: pytest.fail("lod_idx < max_level must not take the native route"))
    rb = W.PackedSPCTracer()(nef, rays, lod_idx=3)
    check_golden(rb, z, f"octa5_{src}_lod3", colour_ulps(src))


def test_float64_colours_fail_as_in_the_reference(W):
    """The reference's f32 rgb buffer refuses float64 colours (packed_spc_tracer.py:87): such a field takes the reference body and
    raises the same error rather than being rendered natively."""
    z = np.load(GOLDEN)
    nef = W.SPCField(dev(z["octa5_octree"]), features_dict={"normals": dev(z["octa5_normals"].astype(np.float64))})
    assert nef.colors.dtype == torch.float64 and W.ops.spc_colors(nef) is None
    with pytest.raises(RuntimeError, match="dtypes match"):
        W.PackedSPCTracer()(nef, W.Rays(dev(z["octa5_origins"]), dev(z["octa5_dirs"])))


# ---- against the existing traversal -----------------------------------------------------------------------------------------
def first_nuggets(W, oct, o, d, level):
    ridx, pidx, depth, offsets = W.ops.raytrace(oct, o, d, level)
    cnt = torch.diff(offsets)
    hit = cnt > 0
    first = offsets[:-1][hit]
    return hit, pidx[first], depth[first, 0]


def index_colors(T):
    """[T, 3] colours: the point index (exact in fp32 below 2^24) and two values derived from it."""
    i = torch.arange(T, dtype=torch.float32, device="cuda")
    return torch.stack([i, i * 0.5 + 0.25, -i], 1).contiguous()


def check_against_raytrace(W, oct, o, d, level, T):
    colors = index_colors(T)
    rb = W.ops.spc_trace(oct, o, d, level, colors, 0)
    hit, pidx, entry = first_nuggets(W, oct, o, d, level)
    assert torch.equal(rb.hit, hit)
    assert torch.equal(rb.rgb[hit], colors[pidx.long()]) and torch.equal(rb.rgb[hit, 0], pidx.float())
    assert np.array_equal(bits(rb.depth[hit, 0].cpu().numpy()), bits(entry.cpu().numpy()))
    assert bool((rb.alpha[hit] == 1).all())
    miss = ~hit
    assert not rb.depth[miss].any() and not rb.rgb[miss].any() and not rb.alpha[miss].any()
    return rb


NAMES = ["lego5", "lego6", "lego7", "corner_lo4", "corner_hi4", "dense1", "dense2", "dense3", "checker4", "faces5", "random8", "random9", "random10"]


@pytest.mark.parametrize("name", NAMES)
def test_first_nugget_of_raytrace_and_exact(W, name):
    pts, level = OR.octree_points(name)
    spc = O.octree_to_spc(O.points_to_octree(pts, level))
    idx = OR.OctIndex(spc)
    o, d, groups = OR.adversarial_rays(pts, level)
    blas = W.OctreeAS(dev(spc.octree))
    oct = blas.tensors()
    T = int(spc.pyramid[1, level] + spc.pyramid[0, level])
    for lv in sorted({1, max(level // 2, 1), level - 1, level} - {0}):
        rb = check_against_raytrace(W, oct, dev(o), dev(d), lv, T)
        hit, pidx, depth = rb.hit.cpu().numpy(), rb.rgb[:, 0].cpu().numpy().astype(np.int64), rb.depth[:, 0].cpu().numpy().astype(np.float64)
        ref = OR.nuggets(idx, o, d, lv)
        sure = np.unique(ref["ray"][ref["exact"] & ~ref["amb"]])
        assert hit[sure].all(), "a ray with an unambiguous exact nugget missed"
        rk = (ref["ray"] << 32) | ref["pidx"]
        rays = np.flatnonzero(hit)
        kk = (rays << 32) | pidx[rays]
        pos = np.searchsorted(np.sort(rk), kk)
        srt = np.argsort(rk)
        assert (rk[srt][np.minimum(pos, rk.shape[0] - 1)] == kk).all(), "a hit outside the exact-or-ambiguous nuggets"
        row = srt[np.minimum(pos, rk.shape[0] - 1)]
        assert (np.abs(depth[rays] - ref["entry"][row]) <= ref["r_entry"][row]).all(), "hit depth outside the rounding radius"
        if name.startswith(("dense", "faces")):                        # zero direction components and rays along cell faces hit
            assert hit[groups["zero_components_on_grid"]].any() and hit[groups["along_faces"]].any()
        ino = groups["in_occupied"]
        assert hit[ino].all() and not depth[ino].any()               # origin inside an occupied cell: entry clamped to 0
        print(f"SPCREPORT {name} level={lv} rays={o.shape[0]} hits={int(hit.sum())} ambiguous={int(ref['amb'].sum())}")


def test_misses_and_rays_past_the_cube(W):
    pts, level = OR.octree_points("dense3")
    blas = W.OctreeAS(dev(O.points_to_octree(pts, level)))
    rng = np.random.default_rng(5)
    o = rng.uniform(-1, 1, (256, 3))
    ax = rng.integers(0, 3, 256)
    s = rng.choice([-1.0, 1.0], 256)
    o[np.arange(256), ax] = s * rng.uniform(1.0 + 2 ** -20, 3.0, 256)             # past a face of the cube ...
    d = OR._unit(rng.standard_normal((256, 3)))
    d[np.arange(256), ax] = s * np.abs(d[np.arange(256), ax]) + s * 1e-3               # ... moving away from it
    beside = np.array([[-3.0, 1.5, 0.2], [0.2, -3.0, -1.0 - 2 ** -23], [1.0, 1.0, 3.0]], f32)   # parallel to the cube, outside it
    dirs = np.array([[1.0, 0.0, 0.0], [0.0, 1.0, 0.0], [0.0, 0.0, -1.0]], f32)
    o, d = np.concatenate([o.astype(f32), beside]), np.concatenate([d.astype(f32), dirs])
    rb = check_against_raytrace(W, blas.tensors(), dev(o), dev(d), level, int(blas.pyramid[1, level] + blas.pyramid[0, level]))
    assert not rb.hit.any()


@pytest.mark.parametrize("R", [0, 1, (1 << 20) + 3])
def test_ray_counts(W, R):
    pts, level = OR.octree_points("random8")
    blas = W.OctreeAS(dev(O.points_to_octree(pts, level)))
    oct = blas.tensors()
    T = int(blas.pyramid[1, level] + blas.pyramid[0, level])
    g = torch.Generator(device="cuda").manual_seed(R)
    o = torch.rand(R, 3, device="cuda", generator=g) * 3.0 - 1.5
    d = torch.nn.functional.normalize(torch.randn(R, 3, device="cuda", generator=g), dim=-1)
    colors = index_colors(T)
    n0 = W._cabi.launch_count()
    rb = W.ops.spc_trace(oct, o, d, level, colors, 0)
    assert W._cabi.launch_count() - n0 == (0 if R == 0 else 1)
    assert rb.depth.shape == (R, 1) and rb.hit.shape == (R,) and rb.rgb.shape == (R, 3) and rb.alpha.shape == (R, 1)
    if R:
        check_against_raytrace(W, oct, o, d, level, T)


def test_colour_rows_are_checked(W):
    """The kernel gathers colors[pidx - point_offset]: too few rows, a row stride other than 1 or an offset past the level is refused."""
    pts, level = OR.octree_points("dense2")
    blas = W.OctreeAS(dev(O.points_to_octree(pts, level)))
    o, d = dev(np.zeros((4, 3), f32)), dev(np.ones((4, 3), f32))
    first, M = int(blas.pyramid[1, level]), int(blas.pyramid[0, level])
    ok = torch.zeros(M, 3, device="cuda")
    W.ops.spc_trace(blas.tensors(), o, d, level, ok, first)
    for colors, off in ((ok[:-1], first), (torch.zeros(M, 3, 2, device="cuda")[..., 0], first), (ok, first + 1), (ok.double(), first)):
        with pytest.raises(W.WispB200Error):
            W.ops.spc_trace(blas.tensors(), o, d, level, colors, off)


# ---- install() ----------------------------------------------------------------------------------------------------------------
@pytest.fixture
def fake_wisp(W):
    """A stand-in for the modules install() imports, with wisp's class names; PackedSPCTracer is the reference's interface
    (bg_color (0, 0, 0), channels) whose own trace() must not run."""
    class Stub:
        def __getattr__(self, name):
            raise AssertionError(f"stub {name}")

    def cls(name, *methods, base=object):
        return type(name, (base,), {m: (lambda self, *a, **k: None) for m in methods})

    class RenderBuffer:
        def __init__(self, **kw):
            self.__dict__.update(kw)
            self.order = list(kw)

    class PackedSPCTracer(W.tracers.BaseTracer):
        def __init__(self):
            super().__init__()
            self.bg_color = (0.0, 0.0, 0.0)

        def get_supported_channels(self):
            return {"depth", "hit", "rgb", "alpha"}

        def get_required_nef_channels(self):
            return {"rgb"}

        def trace(self, nef, rays, channels, extra_channels, lod_idx=None):
            raise AssertionError("the unpatched reference body ran")

    mods = {
        "wisp": {}, "wisp.ops": {}, "wisp.ops.grid": {"hashgrid": lambda *a: None},
        "wisp.accelstructs": {"OctreeAS": cls("OctreeAS", "query", "raytrace", "_raymarch_ray", "_raymarch_voxel", "_raymarch_uniform")},
        "wisp.accelstructs.base_as": {"ASQueryResults": Stub, "ASRaymarchResults": Stub, "ASRaytraceResults": Stub},
        "wisp.core": {"RenderBuffer": RenderBuffer},
        "wisp.models": {}, "wisp.models.grids": {n: cls(n, "interpolate") for n in ("HashGrid", "OctreeGrid", "TriplanarGrid")},
        "wisp.models.nefs": {"NeuralRadianceField": cls("NeuralRadianceField", "prune"), "NeuralSDF": cls("NeuralSDF", "sdf")},
        "wisp.tracers": {"PackedRFTracer": cls("PackedRFTracer", "trace"), "PackedSDFTracer": cls("PackedSDFTracer", "trace"),
                         "PackedSPCTracer": PackedSPCTracer},
    }
    saved = {k: sys.modules.get(k) for k in list(sys.modules) if k == "wisp" or k.startswith("wisp.")}
    for k in saved:
        del sys.modules[k]
    for k, attrs in mods.items():
        m = types.ModuleType(k)
        m.__path__ = []
        m.__dict__.update(attrs)
        sys.modules[k] = m
    try:
        yield sys.modules["wisp.tracers"].PackedSPCTracer, RenderBuffer
    finally:
        from wisp_b200 import install as I
        I.uninstall()
        for k in mods:
            sys.modules.pop(k, None)
        sys.modules.update({k: v for k, v in saved.items() if v is not None})


def test_install_renders_wisp_tracer_natively(W, fake_wisp):
    from wisp_b200 import install as I
    Tracer, RenderBuffer = fake_wisp
    z = np.load(GOLDEN)
    nef, rays = golden_field(W, z, "rand7", "coords")
    assert I.install() is True
    tracer = Tracer()
    tracer(nef, rays)
    n0 = W._cabi.launch_count()
    rb = tracer(nef, rays)
    assert W._cabi.launch_count() - n0 == 1
    assert isinstance(rb, RenderBuffer) and rb.order == ["depth", "hit", "rgb", "alpha"]
    check_golden(rb, z, "rand7_coords")
