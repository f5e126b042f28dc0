"""GPU tests (-m gpu) of the kernels that decide where samples are: wb_query, the 'ray' marcher (wb_raymarch_ray_count / _fill,
wb_rf_march_fill), wb_scan_counts, wb_raytrace_* with and without the nugget cache, and the 'voxel' / 'uniform' samplers.

Inputs are the adversarial octrees and rays of tests/octree_reference.py (single voxels in the corners, dense, checkerboard,
1 % random up to level 10, sparse lines to level 15, an occupied box touching the +-1 faces; origins on dyadic faces / edges /
corners and one ulp beside them, +-0.0 and 1e-13 / denormal direction components, unnormalised directions, far origins).
Every output is bit-exact against the C oracle, and the oracle-independent statements are checked as well:
  - query == cell_of + descent;
  - the marcher's hits == march_hits on the candidate depths, and neither the bounding-box cull nor the coarse word skipping
    changes a hit mask;
  - raytrace nuggets == the exact nuggets up to ambiguous cells, with entry / exit within the rounding radius.
Each case prints one TRAVREPORT line: counts, ambiguous cells and max |k - exact| / radius (<= 1)."""
import ctypes as C

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import oracle as O

import octree_reference as OR

f32 = np.float32
_SPC = {}


@pytest.fixture(scope="module")
def W():
    import wisp_b200
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return wisp_b200


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def bits(a):
    return np.ascontiguousarray(a).view(np.uint32 if np.asarray(a).dtype == np.float32 else np.asarray(a).dtype)


def octree_case(name):
    """-> (oracle SPC, OctIndex, points, level, rays o, d, groups), cached per module."""
    if name not in _SPC:
        pts, level = OR.octree_points(name)
        spc = O.octree_to_spc(O.points_to_octree(pts, level))
        o, d, groups = OR.adversarial_rays(pts, level)
        _SPC[name] = (spc, OR.OctIndex(spc), pts, level, o, d, groups)
    return _SPC[name]


# ---- query ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["lego6", "corner_hi4", "dense3", "checker4", "random10", "lines15", "faces5"])
def test_query_is_cell_of_plus_descent(W, name):
    spc, idx, pts, level, o, d, _ = octree_case(name)
    rng = np.random.default_rng(1)
    k = (rng.integers(0, (1 << level) + 1, (3000, 3)) / 2.0 ** (level - 1) - 1.0).astype(f32)
    inside = ((pts[rng.integers(0, pts.shape[0], 3000)] + rng.uniform(0, 1, (3000, 3))) / 2.0 ** (level - 1) - 1.0).astype(f32)
    coords = np.concatenate([o, k, np.nextafter(k, f32(-2)), np.nextafter(k, f32(2)), inside,
                             np.array([[-2.0 ** -60, 2.0 ** -60, -0.0], [1.0, -1.0, 0.0], [-1e-45, 1e-45, 0.5]], f32)])
    blas = W.OctreeAS(dev(spc.octree))
    levels = range(1, level + 1) if level >= 11 else sorted({1, level // 2, level})
    for lv in levels:
        for wp in (False, True):
            got = blas.query(dev(coords), level=lv, with_parents=wp).pidx.cpu().numpy()
            assert np.array_equal(got, idx.query(coords, lv, with_parents=wp)), (lv, wp)
            assert np.array_equal(got, O.query(spc, coords, lv, with_parents=wp)), (lv, wp)


# ---- raymarch 'ray' ---------------------------------------------------------------------------------------------------------
def _near_far(mode, R, rng):
    if mode == "scalar":
        return 0.0, 6.0
    near = rng.uniform(-1.0, 2.0, R).astype(f32)
    far = (near + rng.uniform(0.5, 6.0, R)).astype(f32)
    near[:16] = f32(-3.0)                       # near < 0
    far[16:32] = near[16:32]                    # far == near
    far[32:48] = near[32:48] - f32(1.5)         # far < near
    far[48:64] = f32(1e6)
    return near, far


MARCH = [  # octree, march level, n, near/far, jitter, COARSE_LEVEL
    ("lego5", 5, 1, "scalar", "seeded", 6), ("lego6", 6, 2, "pernear", "explicit", 2), ("lego7", 7, 2048, "scalar", "explicit", 6),
    ("lego7", 5, 64, "pernear", "explicit", 2), ("dense1", 1, 31, "scalar", "explicit", 6), ("dense3", 3, 32, "pernear", "explicit", 2),
    ("checker4", 4, 33, "scalar", "explicit", 2), ("corner_lo4", 4, 4096, "scalar", "seeded", 2), ("corner_hi4", 4, 2049, "pernear", "seeded", 2),
    ("faces5", 5, 2047, "pernear", "explicit", 6), ("random8", 8, 64, "scalar", "seeded", 6), ("random10", 10, 33, "pernear", "explicit", 6),
    ("lines11", 11, 256, "scalar", "explicit", 6), ("lines12", 12, 100, "pernear", "seeded", 0), ("faces5", 5, 32, "scalar", "explicit", 0),
]


@pytest.mark.parametrize("name,level,n,nf,jmode,coarse", MARCH, ids=lambda v: str(v))
def test_raymarch_ray(W, name, level, n, nf, jmode, coarse):
    from wisp_b200 import ops
    spc, idx, pts, _, o, d, _ = octree_case(name)
    R = o.shape[0]
    rng = np.random.default_rng(n)
    near, far = _near_far(nf, R, rng)
    if jmode == "explicit":
        jit = rng.random((R, n), dtype=f32)
        jit[::2, 0] = 0.0
        jit[1::2, -1] = np.nextafter(f32(1), f32(0))
        jit[:, n // 2] = np.nextafter(f32(1), f32(0))
    else:
        jit = OR.jitter_stream(7, R, n)
    near_t = near if nf == "scalar" else dev(near)[:, None]
    far_t = far if nf == "scalar" else dev(far)[:, None]
    jt = dev(jit) if jmode == "explicit" else None
    saved = ops.COARSE_LEVEL
    try:
        ops.COARSE_LEVEL = coarse
        blas = W.OctreeAS(dev(spc.octree))
        oct = blas.tensors()
        ms = ops.march_count(oct, dev(o), dev(d), near_t, far_t, n, level, jitter=jt, seed=7)
        assert (oct.bbox is not None) == (level <= 10)
        assert (oct.coarse is not None) == (level <= 10 and min(level - 1, coarse) >= 2)
        ridx, samples, depth, deltas, boundary = ops.march_fill_reference_layout(ms, "cuda")
        rec_t, rec_delta, rec_ray = ops.march_fill_records(ms, "cuda")
        hm, cnt = ms.hitmask.cpu().numpy(), ms.counts.cpu().numpy()
        # culling is sound: no bounding box (and so no coarse mask), and no coarse mask, give the same hits
        oct.bbox = None
        m2 = ops.march_count(oct, dev(o), dev(d), near_t, far_t, n, level, jitter=jt, seed=7)
        ops.COARSE_LEVEL = 0
        b3 = W.OctreeAS(dev(spc.octree))
        m3 = ops.march_count(b3.tensors(), dev(o), dev(d), near_t, far_t, n, level, jitter=jt, seed=7)
        assert b3.tensors().coarse is None
    finally:
        ops.COARSE_LEVEL = saved
    for m in (m2, m3):
        assert m.total == ms.total and np.array_equal(m.counts.cpu().numpy(), cnt) and np.array_equal(m.hitmask.cpu().numpy(), hm)
    ref = O.raymarch_ray(spc, o, d, near, far, n, level, jitter_arr=jit if jmode == "explicit" else None, seed=7)
    assert ms.total == ref["ridx"].shape[0] and np.array_equal(cnt, ref["counts"])
    assert np.array_equal(ridx.cpu().numpy(), ref["ridx"]) and np.array_equal(boundary.cpu().numpy(), ref["boundary"])
    for got, exp in ((samples, ref["samples"]), (depth, ref["depth_samples"]), (deltas, ref["deltas"])):
        assert np.array_equal(bits(got.cpu().numpy()), bits(exp))
    assert np.array_equal(bits(rec_t.cpu().numpy()), bits(ref["depth_samples"][:, 0]))
    assert np.array_equal(bits(rec_delta.cpu().numpy()), bits(ref["deltas"][:, 0]))
    assert np.array_equal(rec_ray.cpu().numpy(), ref["ridx"])
    assert np.array_equal(ms.offsets.cpu().numpy(), np.concatenate([[0], np.cumsum(cnt, dtype=np.int64)]))
    # hits == cell_of + descent of fma(d, t, o) on the candidate depths (which are the oracle's, bit for bit)
    dep = OR.march_depths(R, n, near, far, jit)
    assert np.array_equal(bits(dep[ref["ridx"], ref["step_idx"]]), bits(ref["depth_samples"][:, 0]))
    hits = OR.march_hits(idx, o, d, dep, level)
    assert np.array_equal(OR.hit_matrix_from_mask(hm, n), hits)
    print(f"TRAVREPORT march {name} level={level} n={n} {nf} {jmode} coarse={coarse} rays={R} samples={ms.total} "
          f"rays_hit={int((cnt > 0).sum())} ambiguous=0 max|k-exact|/radius=0 (bit-exact)")


# ---- raytrace ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name,level", [("lego5", 5), ("lego6", 6), ("lego7", 7), ("lego7", 4), ("corner_lo4", 4), ("corner_hi4", 4),
                                        ("dense1", 1), ("dense2", 2), ("dense3", 3), ("checker4", 4), ("random8", 8), ("random9", 9),
                                        ("random10", 10), ("lines11", 11), ("lines12", 12), ("lines15", 15), ("faces5", 5)])
def test_raytrace_against_oracle_and_exact(W, name, level):
    spc, idx, pts, _, o, d, _ = octree_case(name)
    blas = W.OctreeAS(dev(spc.octree))
    rt = blas.raytrace(W.Rays(dev(o), dev(d)), level, with_exit=True)
    ridx, pidx, depth = rt.ridx.cpu().numpy(), rt.pidx.cpu().numpy(), rt.depth.cpu().numpy()
    ref = O.raytrace(spc, o, d, level)
    assert np.array_equal(ridx, ref["ridx"]) and np.array_equal(pidx, ref["pidx"]) and np.array_equal(bits(depth), bits(ref["depth"]))
    n, amb, ratio = OR.check_nuggets(OR.nuggets(idx, o, d, level), spc, level, ridx, pidx, depth)
    print(f"TRAVREPORT raytrace {name} level={level} rays={o.shape[0]} nuggets={n} ambiguous={amb} max|k-exact|/radius={ratio:.3f}")


def test_raytrace_nugget_cache_sizes(W):
    """Rays with more than 200 nuggets (diagonals of a dense level-7 octree), R not a multiple of 128: the cached single traversal
    gives exactly the nuggets of the two-traversal form for every cache size."""
    pts, level = OR.octree_points("dense7")
    spc = O.octree_to_spc(O.points_to_octree(pts, level))
    rng = np.random.default_rng(2)
    tgt = rng.uniform(-0.3, 0.3, (300, 3)).astype(f32)
    src = (np.sign(rng.uniform(-1, 1, (300, 3))) * 1.6 + rng.uniform(-0.05, 0.05, (300, 3))).astype(f32)
    o, d = src, (tgt - src).astype(f32)
    blas = W.OctreeAS(dev(spc.octree))
    outs = []
    old = W.ops.RAYTRACE_CACHE_K
    try:
        for K in (0, 1, 2, 24, 200):
            W.ops.RAYTRACE_CACHE_K = K
            outs.append([t.cpu().numpy() for t in W.ops.raytrace(blas.tensors(), dev(o), dev(d), level)])
    finally:
        W.ops.RAYTRACE_CACHE_K = old
    counts = np.diff(outs[0][3])
    assert counts.max() > 200 and (counts > 24).sum() > 100
    for other in outs[1:]:
        for a, b in zip(outs[0], other):
            assert np.array_equal(bits(a), bits(b))
    ref = O.raytrace(spc, o, d, level)
    assert np.array_equal(outs[0][1], ref["pidx"]) and np.array_equal(bits(outs[0][2]), bits(ref["depth"]))
    print(f"TRAVREPORT raytrace-cache dense7 rays=300 nuggets={outs[0][0].shape[0]} max_per_ray={int(counts.max())} ambiguous=0 "
          f"max|k-exact|/radius=0 (bit-exact)")


# ---- 'voxel' / 'uniform' samplers -----------------------------------------------------------------------------------------------
def _sampler_rays(level):
    """adversarial rays of faces5 + rays whose nugget depths are integers over the uniform scale (ceilf ties) + origins 1e5 away."""
    spc, idx, pts, _, o, d, _ = octree_case("faces5")
    h = 2.0 ** (level - 1)
    rng = np.random.default_rng(4)
    y = (rng.integers(0, 1 << level, 32) + 0.5) / h - 1.0
    z = (rng.integers(0, 1 << level, 32) + 0.5) / h - 1.0
    ot = np.stack([np.full(32, -2.0), y, z], 1).astype(f32)          # entry at t = 1, exits at 1 + k / 16
    dt = np.tile(np.array([[1.0, 0.0, 0.0]], f32), (32, 1))
    dt[16:] *= f32(0.5)                                              # entry at t = 2
    dirn = OR._unit(rng.standard_normal((32, 3)))
    of = (rng.uniform(-0.9, 0.9, (32, 3)) + dirn * 1e5).astype(f32)
    return spc, np.concatenate([o, ot, of]).astype(f32), np.concatenate([d, dt, -dirn]).astype(f32)


@pytest.mark.parametrize("kind,n", [("voxel", 1), ("voxel", 3), ("voxel", 7), ("voxel", 64), ("uniform", 16), ("uniform", 1024)])
def test_nugget_samplers_vs_oracle(W, kind, n):
    spc, o, d = _sampler_rays(5)
    R = o.shape[0]
    blas = W.OctreeAS(dev(spc.octree))
    rays = W.Rays(dev(o), dev(d), 0.0, 10.0)
    rt = O.raytrace(spc, o, d, 5)
    if kind == "voxel":
        jit = np.random.default_rng(n).random((rt["ridx"].shape[0], n), dtype=f32)
        jit[::3, 0] = 0.0
        jit[1::3, -1] = np.nextafter(f32(1), f32(0))
        got = blas.raymarch(rays, 'voxel', n, 5, jitter=dev(jit))
        ref = O.raymarch_voxel(spc, o, d, n, 5, jitter_arr=jit)
        seeded = blas.raymarch(rays, 'voxel', n, 5, seed=3)
        rs = O.raymarch_voxel(spc, o, d, n, 5, seed=3)
        assert np.array_equal(bits(seeded.depth_samples.cpu().numpy()), bits(rs["depth_samples"]))
        extra = ""
    else:
        got = blas.raymarch(rays, 'uniform', n, 5)
        ref = O.raymarch_uniform(spc, o, d, n, 5)
        scale = ref["scale"]
        prod = (np.float32(scale) * rt["depth"]).astype(f32)
        ties = int((prod == np.ceil(prod)).sum())
        assert ties > 0                                              # the ceilf ties are exercised
        assert (prod > 2 ** 24).any() or n < 1024                    # and depths beyond fp32's integer range
        cnt = np.ceil(prod[:, 1]).astype(np.int64) - np.ceil(prod[:, 0]).astype(np.int64)
        first = np.r_[True, rt["ridx"][1:] != rt["ridx"][:-1]]
        dropped_first = np.unique(rt["ridx"][first & (cnt == 0)])
        later = np.unique(rt["ridx"][~first & (cnt > 0)])
        assert np.intersect1d(dropped_first, later).size > 0         # rays whose first nugget keeps no sample
        extra = f" ceil_ties={ties} dropped_first={dropped_first.size}"
    assert np.array_equal(got.ridx.cpu().numpy(), ref["ridx"]) and np.array_equal(got.boundary.cpu().numpy(), ref["boundary"])
    for a, b in ((got.samples, ref["samples"]), (got.depth_samples, ref["depth_samples"]), (got.deltas, ref["deltas"])):
        assert np.array_equal(bits(a.cpu().numpy()), bits(b))
    print(f"TRAVREPORT {kind} n={n} rays={R} nuggets={rt['ridx'].shape[0]} samples={ref['ridx'].shape[0]}{extra} ambiguous=0 "
          f"max|k-exact|/radius=0 (bit-exact)")


# ---- scan -----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("R", [0, 1, 4095, 4096, 4097, 1 << 20, (1 << 20) + 1, 3 * (1 << 20) + 7])
def test_scan_counts(W, R):
    rng = np.random.default_rng(R)
    c = rng.integers(0, 2000, R).astype(np.int32)
    if R > 10:
        c[rng.random(R) < 0.3] = 0
        c[R // 3: R // 3 + min(R // 4, 300000)] = 0                  # a run of zeros across chunks
        c[rng.integers(0, R, max(R // 1000, 1))] = 2 ** 31 - 1        # large values
    L = W._cabi.lib()
    counts = dev(c) if R else torch.zeros(1, dtype=torch.int32, device="cuda")
    offsets = torch.full((R + 1,), -7, dtype=torch.int64, device="cuda")
    wsb = int(L.wb_scan_workspace_bytes(C.c_int64(R)))
    ws = torch.empty(wsb, dtype=torch.uint8, device="cuda")
    W._cabi.check(L.wb_scan_counts(W._cabi.ptr(counts), C.c_int64(R), W._cabi.ptr(offsets), W._cabi.ptr(ws), C.c_int64(wsb), W._cabi.stream()))
    exp = np.concatenate([[0], np.cumsum(c.astype(np.int64))])
    assert np.array_equal(offsets.cpu().numpy(), exp)
    print(f"TRAVREPORT scan R={R} total={int(exp[-1])} ambiguous=0 max|k-exact|/radius=0 (exact)")
