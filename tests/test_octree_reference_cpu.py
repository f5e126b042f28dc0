"""CPU tests of tests/octree_reference.py, the exact reference of the octree traversal kernels, against the C oracle
(oracle/wisp_oracle.c) on the adversarial octrees and rays of the GPU tests (tests/test_gpu_octree_traversal.py):
  - cell_of is floor((x + 1) * 2^(L-1)) on the values where float64 rounds, and oracle query == cell_of + descent;
  - every oracle nugget is an exact nugget or an ambiguous cell, every unambiguous exact nugget is an oracle nugget, and the
    oracle's entry / exit lie within the rounding radius: this pins the nugget definition the kernel and the oracle share
    against an independent statement of it;
  - the oracle's 'ray' samples are march_depths / march_hits: candidate depths bit for bit, hits exactly."""
from fractions import Fraction

import numpy as np
import pytest

from oracle import oracle as O

import octree_reference as OR

f32 = np.float32

OCTREES = ["lego5", "corner_lo4", "corner_hi4", "dense2", "checker4", "random8", "lines11", "faces5"]


def _spc(name):
    pts, level = OR.octree_points(name)
    spc = O.octree_to_spc(O.points_to_octree(pts, level))
    return spc, OR.OctIndex(spc), pts, level


def test_cell_of_exact_where_float64_rounds():
    for level in (1, 4, 10, 15):
        h = 2 ** (level - 1)
        xs = np.array([-2.0 ** -60, 2.0 ** -60, -2.0 ** -149, 0.0, -0.0, -1.0, 1.0, np.nextafter(f32(1), f32(0)),
                       np.nextafter(f32(-1), f32(0)), np.nextafter(f32(-1), f32(-2)), -1 + 2.0 ** -level, 0.3, -0.7], f32)
        q, inside = OR.cell_of(xs, level)
        for x, qi, ii in zip(xs, q, inside):
            v = (Fraction(float(x)) + 1) * h
            e = v.numerator // v.denominator
            assert ii == (0 <= e < 2 ** level) and (not ii or qi == e), (level, x, qi, e)
        assert q[0] == h - 1 and q[1] == h and q[3] == h and q[4] == h


@pytest.mark.parametrize("name", OCTREES)
def test_query_is_cell_of_plus_descent(name):
    spc, idx, pts, level = _spc(name)
    o, d, _ = OR.adversarial_rays(pts, level)
    rng = np.random.default_rng(3)
    k = (rng.integers(0, (1 << level) + 1, (2000, 3)) / 2.0 ** (level - 1) - 1.0).astype(f32)
    coords = np.concatenate([o, np.clip(o + d * f32(0.5), -3, 3), k, np.nextafter(k, f32(-2)), np.nextafter(k, f32(2)),
                             rng.uniform(-1.05, 1.05, (4000, 3)).astype(f32), np.array([[-2.0 ** -60, 2.0 ** -60, -0.0]], f32)])
    for lv in sorted({1, level // 2, level}):
        assert np.array_equal(O.query(spc, coords, lv), idx.query(coords, lv))
        assert np.array_equal(O.query(spc, coords, lv, with_parents=True), idx.query(coords, lv, with_parents=True))


@pytest.mark.parametrize("name", OCTREES)
def test_oracle_nuggets_against_exact(name):
    spc, idx, pts, level = _spc(name)
    o, d, groups = OR.adversarial_rays(pts, level)
    for lv in sorted({level, max(level - 2, 0)}):
        ref = OR.nuggets(idx, o, d, lv)
        rt = O.raytrace(spc, o, d, lv)
        n, amb, ratio = OR.check_nuggets(ref, spc, lv, rt["ridx"], rt["pidx"], rt["depth"])
        print(f"TRAVREPORT cpu-oracle {name} level={lv} rays={o.shape[0]} nuggets={n} ambiguous={amb} max|k-exact|/radius={ratio:.3f}")
        assert n > 0 or name.startswith("corner")


def test_nugget_check_catches_a_wrong_definition():
    """The same check fails an oracle whose slab depths carry an extra error, or that loses a nugget of a ray along a face."""
    spc, idx, pts, level = _spc("lego5")
    o, d, groups = OR.adversarial_rays(pts, level)
    ref = OR.nuggets(idx, o, d, level)
    rt = O.raytrace(spc, o, d, level)
    bad = rt["depth"].copy()
    bad[:, 0] = np.where(bad[:, 0] > 0, np.nextafter(np.nextafter(bad[:, 0], f32(9)), f32(9)), bad[:, 0])
    with pytest.raises(AssertionError):
        OR.check_nuggets(ref, spc, level, rt["ridx"], rt["pidx"], bad)
    # an axis-aligned ray running along cell faces: losing one of its nuggets is caught
    g = groups["along_faces"]
    rows = np.flatnonzero((rt["ridx"] >= g.start) & (rt["ridx"] < g.stop))
    assert rows.size > 0
    keep = np.ones(rt["ridx"].shape[0], bool)
    keep[rows[0]] = False
    with pytest.raises(AssertionError):
        OR.check_nuggets(ref, spc, level, rt["ridx"][keep], rt["pidx"][keep], rt["depth"][keep])


@pytest.mark.parametrize("name,n,pernear", [("lego5", 33, False), ("checker4", 64, True), ("faces5", 100, True), ("lines11", 31, False)])
def test_oracle_march_is_march_hits(name, n, pernear):
    spc, idx, pts, level = _spc(name)
    o, d, _ = OR.adversarial_rays(pts, level)
    R = o.shape[0]
    rng = np.random.default_rng(5)
    jit = rng.random((R, n), dtype=f32)
    jit[:, 0] = 0.0
    jit[:, -1] = np.nextafter(f32(1), f32(0))
    if pernear:
        near = rng.uniform(-1.0, 2.0, R).astype(f32); far = (near + rng.uniform(0.0, 6.0, R)).astype(f32)
        near[:8] = far[:8]; far[8:16] = near[8:16] - f32(1.0); far[16:24] = f32(1e6)
    else:
        near, far = 0.0, 6.0
    mr = O.raymarch_ray(spc, o, d, near, far, n, level, jitter_arr=jit)
    dep = OR.march_depths(R, n, near, far, jit)
    assert np.array_equal(dep[mr["ridx"], mr["step_idx"]].view(np.uint32), mr["depth_samples"][:, 0].view(np.uint32))
    hits = OR.march_hits(idx, o, d, dep, level)
    got = np.zeros((R, n), bool)
    got[mr["ridx"], mr["step_idx"]] = True
    assert np.array_equal(got, hits)
    assert np.array_equal(mr["counts"], hits.sum(1))
    # the seeded stream restated in numpy is the oracle's
    js = OR.jitter_stream(77, 5, 9)
    assert all(js[r, s] == O.jitter(77, r, s) for r in range(5) for s in range(9))
