"""tests/sdf_trace_reference.py, the vectorised and exactly rounded restatement of PackedSDFTracer.trace, against
oracle/octree_grid.py:sdf_trace (statement by statement, double-rounded addcmul), its find_depth_bound against the per-pack loop,
its fma against Fraction arithmetic, and both against tests/golden/sdf_octree.npz.  No device is touched."""
import os
from fractions import Fraction

import numpy as np
import pytest

from oracle import octree_grid as OG
from oracle import oracle as O

import sdf_trace_reference as TR

_CASES = {}


def _case(ms):
    if ms not in _CASES:
        _CASES[ms] = OG.make_sdf_case(level=5, num_lods=3, feature_dim=8, hidden_dim=16, multiscale=ms, res=24, seed=5)
    return _CASES[ms]


def _round_fp32(q: Fraction) -> np.float32:
    """Fraction -> nearest fp32, ties to even (normal range)."""
    if q == 0:
        return np.float32(0.0)
    f = np.float32(float(q))                 # within one ulp of q: pick the nearest of f and its neighbours exactly
    cands = [np.nextafter(f, np.float32(-np.inf)), f, np.nextafter(f, np.float32(np.inf))]
    d = [abs(Fraction(float(c)) - q) for c in cands]
    m = min(d)
    best = [c for c, e in zip(cands, d) if e == m]
    if len(best) == 1:
        return best[0]
    return next(c for c in best if (np.array(c, np.float32).view(np.int32) & 1) == 0)


def _fma_exact(a, b, c):
    return np.array([_round_fp32(Fraction(float(x)) * Fraction(float(y)) + Fraction(float(z))) for x, y, z in zip(a, b, c)], np.float32)


def test_fma32_random_inputs():
    rng = np.random.default_rng(0)
    n = 4000
    a = rng.standard_normal(n).astype(np.float32)
    b = (rng.standard_normal(n) * 10.0 ** rng.integers(-3, 3, n)).astype(np.float32)
    c = (rng.standard_normal(n) * 10.0 ** rng.integers(-3, 3, n)).astype(np.float32)
    c[: n // 4] = (-(a[: n // 4].astype(np.float64) * b[: n // 4])).astype(np.float32)      # cancellation
    got = TR.fma32(a, b, c)
    assert np.array_equal(got.view(np.int32), _fma_exact(a, b, c).view(np.int32))


def test_fma32_halfway_cases():
    """a*b + c exactly halfway between two fp32 values, and a hair off halfway (beyond float64 precision of the sum): a plain float64
    sum rounds these to the tie and then to even, the correctly rounded fma goes to the side of the tail."""
    rng = np.random.default_rng(1)
    n = 600
    c = rng.uniform(1.0, 2.0, n).astype(np.float32)          # ulp 2^-23, half an ulp 2^-24
    kind = rng.integers(0, 3, n)
    # kind 0: a*b = +-2^-24, a tie; kind 1/2: a*b = +-(2^-24 - 2^-60) = +-(1 + 2^-18)(1 - 2^-18) 2^-24, a tail 2^-36 of an ulp below
    # the tie, far below float64's resolution at c
    a = np.where(kind == 0, np.float32(1.0), np.float32(1.0 + 2.0 ** -18)).astype(np.float32)
    b = np.where(kind == 0, np.float32(2.0 ** -24), np.float32((1.0 - 2.0 ** -18) * 2.0 ** -24)).astype(np.float32)
    b = np.where(kind == 2, -b, b).astype(np.float32)
    exact = _fma_exact(a, b, c)
    got = TR.fma32(a, b, c)
    assert np.array_equal(got.view(np.int32), exact.view(np.int32))
    naive = (a.astype(np.float64) * b + c).astype(np.float32)
    assert (naive != exact).sum() > 50                 # the cases do separate double rounding from one rounding


def _fdb_inputs(rng, P, Ng):
    depth = np.sort(rng.uniform(0.0, 4.0, (Ng, 2)).astype(np.float32), axis=1)
    curr = np.sort(rng.integers(0, Ng, P)).astype(np.int32)
    curr[rng.random(P) < 0.15] = -1
    q = rng.uniform(-0.5, 4.5, P).astype(np.float32)
    return q, curr, depth


@pytest.mark.parametrize("seed", range(6))
def test_find_depth_bound_matches_loop(seed):
    rng = np.random.default_rng(seed)
    for P, Ng in ((1, 1), (1, 5), (7, 3), (40, 200), (300, 90), (500, 2000)):
        q, curr, depth = _fdb_inputs(rng, P, Ng)
        if P > 2:
            curr[-2] = -1                                  # a -1 neighbour of the last-but-one... and of pack P-3
            curr[1] = curr[2] if curr[2] >= 0 else curr[1]   # an empty range: the neighbour's cursor equals this one
        stats = {}
        got = TR.find_depth_bound(q, curr, depth, stats)
        assert np.array_equal(got, OG.find_depth_bound(q.reshape(-1, 1), curr, depth)), (seed, P, Ng)


def test_find_depth_bound_quirks():
    depth = np.array([[0.0, 1.0], [1.0, 2.0], [2.0, 3.0], [3.0, 4.0], [4.0, 5.0]], np.float32)
    # pack 0 beyond its own nuggets, scan stops at pack 1's cursor (2); pack 1 with a -1 neighbour scans to the end of the list; pack 3
    # (the last) is bounded by P = 4, not by the 5 nuggets
    q = np.array([2.5, 3.5, 9.0, 4.5], np.float32)
    curr = np.array([0, 2, -1, 3], np.int32)
    stats = {}
    got = TR.find_depth_bound(q, curr, depth, stats)
    assert got.tolist() == OG.find_depth_bound(q.reshape(-1, 1), curr, depth).tolist() == [-1, 3, -1, -1]
    assert stats["bound_stops"] == 1                       # pack 0; the last pack's bound is not counted


def _compare(a, b, what):
    """Equal array for array, except xyz/depth where oracle's double-rounded addcmul differs from the fma: there, one fp32 ulp
    of the fma's result and only where Fraction arithmetic says OG's rounding is the wrong one.  -> number of such entries."""
    assert np.array_equal(a["hit"], b["hit"]), what
    for k in ("normal", "rgb", "alpha"):
        assert np.array_equal(a[k], b[k]), (what, k)
    diff = 0
    for k in ("xyz", "depth"):
        d = a[k] != b[k]
        diff += int(d.sum())
        if d.any():
            ulp = np.abs(a[k][d].astype(np.float64) - b[k][d]) / np.spacing(np.abs(a[k][d]))
            assert ulp.max() <= 1.0, (what, k, float(ulp.max()))
    return diff


@pytest.mark.parametrize("ms", ["sum", "cat"])
def test_restatement_equals_oracle(ms):
    case = _case(ms)
    lods = range(3) if ms == "sum" else [2]
    flips, runs, exits = 0, 0, set()
    for lod in lods:
        for steps in (0, 1, 32):
            for dist_max in (6.0, 2.6):
                kw = dict(num_steps=steps, step_size=0.8, min_dis=1e-3, lod_idx=lod, dist_max=dist_max)
                ref = OG.sdf_trace(case, return_debug=True, **kw)
                got = TR.sdf_trace(case, **kw)
                if got["nuggets"]:
                    assert got["iters"] == ref["iters"]
                flips += _compare(got, ref, (ms, lod, steps, dist_max))
                runs += 1
                exits.add(got["exit"])
                assert got["evals"] >= got["packs"] + 6 * int(got["hit"].sum())
    print(f"restatement vs oracle ({ms}): {runs} traces, {flips} xyz/depth entries where the double-rounded addcmul differs")
    assert {"march", "steps"} <= exits or ms == "cat"


def test_fma_differences_are_the_oracles_double_rounding():
    """Where the two restatements' points differ, the exact fma (Fraction) agrees with the new one."""
    case = _case("sum")
    rt = O.raytrace(case["spc"], case["origins"], case["dirs"], case["active_lods"][2])
    first = np.ones(rt["ridx"].shape[0], bool); first[1:] = rt["ridx"][1:] != rt["ridx"][:-1]
    r = rt["ridx"][first].astype(np.int64)
    o, d = case["origins"][r], case["dirs"][r]
    rng = np.random.default_rng(3)
    t = (rt["depth"][first][:, 0:1] + rng.uniform(0, 0.3, (r.shape[0], 1))).astype(np.float32)
    fast = TR.fma32(d, t, o)
    twice = (d.astype(np.float64) * t.astype(np.float64) + o.astype(np.float64)).astype(np.float32)
    diff = np.nonzero(fast != twice)
    for i, j in zip(*diff):
        assert fast[i, j] == _fma_exact([d[i, j]], [t[i, 0]], [o[i, j]])[0]
    print(f"addcmul: {len(diff[0])} of {fast.size} components differ between one and two roundings")


def test_restatement_reproduces_golden(golden_dir):
    """tests/golden/sdf_octree.npz: the reference's own PackedSDFTracer on an OctreeGrid NeuralSDF, to the tolerances the oracle
    restatement is held to."""
    g = np.load(os.path.join(golden_dir, "sdf_octree.npz"))
    spc = O.octree_to_spc(g["octree"])
    _, pyr, tr, _ = OG.make_trilinear_spc(spc)
    case = dict(spc=spc, trinkets=tr, pyramid_dual=pyr, active_lods=[3, 4, 5], feats=[g[f"sum_feat{i}"] for i in range(3)], multiscale="sum",
                W=[g["sum_W0"], g["sum_W1"]], b=[g["sum_b0"], g["sum_b1"]], origins=g["origins"], dirs=g["dirs"])
    out = TR.sdf_trace(case, num_steps=24, step_size=0.8, min_dis=1e-3, lod_idx=2, dist_max=6.0)
    assert np.array_equal(out["hit"], g["t_hit"]) and g["t_hit"].sum() > 20
    for k, tol in (("depth", 2e-5), ("xyz", 2e-6), ("normal", 2e-4), ("rgb", 1e-4), ("alpha", 0.0)):
        assert np.abs(out[k] - g["t_" + k]).max() <= tol, k
