"""wb_mesh_sdf's culling checked bit for bit against the same kernel with culling switched off.

Appending the sentinel triangle (tests/mesh_sdf_bvh_shapes.py) changes nothing under the rule -- its normal is exactly zero and its
det is 0 in every stab direction -- but its |coordinate| of 1e30 grows the distance slack 2^-40 S^2 to ~9e47 and the stab margin to
~9e20, so neither search can skip a triangle, and it collapses the other Morton codes into one, so the tree is a different one.
The fp32 minimum (fminf, NaN ignored) and the stab flags (an OR per direction) do not depend on the visiting order, so
compute_sdf(mesh) must equal compute_sdf(mesh + sentinel) in every bit, magnitude and sign, on every point -- including points the
restatement calls ambiguous, since both runs use the kernel's own pair arithmetic.  A seeded subsample of each run is also checked
against the numpy restatement (tests/mesh_sdf_reference.py), on the mesh without the sentinel."""
import os

import numpy as np
import pytest
import torch

import mesh_sdf_bvh_shapes as B
import mesh_sdf_reference as R
from oracle import mesh_shapes as MS
from test_gpu_mesh_sdf import CASES, against_restatement, sdf

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RESTATE = 5 * 10 ** 5      # restatement pairs per check
UNCULLED = 10 ** 10        # points x triangles per unculled run, at most


@pytest.fixture(scope="module")
def W():
    import wisp_b200
    torch.cuda.set_device(0)
    return wisp_b200


def check(W, V, F, P, seed=0, restate=RESTATE):
    """The culled run equals the unculled one bit for bit on every point; a seeded subsample lies inside the restatement's bound."""
    V, F, P = np.asarray(V, np.float64), np.asarray(F, np.int64), np.asarray(P, np.float64)
    assert P.shape[0] * (F.shape[0] + 1) <= UNCULLED
    got = sdf(W, V, F, P)
    full = sdf(W, *B.with_sentinel(V, F), P)
    diff = np.nonzero(got.view(np.int64) != full.view(np.int64))[0]
    assert diff.size == 0, (f"{diff.size} of {P.shape[0]} points differ from the unculled run", P[diff[:4]], got[diff[:4]],
                            full[diff[:4]])
    if restate:
        k = max(1, min(P.shape[0], restate // max(F.shape[0], 1)))
        idx = np.sort(np.random.default_rng(seed).choice(P.shape[0], k, replace=False))
        against_restatement(got[idx], V, F, P[idx])
    return got


def mesh_of(tris):
    return tris.reshape(-1, 3), np.arange(tris.shape[0] * 3).reshape(-1, 3)


@pytest.mark.parametrize("case", CASES + ["torus_2e5"])
def test_golden_meshes(W, case):
    """The golden's five meshes with tens of thousands of points each, and the 2*10^5-triangle torus at 5*10^4 points (10^10
    pairs unculled)."""
    rng = np.random.default_rng(10)
    if case == "torus_2e5":
        V, F = MS.torus(316, 316, 0.55, 0.25)
        V = V + np.random.default_rng(6).normal(scale=2e-4, size=V.shape)
        P = np.concatenate([MS.dataset_points(V, F, 45000, rng), MS.feature_points(V, F, 1500, rng)])
    else:
        g = np.load(os.path.join(ROOT, "tests", "golden", "ref_mesh_sdf.npz"))
        V, F, Pg = g[f"{case}_V"], g[f"{case}_F"].astype(np.int64), g[f"{case}_points"]
        P = np.concatenate([Pg, MS.dataset_points(V, F, 30000, rng), MS.feature_points(V, F, 3000, rng)])
    assert P.shape[0] >= 30000
    check(W, V, F, P)


SIZES = [2, 3, 4, 5, 31, 32, 33, 127, 128, 129] + [2 ** k + s for k in (8, 10, 12, 14, 16) for s in (-1, 1)]


@pytest.fixture(scope="module")
def big_sphere():
    return MS.noisy_sphere(6, seed=5)          # 81 920 triangles


@pytest.mark.parametrize("T", SIZES)
def test_tree_sizes(W, big_sphere, T):
    """Seeded subsets of T triangles of a noisy sphere: every tree size around the powers of two."""
    V, F = big_sphere
    rng = np.random.default_rng(T)
    F = F[np.sort(rng.choice(F.shape[0], T, replace=False))]
    assert B.leaf_depths(V[F].reshape(-1, 9)).max() <= 61
    n = min(20000, UNCULLED // 10 // (T + 1))
    P = np.concatenate([MS.dataset_points(V, F, n - 3 * min(T, 300), rng), MS.feature_points(V, F, min(T, 300), rng)])
    check(W, V, F, P, seed=T)


def test_fan_of_equal_codes(W):
    """4097 triangles sharing one centroid: every Morton code is equal and the tree splits on index bits alone."""
    tris = B.fan(4097)
    assert np.unique(B.morton_keys(tris) >> np.uint64(32)).size == 1
    V, F = mesh_of(tris)
    rng = np.random.default_rng(11)
    P = np.concatenate([rng.uniform(-1.5, 2.0, (20000, 3)), MS.feature_points(V, F, 1000, rng), np.array([[0.25, -0.125, 0.5]])])
    check(W, V, F, P)


def test_caterpillar(W):
    """Centroids stepping through the 30 Morton bits one at a time, with 1024 triangles on the deepest code: a tree of depth >= 40."""
    tris = B.caterpillar()
    depth = B.leaf_depths(tris).max()
    assert 40 <= depth <= 61, depth
    V, F = mesh_of(tris)
    rng = np.random.default_rng(12)
    cents = tris.reshape(-1, 3, 3).mean(1)
    P = np.concatenate([cents[rng.integers(0, cents.shape[0], 20000)] + rng.normal(size=(20000, 3)) * 10.0 ** rng.uniform(-4, 1, (20000, 1)),
                        rng.uniform(-2, 1025, (5000, 3)), MS.feature_points(V, F, 500, rng)])
    check(W, V, F, P)


@pytest.mark.parametrize("place", ["scale1e-6", "scale1", "scale1e3", "scale1e9", "translate1e6", "half_ulp"])
def test_scale_and_placement(W, place):
    """One mesh scaled by 1e-6 .. 1e9, translated by 1e6 (where the 2^-40 S^2 slack dominates), and with every vertex half an fp32
    ulp off an fp32 value (the boxes' outward rounding matters), with points one fp32 ulp outside the boxes' faces."""
    V, F = MS.noisy_sphere(3, seed=2)
    rng = np.random.default_rng(13)
    P = np.concatenate([MS.dataset_points(V, F, 15000, rng), MS.feature_points(V, F, 1000, rng)])
    if place.startswith("scale"):
        s = float(place[5:])
        V, P = V * s, P * s
    elif place == "translate1e6":
        V, P = V + 1e6, P + 1e6
    else:
        V32 = V.astype(np.float32)
        V = V32.astype(np.float64) + 0.5 * np.spacing(np.abs(V32)).astype(np.float64) * rng.choice([-1.0, 1.0], V.shape)
        P = np.concatenate([P, B.points_near(V[F].reshape(-1, 9), rng, 12)])
    check(W, V, F, P)


def test_ties_and_grazing(W):
    """A coplanar grid of equal triangles with points above its vertices, edge midpoints and centres (equal distances in many
    subtrees); points exactly on the vertices, edges and faces of closed meshes; points on the 13 stab lines through vertices and
    edge midpoints."""
    rng = np.random.default_rng(14)
    V, F = B.flat_grid(32)                          # z extent 0: the Morton z coordinate collapses
    T = V[F]
    sites = np.concatenate([V, (T[:, 0] + T[:, 1]) / 2, (T[:, 1] + T[:, 2]) / 2, (T[:, 2] + T[:, 0]) / 2, T.mean(1)])
    P = np.concatenate([sites + [0.0, 0.0, h] for h in (0.0, 1e-3, -1e-3, 0.25, 2.0)])
    check(W, V, F, P)
    for V, F in (MS.icosphere(3, 0.6), MS.cube(), MS.torus()):
        T = V[F]
        sites = np.concatenate([V, (T[:, 0] + T[:, 1]) / 2, (T[:, 1] + T[:, 2]) / 2, (T[:, 2] + T[:, 0]) / 2])
        on_lines = (sites[rng.integers(0, sites.shape[0], 6000)] + R.STAB_DIRS[rng.integers(0, 13, 6000)] *
                    rng.choice([-1.7, -0.3, 0.3, 1.7], (6000, 1)))
        P = np.concatenate([MS.feature_points(V, F, 1500, rng), sites, on_lines])
        check(W, V, F, P)


HUGE = np.array([[0.0, 0.0, 1e4], [5e9, 0.0, 1e4], [0.0, 5e9, 1e4]])
DECOY = np.array([[-2.0, -2.0, -1.0], [4.0, -2.0, -1.0], [-2.0, 4.0, -1.0]])


def test_overflowing_normal(W):
    """A triangle with edges of 5e9 has fp32 |n|^2 = inf and idot2(n) = 0: under the rule its face distance is 0 at (1, 1, 0), 1e4
    below it, so the point's value is 0 even with the decoy 1 away.  Culling that triangle once the decoy sets best = 1 returned 1."""
    V, F = np.concatenate([HUGE, DECOY]), np.array([[0, 1, 2], [3, 4, 5]])
    P = np.array([[1.0, 1.0, 0.0], [0.5, 0.5, -0.5], [3.0, -1.0, 2.0], [1e3, 2e3, 0.0], [-5.0, -5.0, 0.0], [1.0, 1.0, -30.0]])
    got = check(W, V, F, P)
    assert abs(got[0]) == 0.0, f"compute_sdf at (1, 1, 0) = {got[0]!r}; the rule gives 0 (the huge triangle's idot2(n) is 0)"
    # a unit mesh with one far triangle of 5e9 edges above it
    Vs, Fs = MS.icosphere(3, 0.6)
    V, F = np.concatenate([Vs, HUGE]), np.concatenate([Fs, [[Vs.shape[0], Vs.shape[0] + 1, Vs.shape[0] + 2]]])
    rng = np.random.default_rng(15)
    P = np.concatenate([MS.dataset_points(Vs, Fs, 10000, rng), MS.feature_points(Vs, Fs, 500, rng), rng.uniform(-5, 5, (2000, 3))])
    got = check(W, V, F, P)
    under = (P[:, 0] > 1e-3) & (P[:, 1] > 1e-3)          # the projection falls inside the far triangle
    assert under.sum() > 2000 and np.all(got[under] == 0.0)
    # tiny triangles whose fp32 |n|^2 is subnormal or underflows, beside a decoy, every point against the restatement
    e = 10.0 ** np.linspace(-11.6, -9.4, 300)[:, None]
    c = rng.uniform(-0.3, 0.3, (300, 3))
    tris = np.concatenate([np.concatenate([c, c + e * [1.0, 0.0, 0.0], c + e * [0.0, 1.0, 0.0]], 1), DECOY.reshape(1, 9)])
    V, F = mesh_of(tris)
    P = np.concatenate([B.points_near(tris[:-1], rng, 12), rng.uniform(-1, 1, (3000, 3))])
    check(W, V, F, P, restate=P.shape[0] * F.shape[0])


@pytest.mark.parametrize("N", [1, 127, 128, 129])
def test_point_counts(W, N):
    """N around one block of kMsdfThreads = 128 points."""
    V, F = MS.torus()
    P = MS.dataset_points(V, F, N, np.random.default_rng(N)) if N >= 5 else MS.near_points(V, F, N, np.random.default_rng(N))
    check(W, V, F, P)


def test_infinite_and_huge_points(W):
    """Points with +-inf coordinates and with 1e300: the rule gives +inf (every distance overflows; no stab has a t >= 0 hit)."""
    V, F = MS.torus()
    rng = np.random.default_rng(16)
    P = MS.near_points(V, F, 64, rng)
    P[0:8, 0], P[8:16, 1], P[16:24, 2] = np.inf, -np.inf, 1e300
    P[24:32] = [-1e300, 1e300, np.inf]
    P[32:36] = np.inf
    got = check(W, V, F, P)
    assert np.all(got[:36] == np.inf), got[:36]
    ref = R.mesh_sdf(V[F].reshape(-1, 9), P[:36])
    assert np.all(ref["sdf"] == np.inf)
