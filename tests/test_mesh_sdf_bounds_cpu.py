"""CPU checks of the two culling lemmas wb_mesh_sdf rests on (stated above wb_msdf_query_kernel), on the restatement's per-pair
arithmetic (tests/mesh_sdf_reference.py), of the sentinel the GPU tests use as an unculled oracle, of the tree depths of the meshes
aimed at the hierarchy (tests/mesh_sdf_bvh_shapes.py), and of wb_mesh_sdf's triangle-count limit.

  distance: every pair distance d2 >= box_d2 (1 - 2^-20) - 2^-40 S^2, box_d2 measured to the triangle's leaf box (tri_box: fp32
            rounded outward, the whole space for NaN triangles and for triangles whose fp32 |n|^2 overflows), S = max|p_i| + the
            fp32 max |vertex coordinate| rounded up;
  stab:     every accepted Moller-Trumbore hit lies on a line that meets the leaf box grown by m = 2^-30 S + 2^-40 E^2 (S + E) 1e8,
            E the fp32 longest edge rounded up.
S and E are the triangle's own, never larger than the mesh-wide values the kernel uses, so each check is at least as strict."""
import numpy as np
import pytest
import torch

import mesh_sdf_bvh_shapes as B
import mesh_sdf_reference as R
import wisp_b200 as W
from oracle import mesh_shapes as MS

F32 = np.float32


def _up32(x):
    return R._f32_up(np.asarray(x, np.float64)).astype(np.float64)


def box_d2(lo, hi, P):
    """wb_msdf_query_kernel's box_dist2 for every pair of the points P [n, 3] with the boxes [T, 3] -> [n, T]."""
    lo, hi = lo.astype(np.float64)[None], hi.astype(np.float64)[None]
    with np.errstate(invalid="ignore"):
        g = np.fmax(np.fmax(lo - P[:, None], P[:, None] - hi), 0.0)
    return g[..., 0] * g[..., 0] + g[..., 1] * g[..., 1] + g[..., 2] * g[..., 2]


def box_line(lo, hi, P, d, m):
    """wb_msdf_query_kernel's box_line: does the line P + t d meet the box grown by m [n, T]?"""
    lo, hi = lo.astype(np.float64)[None], hi.astype(np.float64)[None]
    ok = np.ones(m.shape, bool)
    tmin, tmax = np.full(m.shape, -np.inf), np.full(m.shape, np.inf)
    with np.errstate(invalid="ignore", over="ignore"):
        for a in range(3):
            p = P[:, None, a]
            if d[a] == 0.0:
                ok &= ~((p < lo[..., a] - m) | (p > hi[..., a] + m))
            else:
                t1, t2 = (lo[..., a] - m - p) * (1.0 / d[a]), (hi[..., a] + m - p) * (1.0 / d[a])
                tmin, tmax = np.fmax(tmin, np.fmin(t1, t2)), np.fmin(tmax, np.fmax(t1, t2))
    return ok & (tmin <= tmax)


def scale_terms(tris, P):
    """Per pair: S = max|p_i| + R (R = the triangle's max |vertex coordinate|, fp32 rounded up) and E (its longest edge, fp32
    rounded up) -> S [n, T], E [T]."""
    v = tris.reshape(-1, 3, 3)
    R_ = _up32(np.abs(tris).max(1))
    e2 = np.max([((v[:, (k + 1) % 3] - v[:, k]) ** 2).sum(1) for k in range(3)], axis=0)
    return np.abs(P).max(1)[:, None] + R_[None], _up32(np.sqrt(e2))


def distance_violations(tris, P, box=R.tri_box):
    d2 = R.pair_d2(P, tris).astype(np.float64)
    lo, hi = box(tris)
    S, _ = scale_terms(tris, P)
    bound = box_d2(lo, hi, P) * (1.0 - 2.0 ** -20) - 2.0 ** -40 * S * S
    return ~np.isnan(d2) & (d2 < bound)


def stab_violations(tris, P, grow=True):
    """Accepted hits whose line misses the leaf box grown by m (by nothing for grow=False) [n, T], and the number of hits."""
    lo, hi = R.tri_box(tris)
    S, E = scale_terms(tris, P)
    m = 2.0 ** -30 * S + 2.0 ** -40 * E * E * (S + E) * 1e8 if grow else np.zeros(S.shape)
    bad, hits = np.zeros(S.shape, bool), 0
    for i, d in enumerate(R.STAB_DIRS):
        hit, _ = R.stab_hits(P, tris, i)
        hits += int(hit.sum())
        bad |= hit & ~box_line(lo, hi, P, d, m)
    return bad, hits


def families(rng, T=48):
    """(name, tris [T, 9]) at scales 1e-6 .. 1e10: slivers (relative normal 1e-17 .. 1e-6), tiny triangles (fp32-subnormal |n|^2),
    huge triangles, axis-aligned triangles and vertices half an fp32 ulp off an fp32 value."""
    for scale in (1e-6, 1e-2, 1.0, 1e3, 1e6, 1e10):
        c = rng.uniform(-1, 1, (T, 3)) * scale
        L = scale * 10.0 ** rng.uniform(-3, 0, (T, 1))
        a, b = rng.normal(size=(T, 3)), rng.normal(size=(T, 3))
        a /= np.linalg.norm(a, axis=1, keepdims=True)
        b -= (a * b).sum(1, keepdims=True) * a
        b /= np.linalg.norm(b, axis=1, keepdims=True)
        rel = 10.0 ** rng.uniform(-17, -6, (T, 1))
        t = rng.uniform(-0.5, 1.5, (T, 1))
        yield f"sliver@{scale:g}", np.concatenate([c, c + L * a, c + L * (t * a + rel * b)], 1)
        e = 10.0 ** rng.uniform(-11.5, -9.2, (T, 1))                 # |n|^2 ~ e^4: from fp32-subnormal to normal
        yield f"tiny@{scale:g}", np.concatenate([c, c + e * a, c + e * b * rng.uniform(0.3, 3, (T, 1))], 1)
        yield f"huge@{scale:g}", np.concatenate([c, c + 30 * L * a, c + 30 * L * b], 1)
        ax = np.zeros((T, 9))
        k = rng.integers(0, 3, T)
        for j in range(T):
            u, w = (k[j] + 1) % 3, (k[j] + 2) % 3
            ax[j, 0:3] = c[j]
            ax[j, 3:6] = c[j]; ax[j, 3 + u] += L[j, 0]
            ax[j, 6:9] = c[j]; ax[j, 6 + w] += L[j, 0] * rng.uniform(0.1, 2)
        yield f"axis@{scale:g}", ax
        v = np.concatenate([c, c + L * a, c + L * b], 1).astype(F32)
        half = np.spacing(np.abs(v)).astype(np.float64) * 0.5 * rng.choice([-1.0, 0.0, 1.0], v.shape)
        yield f"fp32-half-ulp@{scale:g}", v.astype(np.float64) + half


def test_distance_lemma():
    rng = np.random.default_rng(0)
    pairs = 0
    for name, tris in families(rng):
        P = B.points_near(tris, rng)
        bad = distance_violations(tris, P)
        pairs += bad.size
        assert not bad.any(), (name, int(bad.sum()), np.argwhere(bad)[:3])
    assert pairs > 5 * 10 ** 5


def test_stab_lemma():
    """Points on the 13 stab lines through points on (and just off) each triangle: every accepted hit's line meets the grown box."""
    rng = np.random.default_rng(1)
    hits = 0
    for name, tris in families(rng, T=24):
        v = tris.reshape(-1, 3, 3)
        size = np.abs(v - v.mean(1, keepdims=True)).max((1, 2))[:, None]
        pts = []
        for d in R.STAB_DIRS:
            bary = rng.dirichlet((1.0, 1.0, 1.0), v.shape[0]) * rng.uniform(0.999, 1.001, (v.shape[0], 1))
            pts.append((v * bary[:, :, None]).sum(1) + d * size * rng.uniform(-3, 3, (v.shape[0], 1)))
        bad, n = stab_violations(tris, np.concatenate(pts))
        hits += n
        assert not bad.any(), (name, int(bad.sum()))
    assert hits > 2000, hits


def grazing(rng, scale, far, T=48):
    """fp32-exact triangles with v0 alone on the low x face of the box, and lines along the 4 stab directions with d_x = 0 through
    v0 moved one double ulp outside that face, offset along the line by up to `far` times the scale.  The lines miss the box; the
    triangles' planes meet them within ~1e-16 of v0, where the rounding of u and w can accept the hit."""
    v = (rng.uniform(-1, 1, (T, 3, 3)) * scale).astype(F32).astype(np.float64)
    v[:, 1:, 0] = (v[:, :1, 0] + np.abs(v[:, 1:, 0] - v[:, :1, 0]) + 0.05 * scale).astype(F32)
    pts = []
    for k in (1, 2, 3, 6):
        on = v[:, 0].copy()
        on[:, 0] = np.nextafter(on[:, 0], -np.inf)
        pts.append(on + R.STAB_DIRS[k] * scale * far * rng.uniform(-1, 1, (T, 1)))
    return v.reshape(-1, 9), np.concatenate(pts)


def test_stab_lemma_grazing_lines():
    """Hits accepted only through rounding, on lines that miss the ungrown leaf box: the margin m is what keeps them, and it does."""
    rng = np.random.default_rng(4)
    missed = 0
    for scale in (1e-6, 1e-2, 1.0, 1e3, 1e6):
        for far in (1.0, 1e2, 1e4):
            tris, P = grazing(rng, scale, far)
            bad, _ = stab_violations(tris, P)
            assert not bad.any(), (scale, far, int(bad.sum()))
            missed += int(stab_violations(tris, P, grow=False)[0].sum())
    assert missed > 100, missed


def test_overflowing_normal_is_exempt():
    """A triangle with edges of 5e9 has |n|^2 = 6.25e38, inf in fp32: idot2(n) = 0 and its face distance is 0 at the point (1, 1, 0),
    1e4 below it.  The outward-rounded box alone violates the distance lemma there (box_d2 = 1e8 against a pair distance of 0,
    with a 'decoy' at distance 1 culling it); tri_box gives that triangle the whole space and keeps the decoy's box."""
    huge = [0.0, 0.0, 1e4, 5e9, 0.0, 1e4, 0.0, 5e9, 1e4]
    decoy = [-2.0, -2.0, -1.0, 4.0, -2.0, -1.0, -2.0, 4.0, -1.0]
    tris, P = np.array([huge, decoy]), np.array([[1.0, 1.0, 0.0]])
    assert R.pair_d2(P, tris).tolist() == [[0.0, 1.0]]
    assert distance_violations(tris, P, box=R.outward_box).tolist() == [[True, False]]
    assert not distance_violations(tris, P).any()
    lo, hi = R.tri_box(tris)
    assert np.all(lo[0] == -np.inf) and np.all(hi[0] == np.inf)
    assert np.array_equal(lo[1], F32([-2, -2, -1])) and np.array_equal(hi[1], F32([4, 4, -1]))
    r = R.mesh_sdf(tris, P)
    assert r["sdf"][0] == 0.0 and r["sign_ok"][0]
    # just below the overflow the box stays finite and the lemma holds
    small = np.array(huge) * np.array([1, 1, 1, 0.8, 1, 1, 1, 0.8, 1])
    assert np.isfinite(R.tri_box(small)[0]).all() and not distance_violations(small[None], P).any()
    # the exemption's FMA margin: every triangle whose fp32 |n|^2 overflows is exempt, at the threshold too
    edge = np.sqrt(np.sqrt(float.fromhex("0x1.ffffffp127"))) * (1.0 + 2.0 ** -44 * np.arange(-64, 65))
    t = np.zeros((edge.size, 9))
    t[:, 3], t[:, 7] = edge, edge
    with np.errstate(over="ignore"):
        over = R._idot2(np.stack([0 * edge, 0 * edge, edge * edge], 1)) == 0.0        # |n| = edge^2
    assert over.any() and (~over).any()
    assert np.all(np.isinf(R.tri_box(t)[0][over]))


def test_subnormal_normals_keep_the_lemma():
    """Tiny triangles whose fp32 |n|^2 is subnormal (down to where the reciprocal overflows) next to a decoy, with points on, above
    and beside them: no violation, and below ~2.9e-39 the face distance is never short (inf, or NaN and ignored)."""
    rng = np.random.default_rng(2)
    e = 10.0 ** np.linspace(-11.6, -9.4, 200)[:, None]
    c = rng.uniform(-0.3, 0.3, (200, 3))
    tris = np.concatenate([c, c + e * [1.0, 0.0, 0.0], c + e * [0.0, 1.0, 0.0]], 1)
    n2 = (e[:, 0] ** 2) ** 2
    assert (n2 < 1.2e-38).sum() > 50 and (n2 < 2.9e-39).sum() > 20
    tris = np.concatenate([tris, [[-2.0, -2.0, -1.0, 4.0, -2.0, -1.0, -2.0, 4.0, -1.0]]])
    P = B.points_near(tris[:-1], rng)
    assert not distance_violations(tris, P).any()


def test_sentinel_is_inert_under_the_rule():
    """The sentinel triangle changes no sdf bit and no inside flag of the restatement (its tol does grow with the coordinates, so
    it is never compared)."""
    rng = np.random.default_rng(3)
    for V, F in (MS.cube(), MS.torus(), MS.open_mesh(), B.flat_grid(6)):
        P = np.concatenate([MS.feature_points(V, F, 60, rng), MS.near_points(V, F, 300, rng), MS.uniform_points(200, rng),
                            V[F[rng.integers(0, F.shape[0], 40), 0]] + R.STAB_DIRS[rng.integers(0, 13, 40)] * rng.uniform(-1, 1, (40, 1))])
        a = R.mesh_sdf(V[F].reshape(-1, 9), P)
        V2, F2 = B.with_sentinel(V, F)
        b = R.mesh_sdf(V2[F2].reshape(-1, 9), P)
        assert np.array_equal(a["sdf"].view(np.int64), b["sdf"].view(np.int64)) and np.array_equal(a["inside"], b["inside"])


def test_tree_depths():
    """The caterpillar's deepest leaf is at least 40 levels down; every mesh the GPU tests build stays within the query stack."""
    cat = B.leaf_depths(B.caterpillar())
    assert cat.max() >= 40, cat.max()
    keys = np.sort(B.morton_keys(B.caterpillar())) >> np.uint64(32)
    assert {int(k).bit_length() for k in keys} == set(range(31))         # codes 0, 2^0 .. 2^29 and 2^30 - 1
    assert B.leaf_depths(B.fan(1000)).max() == 10                       # equal codes: split on the index bits
    V, F = B.flat_grid(16)
    assert np.all((B.morton_keys(V[F].reshape(-1, 9)) >> np.uint64(32)) & np.uint64(0x09249249) == 0)     # z collapsed
    for tris in (B.caterpillar(), B.fan(1 << 17), V[F].reshape(-1, 9)):
        assert B.leaf_depths(tris).max() <= 61
        V2 = np.concatenate([tris.reshape(-1, 3), B.SENTINEL[None]])
        F2 = np.concatenate([np.arange(tris.shape[0] * 3).reshape(-1, 3), [[V2.shape[0] - 1] * 3]])
        assert B.leaf_depths(V2[F2].reshape(-1, 9)).max() <= 61


def test_triangle_count_limit():
    """Node ids and the box offsets 2 node are int, the largest 2 (2T - 2): wb_mesh_sdf and its workspace query refuse T > 2^29."""
    L = W._cabi.lib()
    for T in (2 ** 29 + 1, 2 ** 30, 2 ** 31 - 1):
        assert L.wb_mesh_sdf_workspace_bytes(T) < 0
        assert "num_triangles" in L.wb_last_error().decode()
    with pytest.raises(W.WispB200Error, match="num_triangles"):
        L.wb_mesh_sdf(None, 2 ** 29 + 1, None, 1, None, 0, None, None)
    if torch.cuda.is_available():
        assert L.wb_mesh_sdf_workspace_bytes(2 ** 29) > 2 ** 29 * 9 * 8
