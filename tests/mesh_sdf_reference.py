"""A vectorised numpy restatement of wisp.ops.mesh.compute_sdf's rule (wisp/csrc/external/mesh2sdf_kernel.cu:334-584, 844-903),
brute force over every point-triangle pair, with the reference's fp32 roundings written out as np.float32 casts:
  - per pair, in float64: p_k = p - v_k, e10 = v1 - v0, e21 = v2 - v1, e02 = v0 - v2, n = e10 x e02, c_k = e_k x n;
  - idot2(a) = fp32(1) / fp32(|a|^2) (__frcp_rn of the fp32-rounded squared length), widened;
  - s_k = copysignf(1, fp32(c_k . p_k)); the face distance (n . p0)^2 idot2(n) when s1 + s2 + s3 >= 2, else the fminf of the three
    edge distances |e_k x - p_k|^2 with x = fmaxf(0, fminf(fp32(e_k . p_k idot2(e_k)), 1)); negative -> 0; a zero normal adds nothing;
  - the point's fp32 minimum over pairs (fminf: NaN ignored), sqrtf of it, negated when every one of the 13 stab directions (the
    fp32 literals of :368-380) has a Moller-Trumbore hit with t >= 0 and one with t < 0; |det| < 1e-8 skipped, inv_det = 1 / det.
Beside the value it reports, per point, whether the sign and the face/edge branch of the minimising pair are unambiguous: every
predicate they rest on (det against +-1e-8, u, v, u + v and t against their bounds, the three c_k . p_k against 0, the normal
against 0) lies farther from its threshold than a float64 error bound on that value (generous: 64 ulps of the products' magnitudes,
so FMA contraction or another summation order cannot cross it).  `tol` is the distance bound that follows: 1 fp32 ulp, plus, when
the minimum comes from an edge branch or an ambiguous one, the displacement of one fp32 ulp of the edge parameter (2^-24 |edge|), plus
the absolute float64 rounding of the pair arithmetic (256 ulps of the coordinates' magnitude, which only matters for points on the
surface), plus, when a pair with a nonzero normal can take its other face/edge branch under another rounding (some c_k . p_k
within its bound of 0 and none surely negative) and that branch would give less than the minimum, the difference; it is
inf when a triangle whose normal is zero up to rounding would set the minimum if it took part.
pair_d2, stab_hits and tri_box expose the per-pair distance, the per-pair stab test and wb_mesh_sdf's leaf box, for checks of the
kernel's culling bounds.
"""
from __future__ import annotations

import numpy as np

STAB_DIRS = np.array([[1.0, 0.0, 0.0], [0.0, 1.0, 0.0], [0.0, 0.0, 1.0],
                      [0.0, 0.707106781, 0.707106781], [0.707106781, 0.0, 0.707106781], [0.707106781, 0.707106781, 0.0],
                      [0.0, 0.707106781, -0.707106781], [0.707106781, 0.0, -0.707106781], [0.707106781, -0.707106781, 0.0],
                      [0.577350269, 0.577350269, 0.577350269], [-0.577350269, 0.577350269, 0.577350269],
                      [0.577350269, -0.577350269, 0.577350269], [0.577350269, 0.577350269, -0.577350269]],
                     np.float32).astype(np.float64)
EPS = 2.0 ** -53
K = 64 * EPS            # error bound factor on |products|
F32 = np.float32
N2_EXEMPT = float.fromhex("0x1.ffffffp127") * (1.0 - 2.0 ** -40)     # wb_mesh_sdf.cu's kMsdfN2Exempt


def _dot(a, b):
    return a[..., 0] * b[..., 0] + a[..., 1] * b[..., 1] + a[..., 2] * b[..., 2]


def _cross(a, b):
    return np.stack([a[..., 1] * b[..., 2] - a[..., 2] * b[..., 1], a[..., 2] * b[..., 0] - a[..., 0] * b[..., 2],
                     a[..., 0] * b[..., 1] - a[..., 1] * b[..., 0]], -1)


def _norm(a):
    return np.sqrt(_dot(a, a))


def _idot2(a):
    with np.errstate(divide="ignore", over="ignore"):
        return (F32(1.0) / _dot(a, a).astype(F32)).astype(np.float64)


def _sign32(x):
    with np.errstate(over="ignore", invalid="ignore"):
        return np.copysign(F32(1.0), x.astype(F32)).astype(np.float64)


def _clamp32(x):
    with np.errstate(over="ignore", invalid="ignore"):
        return np.fmax(F32(0.0), np.fmin(x.astype(F32), F32(1.0))).astype(np.float64)


def _dist2(a, x, b):
    t = a * x[..., None] - b
    return _dot(t, t)


def _pairs(P, tris):
    """The distance half of the rule for all pairs of the points P [n, 3] with the triangles [T, 9]: the edges, the normal, the
    p_k, the three c_k . p_k, the branch sum s, the edge and face distances and the fp32 d2 [n, T] (NaN for a zero normal)."""
    v0, v1, v2 = tris[:, 0:3], tris[:, 3:6], tris[:, 6:9]
    e10, e21, e02 = v1 - v0, v2 - v1, v0 - v2
    nor = _cross(e10, e02)
    c = [_cross(e10, nor), _cross(e21, nor), _cross(e02, nor)]
    es = [e10, e21, e02]
    p = [P[:, None, :] - v[None] for v in (v0, v1, v2)]
    with np.errstate(invalid="ignore", over="ignore"):
        dots = [_dot(c[k][None], p[k]) for k in range(3)]
        s = _sign32(dots[0]) + _sign32(dots[1]) + _sign32(dots[2])
        ed = [_dist2(es[k][None], _clamp32(_dot(es[k][None], p[k]) * _idot2(es[k])[None]), p[k]).astype(F32) for k in range(3)]
        edge = np.fmin(ed[0], np.fmin(ed[1], ed[2])).astype(np.float64)
        dn = _dot(nor[None], p[0])
        face = dn * dn * _idot2(nor)[None]
        d2 = np.where(s < 2.0, edge, face)
        d2 = np.where(d2 < 0.0, 0.0, d2)
        valid = np.any(nor != 0.0, axis=1)
        d2 = np.where(valid[None], d2, np.nan).astype(F32)           # a zero normal: ignored by fminf
    return es, nor, p, dots, s, edge, face, d2


def _stab(p0, e10, e20, qv, d):
    """Moller-Trumbore along direction d for the pairs p0 [n, T, 3] x (e10, e20) [T, 3]: det [T], whether it is tested, and u, w, t
    [n, T]."""
    pv = _cross(np.broadcast_to(d, e20.shape), e20)
    det = _dot(e10, pv)
    tested = ~((det > -1e-8) & (det < 1e-8))
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        inv_det = 1.0 / det
        u = _dot(p0, pv[None]) * inv_det[None]
        w = _dot(np.broadcast_to(d, qv.shape), qv) * inv_det[None]
        t = _dot(e20[None], qv) * inv_det[None]
    return det, tested, u, w, t


def pair_d2(P, tris):
    """The rule's fp32 squared distance of every pair of the points P [n, 3] with the triangles [T, 9] -> [n, T]; NaN where the
    triangle's normal is exactly zero (the pair adds nothing to the fminf)."""
    return _pairs(np.asarray(P, np.float64).reshape(-1, 3), np.asarray(tris, np.float64).reshape(-1, 9))[-1]


def stab_hits(P, tris, i):
    """The rule's Moller-Trumbore test along stab direction i for every pair -> (hit [n, T]: tested and inside the triangle, t)."""
    P, tris = np.asarray(P, np.float64).reshape(-1, 3), np.asarray(tris, np.float64).reshape(-1, 9)
    e10, e20 = tris[:, 3:6] - tris[:, 0:3], tris[:, 6:9] - tris[:, 0:3]
    p0 = P[:, None, :] - tris[None, :, 0:3]
    _, tested, u, w, t = _stab(p0, e10, e20, _cross(p0, e10[None]), STAB_DIRS[i])
    with np.errstate(invalid="ignore"):
        return tested[None] & ~((u < 0.0) | (u > 1.0)) & ~((w < 0.0) | (u + w > 1.0)), t


def _f32_down(x):
    with np.errstate(over="ignore"):
        f = x.astype(F32)
    return np.where(f.astype(np.float64) > x, np.nextafter(f, F32(-np.inf)), f)


def _f32_up(x):
    with np.errstate(over="ignore"):
        f = x.astype(F32)
    return np.where(f.astype(np.float64) < x, np.nextafter(f, F32(np.inf)), f)


def outward_box(tris):
    """Each triangle's [T, 9] bounding box rounded outward to fp32 -> (lo, hi) fp32 [T, 3]."""
    tris = np.asarray(tris, np.float64).reshape(-1, 3, 3)
    return _f32_down(tris.min(1)), _f32_up(tris.max(1))


def tri_box(tris):
    """wb_mesh_sdf's leaf box: the outward-rounded box, or the whole space for a triangle with a NaN coordinate (its stab hits are
    all negative) or one whose fp32 |n|^2 overflows (idot2(n) = 0: the face distance is 0 wherever the projection falls inside),
    with the kernel's margin for another FMA contraction of n."""
    tris = np.asarray(tris, np.float64).reshape(-1, 9)
    lo, hi = outward_box(tris)
    e10, e02 = tris[:, 3:6] - tris[:, 0:3], tris[:, 0:3] - tris[:, 6:9]
    nor = _cross(e10, e02)
    with np.errstate(over="ignore", invalid="ignore"):          # the overflow test with its FMA margin, as the kernel writes it
        whole = np.isnan(tris).any(1) | ~(_dot(nor, nor) + 2.0 ** -40 * _dot(e10, e10) * _dot(e02, e02) < N2_EXEMPT)
    lo[whole], hi[whole] = -np.inf, np.inf
    return lo, hi


def _chunk(P, tris):
    """All pairs of the points P [n, 3] with the triangles [T, 9]."""
    n = P.shape[0]
    es, nor, p, dots, s, edge, face, d2 = _pairs(P, tris)
    e10, e21, e02 = es
    e20 = -e02
    d2_for_min = np.where(np.isnan(d2), np.inf, d2)
    best = d2_for_min.min(axis=1)
    # a nearly zero normal may be exactly zero under another rounding (FMA): such a pair may or may not take part
    nor_amb = _norm(nor) <= K * _norm(e10) * _norm(e02)
    with np.errstate(invalid="ignore", over="ignore"):
        d2_amb = np.where(nor_amb[None], np.where(s < 2.0, edge, face), np.inf).astype(F32)
    dist_ok = ~(np.where(np.isnan(d2_amb), np.inf, d2_amb).min(axis=1) < best)
    arg = d2_for_min.argmin(axis=1)
    rows = np.arange(n)
    # the minimising pair's branch: unambiguous when each c_k . p_k and the normal clear their error bounds
    nn = _norm(nor)
    branch_ok = np.ones(n, bool)
    emax = np.maximum(np.maximum(_norm(e10), _norm(e21)), _norm(e02))
    for k in range(3):
        bound = 2 * K * _norm(es[k])[arg] * _norm(e10)[arg] * _norm(e02)[arg] * _norm(p[k][rows, arg])
        branch_ok &= np.abs(dots[k][rows, arg]) > bound
    branch_ok &= nn[arg] > K * _norm(e10)[arg] * _norm(e02)[arg]
    is_edge = s[rows, arg] < 2.0
    edge_term = np.where(is_edge | ~branch_ok, emax[arg] * 2.0 ** -24, 0.0)
    edge_term = np.where(np.isfinite(best), edge_term, 0.0)
    # the float64 rounding of the pair's own arithmetic, absolute: it dominates for points on the surface (distances ~1e-17)
    scale = np.abs(P).max(1) + np.abs(tris).max()
    edge_term = edge_term + K * scale * 4
    # a pair with a nonzero normal whose branch can flip under another rounding may take its other branch; that only matters where
    # the other value undercuts the minimum by more than the terms above, e.g. a triangle whose fp32 |n|^2 underflows (face
    # distance inf or NaN) at a point on one of its edge lines (c_k . p_k = 0 here, tiny and negative under FMA: an edge distance
    # instead).  The face branch needs all three signs +1, so the branch can flip when some sign is ambiguous and none is surely
    # -1.  A zero normal is left out: the kernel drops that pair before either branch.
    amb_any, neg_sure = np.zeros(d2.shape, bool), np.zeros(d2.shape, bool)
    for k in range(3):
        amb_k = np.abs(dots[k]) <= 2 * K * (_norm(es[k]) * _norm(e10) * _norm(e02))[None] * _norm(p[k])
        amb_any |= amb_k
        neg_sure |= ~amb_k & (_sign32(dots[k]) < 0.0)
    amb = amb_any & ~neg_sure & np.any(nor != 0.0, axis=1)[None]
    with np.errstate(invalid="ignore", over="ignore"):
        other = np.where(amb, np.where(s < 2.0, face, edge), np.inf).astype(F32)
    other = np.where(np.isnan(other), np.inf, other).min(axis=1)
    with np.errstate(invalid="ignore"):
        undercut = np.sqrt(best.astype(np.float64)) - np.sqrt(np.maximum(other, F32(0.0)).astype(np.float64))
    edge_term = edge_term + np.where(other < best, undercut, 0.0)
    edge_term = np.where(dist_ok, edge_term, np.inf)

    # the stab: per direction, whether a positive / negative hit is certain or possible under the error bounds
    pos_c, pos_p, neg_c, neg_p, pos, neg = (np.zeros((n, 13), bool) for _ in range(6))
    n10, n20, np0 = _norm(e10), _norm(e20), _norm(p[0])
    qv = _cross(p[0], e10[None])
    for i, d in enumerate(STAB_DIRS):
        det, tested, u, w, t = _stab(p[0], e10, e20, qv, d)
        derr = K * n10 * n20
        sure_test = np.abs(det) >= 1e-8 + derr
        sure_skip = np.abs(det) < 1e-8 - derr
        with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
            ad = np.abs(det)[None]
            su = K * (np0 * n20[None] + np.abs(u) * (n10 * n20)[None]) / ad
            sw = K * (np0 * n10[None] + np.abs(w) * (n10 * n20)[None]) / ad
            st = K * (n20[None] * np0 * n10[None] + np.abs(t) * (n10 * n20)[None]) / ad
            inside = ~((u < 0.0) | (u > 1.0)) & ~((w < 0.0) | (u + w > 1.0))
            in_c = (u - su >= 0.0) & (u + su <= 1.0) & (w - sw >= 0.0) & (u + w + su + sw <= 1.0)
            in_p = (u + su >= 0.0) & (u - su <= 1.0) & (w + sw >= 0.0) & (u + w - su - sw <= 1.0)
            hit = tested[None] & inside
            pos[:, i] = np.any(hit & (t >= 0.0), axis=1)
            neg[:, i] = np.any(hit & ~(t >= 0.0), axis=1)
            pos_c[:, i] = np.any(sure_test[None] & in_c & (t - st >= 0.0), axis=1)
            neg_c[:, i] = np.any(sure_test[None] & in_c & (t + st < 0.0), axis=1)
            pos_p[:, i] = np.any(~sure_skip[None] & in_p & (t + st >= 0.0), axis=1)
            neg_p[:, i] = np.any(~sure_skip[None] & in_p & (t - st < 0.0), axis=1)
    inside_pt = np.all(pos & neg, axis=1)
    sign_ok = np.all(pos_c & neg_c, axis=1) == np.all(pos_p & neg_p, axis=1)
    return best, inside_pt, sign_ok, branch_ok, edge_term


def mesh_sdf(tris: np.ndarray, points: np.ndarray, max_pairs: int = 1 << 18) -> dict:
    """tris f64 [T, 9], points f64 [N, 3] -> dict of f64 [N] 'sdf' (the rule's value) and 'tol' (its distance bound), and bool [N]
    'inside', 'sign_ok' and 'branch_ok'."""
    tris = np.asarray(tris, np.float64).reshape(-1, 9)
    points = np.asarray(points, np.float64).reshape(-1, 3)
    N, T = points.shape[0], tris.shape[0]
    res = {"sdf": np.full(N, np.inf), "tol": np.zeros(N), "inside": np.zeros(N, bool), "sign_ok": np.ones(N, bool),
           "branch_ok": np.ones(N, bool)}
    if T == 0:
        return res
    step = max(1, max_pairs // T)
    for a in range(0, N, step):
        P = points[a:a + step]
        nanp = np.isnan(P).any(1)
        best, inside, sign_ok, branch_ok, edge_term = _chunk(np.where(nanp[:, None], 0.0, P), tris)
        best = np.where(nanp, np.float32(np.inf), best)          # NaN coordinates: every distance NaN, no t >= 0 hit
        inside &= ~nanp
        d = np.sqrt(np.maximum(best, F32(0.0)).astype(F32)).astype(np.float64)
        with np.errstate(invalid="ignore"):
            ulp = np.where(np.isfinite(d), np.spacing(np.abs(d).astype(F32)).astype(np.float64), 0.0)
        res["sdf"][a:a + step] = np.where(inside, -d, d)
        res["tol"][a:a + step] = ulp + np.where(nanp, 0.0, edge_term)
        res["inside"][a:a + step] = inside
        res["sign_ok"][a:a + step] = sign_ok | nanp
        res["branch_ok"][a:a + step] = branch_ok | nanp
    return res
