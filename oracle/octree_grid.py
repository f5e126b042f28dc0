"""Oracle definitions for the OctreeGrid / NGLOD-SDF path (TEST INFRASTRUCTURE, NOT PRODUCT CODE).

[KAOLIN-EXT, PARITY UNPINNED] kaolin.ops.spc.{unbatched_make_dual, unbatched_make_trinkets, unbatched_interpolate_trilinear,
coords_to_trilinear_coeffs} have no source under /root/reference; these numpy restatements follow SURVEY.md Appendix A and the
call sites wisp/ops/spc/constructors.py:31-47 and wisp/models/grids/octree_grid.py:130-163.  Also restated here:
find_depth_bound (wisp/csrc/render/find_depth_bound_cuda.cu:16-45).
"""
from __future__ import annotations

import numpy as np

from . import oracle as O


def _morton_wide(p: np.ndarray, bits: int) -> np.ndarray:
    p = p.astype(np.int64)
    m = np.zeros(p.shape[0], dtype=np.int64)
    for i in range(bits):
        m |= ((p[:, 0] >> i) & 1) << (3 * i + 2)
        m |= ((p[:, 1] >> i) & 1) << (3 * i + 1)
        m |= ((p[:, 2] >> i) & 1) << (3 * i)
    return m


CORNERS = np.array([[(j >> 2) & 1, (j >> 1) & 1, j & 1] for j in range(8)], dtype=np.int64)


def make_trilinear_spc(spc: O.SPC):
    """-> points_dual int16 [Td,3], pyramid_dual int64 [2, L+2], trinkets int32 [T,8] (LEVEL-LOCAL dual index of corner j,
    z fastest), parents int32 [T] (global index of the parent cell, -1 for the root)."""
    L = spc.max_level
    pts = spc.points.astype(np.int64)
    duals, trinkets, parents = [], np.zeros((pts.shape[0], 8), np.int32), np.full(pts.shape[0], -1, np.int32)
    pyr = np.zeros((2, L + 2), np.int64)
    off = 0
    for l in range(L + 1):
        s, c = int(spc.pyramid[1, l]), int(spc.pyramid[0, l])
        cell = pts[s:s + c]
        corners = (cell[:, None, :] + CORNERS[None]).reshape(-1, 3)
        key = _morton_wide(corners, l + 1)
        uk, inv = np.unique(key, return_inverse=True)
        first = np.zeros(uk.shape[0], np.int64); first[inv[::-1]] = np.arange(corners.shape[0])[::-1]
        duals.append(corners[first].astype(np.int16))
        trinkets[s:s + c] = inv.reshape(c, 8).astype(np.int32)
        pyr[0, l] = uk.shape[0]; pyr[1, l] = off; off += uk.shape[0]
        if l > 0:
            ps, pc = int(spc.pyramid[1, l - 1]), int(spc.pyramid[0, l - 1])
            pkey = _morton_wide(pts[ps:ps + pc], l)
            ckey = _morton_wide(cell >> 1, l)
            parents[s:s + c] = (ps + np.searchsorted(pkey, ckey)).astype(np.int32)
    pyr[1, L + 1] = off
    return np.concatenate(duals), pyr, trinkets, parents


def trilinear_coeffs(coords: np.ndarray, points: np.ndarray, level: int) -> np.ndarray:
    """coords_to_trilinear_coeffs: u = 2^level (c*0.5+0.5) - point; [(1-ux)(1-uy)(1-uz), (1-ux)(1-uy)uz, ...] z fastest."""
    u = (2.0 ** level) * (coords.astype(np.float64) * 0.5 + 0.5) - points.astype(np.float64)
    u = u.astype(np.float32); iu = (1.0 - u).astype(np.float32)
    out = np.zeros((coords.shape[0], 8), np.float32)
    for j in range(8):
        cx = u[:, 0] if (j & 4) else iu[:, 0]; cy = u[:, 1] if (j & 2) else iu[:, 1]; cz = u[:, 2] if (j & 1) else iu[:, 2]
        out[:, j] = (cx * cy) * cz
    return out


def interpolate_trilinear(coords: np.ndarray, pidx: np.ndarray, points: np.ndarray, trinkets: np.ndarray, feats: np.ndarray, level: int,
                          half: bool = True) -> np.ndarray:
    """unbatched_interpolate_trilinear for one sample per cell: out = sum_j feats[trinkets[pidx, j]] * coef_j; pidx == -1 -> 0.
    half=True reproduces the call site's `feats.half()` ... `.float()` (octree_grid.py:147-149): features and result rounded to fp16."""
    N, Fd = coords.shape[0], feats.shape[1]
    out = np.zeros((N, Fd), np.float32)
    ok = pidx >= 0
    if ok.any():
        p = pidx[ok].astype(np.int64)
        cf = trilinear_coeffs(coords[ok], points[p], level)
        f = feats.astype(np.float16).astype(np.float32) if half else feats.astype(np.float32)
        acc = np.zeros((p.shape[0], Fd), np.float32)
        for j in range(8):
            acc = acc + f[trinkets[p, j].astype(np.int64)] * cf[:, j:j + 1]
        out[ok] = acc.astype(np.float16).astype(np.float32) if half else acc
    return out


def octree_grid_interpolate(spc: O.SPC, trinkets: np.ndarray, features, active_lods, coords: np.ndarray, lod_idx: int, multiscale: str,
                            half: bool = True) -> np.ndarray:
    """OctreeGrid.interpolate (octree_grid.py:165-219)."""
    base = active_lods[0]
    pidx = O.query(spc, coords, active_lods[lod_idx], with_parents=True)[:, base:]
    feats = [interpolate_trilinear(coords, pidx[:, i], spc.points, trinkets, features[i], active_lods[i], half) for i in range(lod_idx + 1)]
    if lod_idx == 0:
        return feats[0]
    out = np.concatenate(feats, -1)
    if multiscale == "sum":
        out = out.reshape(out.shape[0], lod_idx + 1, -1).sum(-2)
    return out


def find_depth_bound(query: np.ndarray, curr_idxes: np.ndarray, depth: np.ndarray) -> np.ndarray:
    """wisp/csrc/render/find_depth_bound_cuda.cu:16-45 including its quirks: the output starts at -1 (find_depth_bound.cpp),
    the scan of pack i stops at the CURRENT cursor of pack i+1, and the last pack is bounded by num_packs (not num_nugs)."""
    P = query.shape[0]
    out = np.full(P, -1, np.int32)
    q = query.reshape(-1)
    for t in range(P):
        if curr_idxes[t] <= -1:
            continue
        i = int(curr_idxes[t]); mx = P if t == P - 1 else int(curr_idxes[t + 1])
        mx = mx & 0xFFFFFFFF                                     # `uint max_iidx = ...`: a -1 cursor of the next pack wraps around
        while i < mx:
            if i >= depth.shape[0]:
                break
            en, ex = depth[i, 0], depth[i, 1]
            if (q[t] >= en and q[t] <= ex) or q[t] < en:
                out[t] = i
                break
            i += 1
    return out


# ------------------------------------------------------------------------------------------------------------------
# NeuralSDF.sdf + PackedSDFTracer.trace restated in numpy (TEST INFRASTRUCTURE; pinned by tests/golden/sdf_octree*.npz,
# which the reference's own classes produced through oracle/ref_import.py)
# ------------------------------------------------------------------------------------------------------------------
def make_sdf_case(level=5, num_lods=3, feature_dim=8, hidden_dim=16, multiscale="sum", res=20, seed=7, feature_std=0.05,
                  cam=(-2.0, 0.9, -1.6), fov=40.0, radius=0.52):
    """Synthetic app/nglod scene: octahedron-surface octree, OctreeGrid features, NeuralSDF(position_input, 1 hidden layer)
    whose decoder is (|x|+|y|+|z|)/sqrt(3) - 0.3 plus a small feature-driven perturbation (as oracle/make_golden.py:gen_sdf)."""
    rng = np.random.default_rng(seed)
    p = rng.standard_normal((400000, 3)); p = p / np.abs(p).sum(-1, keepdims=True) * radius
    q = np.unique(np.floor(np.clip((2 ** level) * (p + 1.0) / 2.0, 0, 2 ** level - 1)).astype(np.int16), axis=0)
    octree = O.points_to_octree(q, level)
    spc = O.octree_to_spc(octree)
    _, pyr, trinkets, _ = make_trilinear_spc(spc)
    base = level - num_lods + 1
    active = [base + i for i in range(num_lods)]
    feats = [(rng.standard_normal((int(pyr[0, l]) + 1, feature_dim)) * feature_std).astype(np.float32) for l in active]
    in_dim = 3 + (feature_dim if multiscale == "sum" else feature_dim * num_lods)
    b = 1.0 / np.sqrt(in_dim)
    W0 = (rng.uniform(-b, b, (hidden_dim, in_dim)) * 0.05).astype(np.float32)
    W0[:6, :3] = np.array([[1, 0, 0], [-1, 0, 0], [0, 1, 0], [0, -1, 0], [0, 0, 1], [0, 0, -1.0]], np.float32)
    b0 = np.zeros(hidden_dim, np.float32)
    bh = 1.0 / np.sqrt(hidden_dim)
    W1 = (rng.uniform(-bh, bh, (1, hidden_dim)) * 0.05).astype(np.float32); W1[0, :6] = 1.0 / np.sqrt(3.0)
    b1 = np.full(1, -0.3, np.float32)
    o, d = O.look_at_rays(list(cam), [0, 0, 0], res, res, fov)
    return dict(octree=octree, spc=spc, level=level, trinkets=trinkets, pyramid_dual=pyr, active_lods=active, feats=feats, multiscale=multiscale,
                W=[W0, W1], b=[b0, b1], origins=o, dirs=d, feature_dim=feature_dim, hidden_dim=hidden_dim)


def neural_sdf(case, coords: np.ndarray, lod_idx=None) -> np.ndarray:
    """NeuralSDF.sdf (neural_sdf.py:120-155), pos_embedder='none' + position_input: decoder(cat([coords, grid feats])) -> [N,1]."""
    if coords.shape[0] == 0:
        return np.zeros((0, 1), np.float32)
    lod_idx = len(case["active_lods"]) - 1 if lod_idx is None else lod_idx
    f = octree_grid_interpolate(case["spc"], case["trinkets"], case["feats"], case["active_lods"], coords.astype(np.float32), lod_idx, case["multiscale"])
    h = np.concatenate([coords.astype(np.float32), f.astype(np.float32)], -1)
    Ws, bs = case["W"], case["b"]
    for W, b in zip(Ws[:-1], bs[:-1]):
        h = np.maximum(h @ W.T + b, 0.0).astype(np.float32)
    return (h @ Ws[-1].T + bs[-1]).astype(np.float32)


def sdf_trace(case, num_steps=64, step_size=1.0, min_dis=1e-4, lod_idx=None, dist_max=6.0, with_normals=True, return_debug=False, field=None):
    """PackedSDFTracer.trace (packed_sdf_tracer.py:78-174), statement by statement, on numpy arrays.
    Kept quirks: `t += dist` also advances packs that already terminated (so depth drifts by dist per executed iteration after
    the hit while xyz does not); the loop ends when no pack is alive anywhere; find_depth_bound's bounds (see above).
    field(coords, lod_idx) -> [N,1] float32 is the SDF (default: the case's own NeuralSDF, neural_sdf)."""
    spc, o, d = case["spc"], case["origins"], case["dirs"]
    lod_idx = len(case["active_lods"]) - 1 if lod_idx is None else lod_idx
    sdf = field or (lambda x, lod=None: neural_sdf(case, x, lod))
    rt = O.raytrace(spc, o, d, case["active_lods"][lod_idx])
    ridx, depth = rt["ridx"], rt["depth"].copy()
    R = o.shape[0]
    out = dict(xyz=np.zeros((R, 3), np.float32), depth=np.zeros((R, 1), np.float32), hit=np.zeros(R, bool), normal=np.zeros((R, 3), np.float32),
               rgb=np.zeros((R, 3), np.float32), alpha=np.zeros((R, 1), np.float32))
    if ridx.shape[0] == 0:
        if with_normals:
            out["rgb"][:] = 0.5
        return out
    depth[:, 0:1] += np.float32(1e-5)                                         # :91
    first = np.ones(ridx.shape[0], bool); first[1:] = ridx[1:] != ridx[:-1]   # mark_pack_boundaries
    curr = np.nonzero(first)[0].astype(np.int32)
    first_ridx = ridx[first].astype(np.int64)
    no, nd = o[first_ridx], d[first_ridx]
    P = first_ridx.shape[0]
    mask = np.ones(P, bool); hit = np.zeros(P, bool)
    t = depth[first][:, 0:1].copy()
    fma = lambda tt: (nd.astype(np.float64) * tt.astype(np.float64) + no.astype(np.float64)).astype(np.float32)   # addcmul == fma
    x = fma(t)
    dist = np.zeros_like(t)
    step = np.float32(step_size)
    dist[mask] = sdf(x[mask], lod_idx) * np.float32(1.0) * step
    dist_prev = dist.copy()
    iters = 0
    for i in range(num_steps):
        iters += 1
        t = t + dist
        x = np.where(mask[:, None], fma(t), x)
        hit = np.where(mask, np.abs(dist)[:, 0] < np.float32(min_dis * 1.0), hit)
        hit = hit | np.where(mask, np.abs(dist + dist_prev)[:, 0] * np.float32(0.5) < np.float32((min_dis * 5) * 1.0), hit)
        mask = np.where(mask, (t < np.float32(dist_max))[:, 0], mask)
        mask = mask & ~hit
        if not mask.any():
            break
        dist_prev = np.where(mask[:, None], dist, dist_prev)
        nxt = find_depth_bound(t, curr, depth)
        mask = mask & (nxt != -1)
        aabb = nxt != curr
        curr = np.where(mask, nxt, curr)
        t = np.where((mask & aabb)[:, None], depth[curr.astype(np.int64), 0:1], t)
        x = np.where(mask[:, None], fma(t), x)
        if not mask.any():
            break
        dist[mask] = sdf(x[mask], lod_idx) * np.float32(1.0) * step
    hb = np.zeros(R, bool); hb[first_ridx] = hit
    out["hit"] = hb
    out["xyz"][hb] = x[hit]; out["depth"][hb] = t[hit]
    if with_normals:
        eps = np.float32(0.005)
        xh = x[hit]
        g = []
        for a in range(3):
            e = np.zeros(3, np.float32); e[a] = eps
            g.append(sdf(xh + e) - sdf(xh - e))     # lod_idx=None -> finest LOD (gradients.py:29-45)
        grad = np.concatenate(g, -1) / np.float32(0.005 * 2.0) if xh.shape[0] else np.zeros((0, 3), np.float32)
        nrm = np.sqrt((grad.astype(np.float32) ** 2).sum(-1, keepdims=True))
        out["normal"][hb] = grad / np.maximum(nrm, np.float32(1e-5))
        out["rgb"][:] = (out["normal"] + 1.0) / 2.0
    out["alpha"][hb] = 1.0
    if return_debug:
        out["iters"] = iters
    return out
