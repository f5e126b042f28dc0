"""PackedSDFTracer.trace (packed_sdf_tracer.py:78-174) restated in vectorised numpy, exactly rounded, with the counters the tracer
tests need.

The loop is oracle/octree_grid.py:sdf_trace statement for statement, with two differences in how it is computed, not in what:
  * find_depth_bound (find_depth_bound_cuda.cu:16-45) runs over all packs at once, one numpy pass per nugget offset instead of a
    Python loop per pack.  Its quirks are kept: the output starts at -1, the scan of pack p stops at the CURRENT cursor of pack p+1,
    the last pack is bounded by the number of packs (not of nuggets), and a -1 neighbour cursor wraps through `uint`.
  * torch.addcmul(o, d, t) is a correctly rounded fp32 fma.  oracle's restatement rounds the float64 sum to fp32, which rounds
    twice and can differ from a true fma in the last bit; here the float64 sum is rounded to odd first (exact for the final
    rounding to fp32, 53 >= 24 + 2 bits).

Besides the RenderBuffer channels trace() returns:
  evals       field evaluations, as the device counter of wb_sdf_trace counts them: every pack once, the packs still alive after
              each jump, and 6 per hit for the normals
  iters       loop bodies entered;  exit: 'march' / 'jump' (the `if not mask.any(): break` that ended the loop) or 'steps'
  bound_stops scans of find_depth_bound that ended at the next pack's cursor without a nugget (the last pack's bound excluded)
  dist_max_kills  packs the march ended because t reached dist_max
  packs, nuggets, dist0 (the first distance of every pack)
"""
from __future__ import annotations

import numpy as np

_INF = np.float64(np.inf)


def fma32(a, b, c) -> np.ndarray:
    """fp32 fma(a, b, c), correctly rounded.  The float64 product of two fp32 values is exact; TwoSum gives the float64 sum s and
    its exact error e; rounding s to odd (an even s with e != 0 moves one ulp towards e) before the cast to fp32 rounds once."""
    a, b, c = (np.asarray(v, np.float32).astype(np.float64) for v in (a, b, c))
    p = a * b
    s = p + c
    bp = s - c
    e = (p - bp) + (c - (s - bp))
    even = (s.view(np.int64) & 1) == 0
    fix = (e != 0) & even & np.isfinite(s)
    if np.any(fix):
        s = np.where(fix, np.nextafter(s, np.where(e > 0, _INF, -_INF)), s)
    return s.astype(np.float32)


def find_depth_bound(query: np.ndarray, curr: np.ndarray, depth: np.ndarray, stats: dict | None = None) -> np.ndarray:
    """find_depth_bound_cuda.cu:16-45 over all packs at once (see the module docstring for the kept quirks).  query f32 [P] or
    [P,1], curr int32 [P], depth f32 [Ng,2] (entry already offset by 1e-5, as the tracer passes it).  stats['bound_stops'] counts the
    scans that ended at the next pack's cursor without a nugget."""
    q = np.asarray(query, np.float32).reshape(-1)
    curr = np.asarray(curr, np.int32)
    P, Ng = q.shape[0], depth.shape[0]
    out = np.full(P, -1, np.int32)
    if P == 0:
        return out
    mx = np.empty(P, np.int64)
    mx[:-1] = curr[1:].astype(np.int64) & 0xFFFFFFFF          # `uint max_iidx = curr_idxes[tidx+1]`: -1 wraps
    mx[-1] = P                                                 # the last pack: num_packs, not the number of nuggets
    i = curr.astype(np.int64)
    live = np.nonzero(curr > -1)[0]
    i = i[live]
    bound = 0
    while live.size:
        inside = (i < mx[live]) & (i < Ng)
        stop = ~inside
        if stop.any():
            bound += int(np.count_nonzero(stop & (i >= mx[live]) & (live != P - 1)))
            live, i = live[inside], i[inside]
            if not live.size:
                break
        en, ex = depth[i, 0], depth[i, 1]
        qq = q[live]
        found = ((qq >= en) & (qq <= ex)) | (qq < en)
        out[live[found]] = i[found]
        live, i = live[~found], i[~found] + 1
    if stats is not None:
        stats["bound_stops"] = stats.get("bound_stops", 0) + bound
    return out


def trace(origins, dirs, ridx, depth, field, lod_idx, num_steps=64, step_size=1.0, min_dis=1e-4, dist_max=6.0, with_normals=True) -> dict:
    """PackedSDFTracer.trace (packed_sdf_tracer.py:78-174) over the nuggets of a raytrace (ridx int32 [Ng], depth f32 [Ng,2] raw
    entry/exit).  field(x f32 [N,3], lod_idx or None) -> f32 [N,1]; None asks for the finest LOD (the normals)."""
    o, d = np.asarray(origins, np.float32), np.asarray(dirs, np.float32)
    ridx = np.asarray(ridx, np.int32)
    depth = np.asarray(depth, np.float32).copy()
    R, Ng = o.shape[0], ridx.shape[0]
    out = dict(xyz=np.zeros((R, 3), np.float32), depth=np.zeros((R, 1), np.float32), hit=np.zeros(R, bool), normal=np.zeros((R, 3), np.float32),
               rgb=np.zeros((R, 3), np.float32), alpha=np.zeros((R, 1), np.float32))
    stats = dict(evals=0, iters=0, exit="none", bound_stops=0, dist_max_kills=0, packs=0, nuggets=Ng, dist0=np.zeros((0, 1), np.float32))
    if Ng == 0:
        if with_normals:
            out["rgb"][:] = 0.5
        out.update(stats)
        return out
    depth[:, 0:1] += np.float32(1e-5)                                         # :91
    first = np.ones(Ng, bool); first[1:] = ridx[1:] != ridx[:-1]              # mark_pack_boundaries
    curr = np.nonzero(first)[0].astype(np.int32)
    first_ridx = ridx[first].astype(np.int64)
    no, nd = o[first_ridx], d[first_ridx]
    P = first_ridx.shape[0]
    stats["packs"] = P
    addcmul = lambda tt: fma32(nd, tt, no)                                    # torch.addcmul(nug_o, nug_d, t): fma per component
    step = np.float32(step_size)
    min1, min5 = np.float32(min_dis * 1.0), np.float32((min_dis * 5) * 1.0)
    dm = np.float32(dist_max)
    mask = np.ones(P, bool); hit = np.zeros(P, bool)
    t = depth[first][:, 0:1].copy()
    x = addcmul(t)
    dist = np.zeros_like(t)
    dist[mask] = field(x[mask], lod_idx) * np.float32(1.0) * step
    stats["evals"] += P
    stats["dist0"] = dist.copy()
    dist_prev = dist.copy()
    for _ in range(num_steps):
        stats["iters"] += 1
        t = t + dist                                                          # unmasked: dead packs drift
        x = np.where(mask[:, None], addcmul(t), x)
        hit = np.where(mask, np.abs(dist)[:, 0] < min1, hit)
        hit = hit | np.where(mask, np.abs(dist + dist_prev)[:, 0] * np.float32(0.5) < min5, hit)
        far = mask & ~(t < dm)[:, 0] & ~hit
        stats["dist_max_kills"] += int(far.sum())
        mask = np.where(mask, (t < dm)[:, 0], mask)
        mask = mask & ~hit
        if not mask.any():
            stats["exit"] = "march"
            break
        dist_prev = np.where(mask[:, None], dist, dist_prev)
        nxt = find_depth_bound(t, curr, depth, stats)
        mask = mask & (nxt != -1)
        aabb = nxt != curr
        curr = np.where(mask, nxt, curr)
        t = np.where((mask & aabb)[:, None], depth[curr.astype(np.int64), 0:1], t)
        x = np.where(mask[:, None], addcmul(t), x)
        if not mask.any():
            stats["exit"] = "jump"
            break
        dist[mask] = field(x[mask], lod_idx) * np.float32(1.0) * step
        stats["evals"] += int(mask.sum())
    else:
        stats["exit"] = "steps"
    hb = np.zeros(R, bool); hb[first_ridx] = hit
    out["hit"] = hb
    out["xyz"][hb] = x[hit]; out["depth"][hb] = t[hit]
    if with_normals:
        eps = np.float32(0.005)
        xh = x[hit]
        g = []
        for a in range(3):
            e = np.zeros(3, np.float32); e[a] = eps
            g.append(field(xh + e, None) - field(xh - e, None))               # lod_idx=None -> finest LOD (gradients.py:29-45)
        stats["evals"] += 6 * xh.shape[0]
        grad = np.concatenate(g, -1) / np.float32(0.005 * 2.0) if xh.shape[0] else np.zeros((0, 3), np.float32)
        nrm = np.sqrt((grad.astype(np.float32) ** 2).sum(-1, keepdims=True))
        out["normal"][hb] = grad / np.maximum(nrm, np.float32(1e-5))
        out["rgb"][:] = (out["normal"] + 1.0) / 2.0
    out["alpha"][hb] = 1.0
    out.update(stats)
    return out


def sdf_trace(case, num_steps=64, step_size=1.0, min_dis=1e-4, lod_idx=None, dist_max=6.0, with_normals=True, field=None) -> dict:
    """trace() on an oracle.octree_grid.make_sdf_case case, with the arguments of oracle.octree_grid.sdf_trace: the nuggets from
    oracle.raytrace at the LOD's level, the case's own NeuralSDF as the default field."""
    from oracle import octree_grid as OG
    from oracle import oracle as O
    lod_idx = len(case["active_lods"]) - 1 if lod_idx is None else lod_idx
    fn = field or (lambda x, lod=None: OG.neural_sdf(case, x, lod))
    rt = O.raytrace(case["spc"], case["origins"], case["dirs"], case["active_lods"][lod_idx])
    return trace(case["origins"], case["dirs"], rt["ridx"], rt["depth"], fn, lod_idx, num_steps, step_size, min_dis, dist_max, with_normals)
