"""Restatements for the mesh-octree checks (TEST INFRASTRUCTURE, numpy only, NOT PRODUCT CODE).

limit_set(V, F, level)      the cells the reference's sampler (wisp.ops.spc.mesh_to_octree) can ever mark, in float64: the cells
                            whose closed box, grown by h = 2^-(level+1) (the largest jitter), meets a triangle.  Decided by the
                            separating-axis test on 13 axes (the 3 box normals, the face normal, the 9 edge x box-normal crosses);
                            a pair whose separation is at most `tol` along a unit axis counts as meeting (fp32 rounding of the
                            sample positions).  -> bool [res, res, res].
sample_bits(...)            wb_mesh_octree_bits restated draw by draw (the counter-based stream, the 53-bit inverse CDF, the fp32
                            sample, jitter and quantization), for checking the kernel word for word at small sample counts.
octree_cells(octree)        the finest level's cells of an octree as a bool [res, res, res] grid.
"""
from __future__ import annotations

import numpy as np


def limit_set(V, F, level: int, tol: float = 1e-6) -> np.ndarray:
    V = np.asarray(V, np.float64)
    res = 2 ** level
    cell, h = 2.0 / res, 2.0 ** -(level + 1)
    e = 0.5 * cell + h                                      # half extent of a grown cell box
    eye = np.eye(3)
    out = np.zeros((res, res, res), bool)
    for f in np.asarray(F, np.int64):
        T = V[f]
        if not np.all(np.isfinite(T)):
            continue
        lo = np.clip(np.floor((T.min(0) - e - tol + 1.0) / cell).astype(np.int64), 0, res - 1)
        hi = np.clip(np.floor((T.max(0) + e + tol + 1.0) / cell).astype(np.int64), 0, res - 1)
        g = np.stack(np.meshgrid(*[np.arange(lo[a], hi[a] + 1) for a in range(3)], indexing="ij"), -1).reshape(-1, 3)
        v = T[None] - ((g + 0.5) * cell - 1.0)[:, None]    # triangle relative to each cell centre [n, 3, 3]
        ed = [T[1] - T[0], T[2] - T[1], T[0] - T[2]]
        axes = [eye[i] for i in range(3)] + [np.cross(ed[0], ed[1])] + [np.cross(eye[i], ed[j]) for i in range(3) for j in range(3)]
        ok = np.ones(len(g), bool)
        for a in axes:
            na = np.linalg.norm(a)
            if na == 0.0:
                continue
            p = v @ a
            r = e * np.abs(a).sum() + tol * na
            ok &= ~((p.min(1) > r) | (p.max(1) < -r))
        gg = g[ok]
        out[gg[:, 0], gg[:, 1], gg[:, 2]] = True
    return out


def octree_cells(octree) -> np.ndarray:
    """The finest level of an octree (uint8 bytes, numpy or torch) as a bool grid, through this package's spc (CPU)."""
    import torch
    from wisp_b200 import spc as S
    o = torch.as_tensor(np.asarray(octree.cpu() if hasattr(octree, "cpu") else octree, np.uint8))
    ml, pyramid, _ = S.scan_octree(o)
    pts = S.generate_points(o, pyramid)[int(pyramid[1, ml]):int(pyramid[1, ml]) + int(pyramid[0, ml])].long().numpy()
    res = 2 ** ml
    g = np.zeros((res, res, res), bool)
    g[pts[:, 0], pts[:, 1], pts[:, 2]] = True
    return g


# ---- wb_mesh_octree_bits, draw by draw ----------------------------------------------------------------------------------------
def _mix32(x):
    x = x.astype(np.uint32)
    x ^= x >> np.uint32(16); x *= np.uint32(0x21F0AAAD)
    x ^= x >> np.uint32(15); x *= np.uint32(0x735A2D97)
    x ^= x >> np.uint32(15)
    return x


def _draw(key, d: int):
    return _mix32(key ^ np.uint32((d * 0x85EBCA77 + 0x165667B1) & 0xFFFFFFFF))


def _u24(h):
    return (h >> np.uint32(8)).astype(np.float32) * np.float32(2.0 ** -24)


def _quantize(x, res: float):
    q = (np.float32(res) * (x + np.float32(1.0))) * np.float32(0.5)
    return np.floor(np.minimum(np.maximum(q, np.float32(0.0)), np.float32(res - 1.0))).astype(np.int64)


def sample_bits(tris, cdf, num_samples: int, level: int, seed: int, first: int = 0) -> np.ndarray:
    """The uint32 bitmask [(8^level + 31) // 32] that wb_mesh_octree_bits sets for samples first .. first + num_samples - 1 of the
    stream `seed`, from the same tris (f32 [T, 9]) and cdf (f64 [T + 1]) it is given."""
    tris = np.asarray(tris, np.float32).reshape(-1, 9)
    cdf = np.asarray(cdf, np.float64)
    T = tris.shape[0]
    i = np.arange(first, first + num_samples, dtype=np.uint64)
    lo32, hi32 = (i & np.uint64(0xFFFFFFFF)).astype(np.uint32), (i >> np.uint64(32)).astype(np.uint32)
    with np.errstate(over="ignore"):
        key = _mix32(_mix32(np.uint32(seed & 0xFFFFFFFF) + lo32 * np.uint32(0x9E3779B1)) ^ (hi32 * np.uint32(0xC2B2AE35) + np.uint32(0x27D4EB2F)))
        u53 = (_draw(key, 0).astype(np.uint64) << np.uint64(21)) | (_draw(key, 1) >> np.uint32(11)).astype(np.uint64)
        target = u53.astype(np.float64) * 2.0 ** -53 * cdf[T]
        f = np.searchsorted(cdf[1:], target, side="right")
        for k in np.nonzero(f == T)[0]:                     # the target rounded up to the total: the last face of nonzero area
            g = T - 1
            while g > 0 and not cdf[g + 1] > cdf[g]:
                g -= 1
            f[k] = g
        r1, v = _u24(_draw(key, 2)), _u24(_draw(key, 3))
        u = np.sqrt(r1)
        wa, wb, wc = np.float32(1.0) - u, u * (np.float32(1.0) - v), u * v
        t = tris[f]
        h = np.float32(2.0 ** -(level + 1))
        res = float(2 ** level)
        q, qj = [], []
        for k in range(3):
            x = (wa * t[:, k] + wb * t[:, 3 + k]) + wc * t[:, 6 + k]
            j = (_u24(_draw(key, 4 + k)) * np.float32(2.0) - np.float32(1.0)) * h
            q.append(_quantize(x, res)); qj.append(_quantize(x + j, res))
    bits = np.zeros((8 ** level + 31) // 32, np.uint32)
    for c in (q, qj):
        idx = (c[0] << (2 * level)) | (c[1] << level) | c[2]
        np.bitwise_or.at(bits, idx >> 5, (np.uint32(1) << (idx & 31).astype(np.uint32)))
    return bits
