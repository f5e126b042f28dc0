"""Meshes aimed at wb_mesh_sdf's bounding-volume hierarchy, and a numpy restatement of the tree it builds over them.

morton_keys restates wb_msdf_bounds_kernel and wb_msdf_morton_kernel: fp32 centroids, the fp32 centroid bounds, the quantisation
(c - lo) * (1023 / ext) truncated to 10 bits per axis, and the key code << 32 | t.  leaf_depths gives the depth of every leaf of the
Karras tree over the sorted keys: the tree is the binary radix tree, whose internal node between sorted leaves i and i + 1 splits
at delta_i = clz(k_i ^ k_i+1), so leaf j's ancestors are the strict running minima of delta scanned outward from j on each side.
The query kernel's stack holds at most one entry per ancestor: a depth of at most 61 fits kMsdfStack = 64."""
from __future__ import annotations

import numpy as np

import mesh_sdf_reference as R

F32 = np.float32
# A degenerate triangle far off the mesh: it adds nothing under the rule (zero normal, det = 0 in every stab direction), but
# its |coordinate| of 1e30 makes both culling margins cover everything and collapses every other Morton code.
SENTINEL = np.array([1e30, 3.1e29, -2.7e29])


def with_sentinel(V, F):
    """The mesh with the sentinel triangle appended."""
    return np.concatenate([V, SENTINEL[None]]), np.concatenate([F, np.full((1, 3), V.shape[0], F.dtype)])


def _spread10(x):
    x = x.astype(np.uint64) & 0x3FF
    x = (x | (x << 16)) & 0x030000FF
    x = (x | (x << 8)) & 0x0300F00F
    x = (x | (x << 4)) & 0x030C30C3
    x = (x | (x << 2)) & 0x09249249
    return x


def morton_keys(tris):
    """tris f64 [T, 9] -> the uint64 keys wb_msdf_morton_kernel writes (unsorted)."""
    v = np.asarray(tris, np.float64).reshape(-1, 3, 3)
    with np.errstate(over="ignore", invalid="ignore"):
        c = ((v[:, 0] + v[:, 1] + v[:, 2]) * (1.0 / 3.0)).astype(F32)
    fin = np.isfinite(c)
    lo = np.where(fin, c, F32(np.inf)).min(0)
    hi = np.where(fin, c, F32(-np.inf)).max(0)
    code = np.zeros(v.shape[0], np.uint64)
    for a in range(3):
        ext = F32(hi[a] - lo[a])
        with np.errstate(over="ignore", invalid="ignore"):
            q = (c[:, a] - lo[a]) * (F32(1023.0) / ext) if ext > 0 else np.zeros(v.shape[0], F32)
        q = np.fmin(np.fmax(q, F32(0.0)), F32(1023.0))
        code |= _spread10(q.astype(np.uint32)) << np.uint64(2 - a)
    return (code << np.uint64(32)) | np.arange(v.shape[0], dtype=np.uint64)


def _clz64(x):
    hi, lo = (x >> np.uint64(32)).astype(np.float64), (x & np.uint64(0xFFFFFFFF)).astype(np.float64)
    bits = np.where(hi > 0, 32 + np.frexp(hi)[1], np.frexp(lo)[1])          # bit length (exact below 2^53)
    return 64 - bits


def leaf_depths(tris):
    """The number of internal ancestors of every leaf of the Karras tree over tris' sorted keys -> int [T]."""
    k = np.sort(morton_keys(tris))
    T = k.shape[0]
    if T < 2:
        return np.zeros(T, np.int64)
    delta = _clz64(k[:-1] ^ k[1:])

    def records(seq):            # for each prefix seq[:j], the number of its strict minima scanned from the end
        out, stack = np.zeros(len(seq) + 1, np.int64), []
        for j, x in enumerate(seq):
            while stack and stack[-1] >= x:
                stack.pop()
            stack.append(x)
            out[j + 1] = len(stack)
        return out
    left = records(delta.tolist())                  # leaf j: ancestors among delta[0 .. j-1]
    right = records(delta[::-1].tolist())[::-1]     # leaf j: ancestors among delta[j .. T-2]
    return left + right


def _dyadic_tris(centres, offsets):
    """Triangles centre + o0, centre + o1, centre - o0 - o1 (dyadic offsets: the centroid is the centre exactly)."""
    o0, o1 = offsets
    return np.concatenate([centres + o0, centres + o1, centres - o0 - o1], axis=1)


def caterpillar(group: int = 1024):
    """Triangles whose quantised centroids are 2^b on Morton bit b = 0 .. 29 (the centroid bounds are [0, 1023] on every axis, so
    1023 / ext = 1 and a centroid quantises to itself), plus `group` triangles on centroid 0, the deepest code.  -> tris [T, 9]."""
    cents = [np.zeros(3), np.full(3, 1023.0)]
    for b in range(30):
        c = np.zeros(3)
        c[2 - b % 3] = 2.0 ** (b // 3)
        cents.append(c)
    cents = np.array(cents)
    o0, o1 = np.array([0.25, 0.0, 0.125]), np.array([-0.125, 0.25, 0.0])
    tris = [_dyadic_tris(cents, (o0, o1))]
    s = (1.0 + np.arange(1, group) / 1024.0)[:, None]
    tris.append(_dyadic_tris(np.zeros((group - 1, 3)), (o0 * s, o1[::-1] * s)))
    return np.concatenate(tris)


def fan(T: int, seed: int = 0):
    """T triangles of seeded shapes sharing the centroid (0.25, -0.125, 0.5) exactly: every Morton code is equal."""
    rng = np.random.default_rng(seed)
    o0, o1 = rng.integers(-64, 65, (2, T, 3)) / 64.0
    return _dyadic_tris(np.broadcast_to([0.25, -0.125, 0.5], (T, 3)), (o0, o1))


def flat_grid(n: int, h: float = 0.125):
    """An n x n grid of squares of side h in the plane z = 0, two equal right triangles each: (V, F)."""
    x, y = np.meshgrid(np.arange(n + 1) * h, np.arange(n + 1) * h, indexing="ij")
    V = np.stack([x, y, np.zeros_like(x)], -1).reshape(-1, 3)
    i, j = np.meshgrid(np.arange(n), np.arange(n), indexing="ij")
    a, b, c, d = i * (n + 1) + j, (i + 1) * (n + 1) + j, (i + 1) * (n + 1) + j + 1, i * (n + 1) + j + 1
    F = np.concatenate([np.stack([a, b, c], -1).reshape(-1, 3), np.stack([a, c, d], -1).reshape(-1, 3)])
    return V, F


def points_near(tris, rng, n_per=24):
    """Points around each triangle: on and off the face along its normal, beyond vertices and edges along the axes, at distances
    from 1e-9 to 3 of its size, and one fp32 ulp outside each face of its fp32 box."""
    v = tris.reshape(-1, 3, 3)
    T = v.shape[0]
    size = np.abs(v - v.mean(1, keepdims=True)).max((1, 2))[:, None] + 1e-300
    out = []
    for _ in range(n_per // 6):
        bary = rng.dirichlet((1.0, 1.0, 1.0), T) * rng.uniform(0.9, 1.1, (T, 1))
        on = (v * bary[:, :, None]).sum(1)
        nor = np.cross(v[:, 1] - v[:, 0], v[:, 2] - v[:, 0])
        nn = np.linalg.norm(nor, axis=1, keepdims=True)
        nor = np.where(nn > 0, nor / np.where(nn > 0, nn, 1.0), np.array([0.0, 0.0, 1.0]))
        h = size * 10.0 ** rng.uniform(-9, 0.5, (T, 1)) * rng.choice([-1.0, 1.0], (T, 1))
        out.append(on + h * nor)
        axis = np.eye(3)[rng.integers(0, 3, T)] * rng.choice([-1.0, 1.0], (T, 1))
        out.append(v[np.arange(T), rng.integers(0, 3, T)] + size * 10.0 ** rng.uniform(-9, 0.5, (T, 1)) * axis)
        out.append(on + size * rng.normal(size=(T, 3)))
        lo, hi = R.outward_box(tris)
        a = rng.integers(0, 3, T)
        p = on.copy()
        p[np.arange(T), a] = np.nextafter(lo[np.arange(T), a], F32(-np.inf)).astype(np.float64)
        out.append(p)
        p = on.copy()
        p[np.arange(T), a] = np.nextafter(hi[np.arange(T), a], F32(np.inf)).astype(np.float64)
        out.append(p)
        out.append(v.mean(1) + size * rng.uniform(-3, 3, (T, 3)))
    return np.concatenate(out)
