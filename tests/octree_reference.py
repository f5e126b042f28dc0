"""Exact CPU reference of the octree traversal kernels: wb_query (wb_spc.cu), the 'ray' marcher (wb_raymarch.cu) and the
raytrace nuggets behind the 'voxel' / 'uniform' samplers (wb_raytrace.cu).  numpy + fractions only; no oracle code.

  cell_of(x, L)       the level-L cell of an fp32 coordinate, floor((x + 1) * 2^(L-1)) evaluated exactly (a miss outside
                      [0, 2^L)); Fraction where float64 could round (|x| < 2^-20).
  OctIndex.query      cell_of + descent: the point index of the cell (and of its parents) in the SPC, or -1.
  nuggets(...)        every occupied level-L cell whose slab intersection [max(te, 0), tx] with the ray o + t d (fp32 o, d
                      taken as exact rationals) has positive length -- on an axis with d == 0 the cell is [lo, hi), where cell_of
                      puts the ray's points -- with its entry / exit, the rounding radius of each and the cells whose
                      classification a correctly rounded fp32 evaluation could flip (ambiguous).
  march_depths(...)   the candidate depths of the 'ray' marcher, op by op in fp32 (the documented contract with the
                      reference's torch kernels); the tests pin them bit for bit against the oracle's kept samples.
  march_hits(...)     cell_of + descent of the fp32 points fma(d, t, o) of those depths.

Rounding radius.  The kernels compute each slab depth as fl(fl(lo - o) / d) with lo, hi exact fp32 dyadics, so each depth is
within (2u + u^2)|t| (u = 2^-24) of the exact one, plus 2^-149 for underflow; the entry is a max and the exit a min of such depths,
so the same bound holds for them.  The entry / exit are computed in float64 (relative error <= 2^-51, eight orders below the
radius) and every decision that float64 could get wrong -- a length or a length-minus-radii within 2^-40 |t| of zero -- is
redone with Fraction.
"""
from __future__ import annotations

from fractions import Fraction

import numpy as np

f32, f64 = np.float32, np.float64
U = 2.0 ** -24
RAD = 2 * U + U * U                 # relative radius of fl(fl(lo - o) / d)
TINY = 2.0 ** -149                  # absolute radius: the quotient may underflow
FLT_MAX = float(np.finfo(np.float32).max)


# ---- cells -------------------------------------------------------------------------------------------------------------
def cell_of(x, level: int):
    """-> (q int64, inside bool): q = floor((x + 1) * 2^(level-1)) exactly, inside = 0 <= q < 2^level (NaN: outside)."""
    x = np.asarray(x, dtype=f32)
    h = 2.0 ** (level - 1)
    xd = x.astype(f64)
    with np.errstate(invalid="ignore", over="ignore"):
        y = (xd + 1.0) * h                        # exact for |x| >= 2^-28: x + 1 needs at most 53 bits, * 2^(L-1) is exact
        q = np.floor(y)
    small = np.abs(xd) < 2.0 ** -20
    for i in np.flatnonzero(small):
        fr = (Fraction(float(xd.flat[i])) + 1) * Fraction(2) ** (level - 1)
        q.flat[i] = float(fr.numerator // fr.denominator)
    inside = np.isfinite(q) & (q >= 0) & (q < 2 ** level)
    return np.where(inside, q, -1).astype(np.int64), inside


def _key(x, y, z):
    return (np.asarray(x, np.int64) << 32) | (np.asarray(y, np.int64) << 16) | np.asarray(z, np.int64)


class OctIndex:
    """Occupied cells of every level of an SPC (points / pyramid of oracle.octree_to_spc) as sorted keys -> point index."""

    def __init__(self, spc):
        self.max_level = int(spc.max_level)
        self.levels = []
        for l in range(self.max_level + 1):
            start, cnt = int(spc.pyramid[1, l]), int(spc.pyramid[0, l])
            p = spc.points[start:start + cnt].astype(np.int64)
            k = _key(p[:, 0], p[:, 1], p[:, 2])
            order = np.argsort(k, kind="stable")
            self.levels.append((k[order], (start + order).astype(np.int64)))

    def lookup(self, level: int, qx, qy, qz):
        """point index of the level cells (qx, qy, qz), -1 where empty."""
        keys, idx = self.levels[level]
        k = _key(qx, qy, qz)
        if keys.shape[0] == 0:
            return np.full(k.shape, -1, np.int64)
        pos = np.minimum(np.searchsorted(keys, k), keys.shape[0] - 1)
        return np.where(keys[pos] == k, idx[pos], -1)

    def query(self, coords, level: int, with_parents: bool = False):
        """OctreeAS.query: cell_of on each axis, then the descent; parents[l] for l = 0..level (-1 below the first empty one)."""
        c = np.asarray(coords, dtype=f32).reshape(-1, 3)
        qs, ins = zip(*(cell_of(c[:, a], level) for a in range(3)))
        inside = ins[0] & ins[1] & ins[2]
        out = np.full((c.shape[0], level + 1), -1, dtype=np.int64)
        for l in range(level + 1):
            s = level - l
            out[:, l] = np.where(inside, self.lookup(l, qs[0] >> s, qs[1] >> s, qs[2] >> s), -1)
        # the tree is nested: a missing cell has no descendants, so every index below the first -1 is -1 already
        return (out if with_parents else out[:, level]).astype(np.int32)


# ---- nuggets -------------------------------------------------------------------------------------------------------------
def _slab64(o, d, cells, level):
    """float64 slab of ray rows o, d [P,3] with cells [P,3] of `level` -> te, tx (-inf / +inf where no axis bounds them),
    and `out` where an axis with d == 0 has o outside the closed cell range."""
    size = 2.0 / (1 << level)
    lo = cells * size - 1.0                                     # exact dyadics
    hi = lo + size
    par = d == 0.0
    with np.errstate(divide="ignore", invalid="ignore"):
        ta = (lo - o) / d
        tb = (hi - o) / d
    tmin = np.where(par, -np.inf, np.minimum(ta, tb))
    tmax = np.where(par, np.inf, np.maximum(ta, tb))
    out = (par & ((o < lo) | (o >= hi))).any(axis=1)
    return tmin.max(axis=1), tmax.min(axis=1), out


def _exact_len(o, d, cell, level):
    """Fraction entry max(te, 0) and exit of one ray / cell (exit None when unbounded); None when a parallel axis misses."""
    size = Fraction(2, 1 << level)
    te, tx = None, None
    for a in range(3):
        lo = int(cell[a]) * size - 1
        hi = lo + size
        oa, da = Fraction(float(o[a])), Fraction(float(d[a]))
        if da == 0:
            if oa < lo or oa >= hi:
                return None
            continue
        ta, tb = (lo - oa) / da, (hi - oa) / da
        a0, a1 = min(ta, tb), max(ta, tb)
        te = a0 if te is None else max(te, a0)
        tx = a1 if tx is None else min(tx, a1)
    en = Fraction(0) if te is None else max(te, Fraction(0))
    return en, tx


def nuggets(index: OctIndex, o, d, level: int):
    """Every occupied level-`level` cell that is an exact nugget of a ray or that fp32 rounding could make one.

    Returns a dict of arrays over those (ray, cell) pairs, sorted by ray, then exact entry, then exit:
      ray, pidx, cell [.,3], entry, exit (float64 within 2^-51 relative of the exact values), r_entry, r_exit (rounding radii),
      exact (exact length > 0), amb (|exact length| <= r_entry + r_exit, or a depth beyond the fp32 range),
      amb_order (the exact entry lies within the radii of the next pair's entry without being equal to it)."""
    o = np.asarray(o, f32).reshape(-1, 3).astype(f64)
    d = np.asarray(d, f32).reshape(-1, 3).astype(f64)
    R = o.shape[0]
    ray = np.arange(R, dtype=np.int64)
    cells = np.zeros((R, 3), np.int64)
    for l in range(level + 1):
        if l > 0:                                                # expand to the occupied children
            ch = np.array([[(c >> 2) & 1, (c >> 1) & 1, c & 1] for c in range(8)], np.int64)
            cells = (2 * cells[:, None, :] + ch[None]).reshape(-1, 3)
            ray = np.repeat(ray, 8)
            occ = index.lookup(l, cells[:, 0], cells[:, 1], cells[:, 2]) >= 0
            cells, ray = cells[occ], ray[occ]
        te, tx, out = _slab64(o[ray], d[ray], cells, l)
        en = np.maximum(te, 0.0)
        # keep every cell whose length is not clearly negative: 2^-16 relative is far outside the fp32 radius (2^-23), so
        # this superset holds every exact nugget and every cell an fp32 slab test could accept, at every level (children
        # lie inside their parent)
        with np.errstate(invalid="ignore"):
            keep = ~out & ((tx - en) >= -(2.0 ** -16) * (np.abs(en) + np.abs(tx)) - 2.0 ** -140)
        cells, ray = cells[keep], ray[keep]
    te, tx, _ = _slab64(o[ray], d[ray], cells, level)
    en = np.maximum(te, 0.0)
    with np.errstate(invalid="ignore"):
        length = tx - en
    r_en = RAD * np.abs(en) + TINY
    r_tx = np.where(np.isinf(tx), 0.0, RAD * np.abs(tx) + TINY)
    exact = length > 0
    amb = np.abs(length) <= r_en + r_tx
    scale = np.abs(en) + np.where(np.isinf(tx), 0.0, np.abs(tx))
    near = (np.abs(length) <= 2.0 ** -40 * scale + TINY) | (np.abs(np.abs(length) - (r_en + r_tx)) <= 2.0 ** -40 * scale + TINY)
    near &= ~np.isinf(tx)
    for i in np.flatnonzero(near):                              # decisions float64 could get wrong: exactly
        r = int(ray[i])
        ex = _exact_len(o[r], d[r], cells[i], level)
        if ex is None:
            exact[i], amb[i] = False, False
            continue
        e_en, e_tx = ex
        ln = e_tx - e_en
        exact[i] = ln > 0
        amb[i] = abs(ln) <= Fraction(RAD) * (abs(e_en) + abs(e_tx)) + 2 * Fraction(TINY)
    amb |= (np.abs(en) > FLT_MAX / 2) | (np.isfinite(tx) & (np.abs(tx) > FLT_MAX / 2))
    sel = exact | amb
    ray, cells, en, tx, r_en, r_tx, exact, amb = (a[sel] for a in (ray, cells, en, tx, r_en, r_tx, exact, amb))
    order = np.lexsort((tx, en, ray))
    ray, cells, en, tx, r_en, r_tx, exact, amb = (a[order] for a in (ray, cells, en, tx, r_en, r_tx, exact, amb))
    amb_order = np.zeros(ray.shape[0], bool)
    if ray.shape[0] > 1:
        same = ray[1:] == ray[:-1]
        gap = en[1:] - en[:-1]
        close = same & (gap > 0) & (gap <= r_en[1:] + r_en[:-1])
        amb_order[:-1] |= close
        amb_order[1:] |= close
    pidx = index.lookup(level, cells[:, 0], cells[:, 1], cells[:, 2])
    return dict(ray=ray, pidx=pidx, cell=cells, entry=en, exit=tx, r_entry=r_en, r_exit=r_tx, exact=exact, amb=amb,
                amb_order=amb_order)


# ---- the 'ray' marcher ---------------------------------------------------------------------------------------------------
def fma32(a, b, c):
    """Correctly rounded fp32 fma(a, b, c) of fp32 arrays: a*b is exact in float64; the float64 sum is corrected where it
    lands on an fp32 rounding midpoint (the only case where rounding twice differs from rounding once)."""
    a, b, c = (np.asarray(v, f32) for v in (a, b, c))
    x = a.astype(f64) * b.astype(f64)
    cd = np.broadcast_to(c.astype(f64), x.shape)
    s = x + cd
    bv = s - x
    err = (x - (s - bv)) + (cd - bv)                            # TwoSum: s + err == x + c exactly
    with np.errstate(over="ignore"):
        r = np.array(s.astype(f32), copy=True)
    r64 = r.astype(f64)
    toward = np.where(s > r64, np.inf, -np.inf).astype(f32)
    nb = np.nextafter(r, toward)
    mid = (s != r64) & (s == (r64 + nb.astype(f64)) / 2) & (err != 0)
    fix = mid & (np.sign(err) == np.sign(nb.astype(f64) - r64))       # the exact sum lies beyond the midpoint, on nb's side
    r[fix] = nb[fix]
    return r


def _mix32(x):
    x = np.asarray(x, np.uint32).copy()
    x ^= x >> np.uint32(16); x *= np.uint32(0x21F0AAAD)
    x ^= x >> np.uint32(15); x *= np.uint32(0x735A2D97)
    x ^= x >> np.uint32(15)
    return x


def jitter_stream(seed: int, R: int, n: int):
    """The counter-based jitter (wb_common.cuh wb_jitter): [R, n] float32."""
    with np.errstate(over="ignore"):
        key = _mix32(np.uint32(seed) + np.arange(R, dtype=np.uint32) * np.uint32(0x9E3779B1))
        step = np.arange(n, dtype=np.uint32) * np.uint32(0x85EBCA77) + np.uint32(0x165667B1)
        h = _mix32(key[:, None] ^ step[None, :])
    return (h >> np.uint32(8)).astype(f32) * f32(1.0 / 16777216.0)


def march_depths(R: int, n: int, near, far, jitter):
    """[R, n] candidate depths of OctreeAS._raymarch_ray: (linspace(0,1,n)[i] + jit / n) * (far - near) + near, op by op in fp32.
    near / far: python floats (scalar: the range is (float)(double(far) - double(near)) of their fp32 values) or [R] arrays."""
    jit = np.asarray(jitter, f32).reshape(R, n)
    i = np.arange(n)
    if n == 1:
        lin = np.zeros(1, f32)
    else:
        step = f32(1.0) / f32(n - 1)
        lo = fma32(np.full(n, step, f32), i.astype(f32), np.zeros(n, f32))
        hi = fma32(np.full(n, -step, f32), (n - 1 - i).astype(f32), np.ones(n, f32))
        lin = np.where(i < n // 2, lo, hi).astype(f32)
    if np.ndim(near) == 0:
        nv = np.full(R, f32(near), f32)
        rng = np.full(R, f32(f64(f32(far)) - f64(f32(near))), f32)
    else:
        nv = np.asarray(near, f32).reshape(R)
        rng = np.asarray(far, f32).reshape(R) - nv
    q = jit / f32(n)                                            # == jit * (1/n) when n is a power of two
    dep = (lin[None, :] + q).astype(f32)
    dep = (dep * rng[:, None]).astype(f32)
    return (dep + nv[:, None]).astype(f32)


def march_hits(index: OctIndex, o, d, depths, level: int):
    """[R, n] bool: the fp32 point fma(d, t, o) of candidate depth t lies in an occupied level cell."""
    o = np.asarray(o, f32).reshape(-1, 3); d = np.asarray(d, f32).reshape(-1, 3)
    t = np.asarray(depths, f32)
    pts = np.stack([fma32(d[:, a:a + 1], t, o[:, a:a + 1]) for a in range(3)], axis=-1)
    return index.query(pts.reshape(-1, 3), level).reshape(t.shape) >= 0


# ---- adversarial octrees and rays (shared by the CPU and the GPU tests) ---------------------------------------------------------
def _lines(level: int):
    n = 1 << level
    i = np.arange(n)
    c = np.full(n, n // 3)
    return np.concatenate([np.stack([i, c, c], 1), np.stack([c, i, n - 1 - c], 1), np.stack([i, i, i], 1),
                           np.stack([i, n - 1 - i, c], 1)]).astype(np.int16)


def octree_points(name: str):
    """-> (quantized points int16 [N,3], level) of the named adversarial octree."""
    from oracle import oracle as O
    kind, level = name.rstrip("0123456789"), int(name[len(name.rstrip("0123456789")):])
    n = 1 << level
    if kind == "lego":
        return O.lego_like_points(level), level
    if kind == "corner_lo":
        return np.zeros((1, 3), np.int16), level
    if kind == "corner_hi":
        return np.full((1, 3), n - 1, np.int16), level
    if kind == "dense":
        return np.argwhere(np.ones((n, n, n), bool)).astype(np.int16), level
    if kind == "checker":
        idx = np.argwhere(np.ones((n, n, n), bool))
        return idx[idx.sum(1) % 2 == 0].astype(np.int16), level
    if kind == "random":                                      # ~1 % occupancy (from level 10 on, of the low octant only)
        rng = np.random.default_rng(level)
        m = n if level < 10 else n // 2
        return rng.integers(0, m, (int(0.01 * m ** 3), 3)).astype(np.int16), level
    if kind == "lines":
        return _lines(level), level
    if kind == "faces":                                       # occupied box = the whole cube: cells on the -x and +z faces + corners
        i = np.arange(n)
        a, b = np.meshgrid(i, i, indexing="ij")
        a, b = a.ravel(), b.ravel()
        corners = np.array([[x, y, z] for x in (0, n - 1) for y in (0, n - 1) for z in (0, n - 1)])
        return np.concatenate([np.stack([np.zeros_like(a), a, b], 1), np.stack([a, b, np.full_like(a, n - 1)], 1),
                               corners]).astype(np.int16), level
    raise ValueError(name)


def _unit(v):
    v = np.asarray(v, f64)
    return (v / np.linalg.norm(v, axis=-1, keepdims=True)).astype(f32)


def adversarial_rays(points, level: int, seed: int = 0, camera: int = 16):
    """Rays of `points`' octree at `level` -> (o, d) float32 [R,3] with the named groups listed in `groups` (name -> slice)."""
    from oracle import oracle as O
    rng = np.random.default_rng(seed)
    n = 1 << level
    h = 2.0 ** (level - 1)
    groups, os_, ds = {}, [], []

    def add(name, o, d):
        o, d = np.asarray(o, f32).reshape(-1, 3), np.asarray(d, f32).reshape(-1, 3)
        start = sum(x.shape[0] for x in os_)
        os_.append(o); ds.append(d)
        groups[name] = slice(start, start + o.shape[0])

    o, d = O.look_at_rays([-3.0, 0.65, -3.0], [0, 0, 0], camera, camera, 30.0)
    add("camera", o, d)
    o, d = O.look_at_rays([2.2, -1.7, 2.9], [0.1, 0.0, -0.05], camera // 2, camera // 2, 45.0)
    add("camera2", o, d)
    pts = np.asarray(points, np.int64)
    sel = pts[rng.integers(0, pts.shape[0], 96)]
    add("in_occupied", ((sel + rng.uniform(0.05, 0.95, sel.shape)) / h - 1.0), _unit(rng.standard_normal((96, 3))))
    add("in_any", rng.uniform(-1, 1, (96, 3)), _unit(rng.standard_normal((96, 3))))
    # origins on dyadic faces / edges / corners of this level (and one coarser level), and one ulp either side
    k = rng.integers(0, n + 1, (64, 3)).astype(f64) / h - 1.0
    k[:16, 1:] = rng.uniform(-1, 1, (16, 2))                     # face
    k[16:32, 2] = rng.uniform(-1, 1, 16)                         # edge
    k[48:] = np.round(k[48:] * (h / 2)) / (h / 2)                # corner of the coarser level
    k = k.astype(f32)
    dk = _unit(rng.standard_normal((64, 3)))
    add("on_grid", k, dk)
    add("on_grid_below", np.nextafter(k, f32(-2)), dk)
    add("on_grid_above", np.nextafter(k, f32(2)), dk)
    # +0.0 / -0.0 direction components
    dz = _unit(rng.standard_normal((64, 3)))
    dz[:16, 0] = 0.0; dz[16:32, 1] = -0.0; dz[32:48, 0] = -0.0; dz[32:48, 2] = 0.0; dz[48:, 1] = 0.0; dz[48:, 2] = -0.0
    add("zero_components", rng.uniform(-1.2, 1.2, (64, 3)), dz)
    add("zero_components_on_grid", k, dz)
    # axis-aligned rays running exactly along cell faces (one coordinate on the grid) and edges (two)
    oa = rng.uniform(-1, 1, (64, 3))
    ax = rng.integers(0, 3, 64)
    for i in range(64):
        for a in range(3):
            if a != ax[i] and (i < 32 or a == (ax[i] + 1) % 3):
                oa[i, a] = rng.integers(0, n + 1) / h - 1.0
        oa[i, ax[i]] = rng.choice([-1.5, 1.5])
    da = np.zeros((64, 3), f32)
    da[np.arange(64), ax] = np.where(oa[np.arange(64), ax] < 0, 1.0, -1.0)
    da[::2] = -da[::2]                                           # half of them point away from the cube
    odd = da[1::2]
    odd[odd == 0] = -0.0                                        # and half of them carry -0.0 in the other components
    add("along_faces", oa, da)
    # direction components below the marcher's 1e-12 cull threshold, and denormal ones
    dt = _unit(rng.standard_normal((64, 3)))
    dt[:32, rng.integers(0, 3)] = rng.choice([1e-13, -1e-13, 1e-40, -1e-40, 1e-44, -3e-39], 32)
    dt[32:, :2] = rng.choice([1e-13, -1e-13, 1e-40, -1e-44], (32, 2))
    add("tiny_components", rng.uniform(-0.99, 0.99, (64, 3)), dt)
    # unnormalised directions
    du = _unit(rng.standard_normal((64, 3)))
    add("short_dirs", rng.uniform(-1.5, 1.5, (32, 3)), du[:32] * f32(1e-3))
    add("long_dirs", rng.uniform(-1.5, 1.5, (32, 3)), du[32:] * f32(1e3))
    # far origins aimed at the cube, and rays pointing away from it
    for dist in (1e3, 1e4):
        dirn = _unit(rng.standard_normal((32, 3)))
        tgt = rng.uniform(-0.9, 0.9, (32, 3))
        add(f"far_{int(dist)}", tgt + dirn * dist, _unit(-dirn))
    oo = rng.uniform(-1.2, 1.2, (32, 3)) + np.sign(rng.uniform(-1, 1, (32, 3))) * 1.5
    add("pointing_away", oo, _unit(oo + rng.uniform(-0.3, 0.3, (32, 3))))
    # rays through the corners of the occupied box and of its 1e-4 widened margin
    lo, hi = pts.min(0) / h - 1.0, (pts.max(0) + 1) / h - 1.0
    cs = np.array([[(hi if (c >> a) & 1 else lo)[a] for a in range(3)] for c in range(8)])
    widened = np.where(cs == lo, cs - 1e-4, cs + 1e-4).astype(f32)
    tg = np.concatenate([cs, widened, np.nextafter(widened, f32(0)), np.nextafter(widened, f32(9))]).astype(f32)
    src = tg + _unit(rng.standard_normal((tg.shape[0], 3))) * 2.5
    add("bbox_corners", src, tg - src.astype(f32))
    # rays grazing a lower face of the occupied box: the origin k ulps outside, a direction component of k ulps per unit depth
    # (above the cull's 1e-12 threshold); from depth ~0.5 on the fp32 points fma(d, t, o) round onto the face, i.e. into the
    # occupied cells, before the exact ray crosses it at depth 1
    go, gd = [], []
    for a in range(3):
        face = pts[pts[:, a] == pts[:, a].min()]
        for k in (1, 2, 3):
            p = face[rng.integers(0, face.shape[0])]
            oa = np.asarray((p + 0.5) / h - 1.0, f32)
            b = f32(lo[a])
            oa[a] = b
            for _ in range(k):
                oa[a] = np.nextafter(oa[a], f32(-2))
            da = np.zeros(3, f32)
            da[a] = f32(f64(b) - f64(oa[a]))
            da[(a + 1) % 3] = f32(0.25 / h)
            go.append(oa); gd.append(da)
    add("grazing_bbox", np.array(go), np.array(gd))
    return np.concatenate(os_).astype(f32), np.concatenate(ds).astype(f32), groups


# ---- checks shared by the CPU and GPU tests ----------------------------------------------------------------------------------
def check_nuggets(ref, spc, level, ridx, pidx, depth):
    """Nuggets (ridx, pidx, depth [.,2]) of a kernel or the oracle against nuggets(): none outside the exact-or-ambiguous set, no
    unambiguous exact one missing, entry / exit within the radii, points[pidx] of `level`, entries non-decreasing along each ray
    (unless the earlier nugget's length is ambiguous).  -> (count, ambiguous, max |k - exact| / radius)."""
    ridx, pidx = np.asarray(ridx, np.int64), np.asarray(pidx, np.int64)
    depth = np.asarray(depth, f32).reshape(-1, 2).astype(f64)
    start, cnt = int(spc.pyramid[1, level]), int(spc.pyramid[0, level])
    assert ((pidx >= start) & (pidx < start + cnt)).all(), "pidx outside the level's points"
    kk = (ridx << 32) | pidx
    assert np.unique(kk).shape[0] == kk.shape[0], "a nugget appears twice"
    rk = (ref["ray"] << 32) | ref["pidx"]
    order = np.argsort(rk)
    pos = np.minimum(np.searchsorted(rk[order], kk), max(rk.shape[0] - 1, 0))
    matched = (rk[order][pos] == kk) if rk.shape[0] else np.zeros(kk.shape, bool)
    bad = np.flatnonzero(~matched)
    assert bad.size == 0, f"{bad.size} nuggets outside the exact-or-ambiguous set, e.g. ray {ridx[bad[:4]]} point {pidx[bad[:4]]} depth {depth[bad[:4]]}"
    row = order[pos]
    need = np.flatnonzero(ref["exact"] & ~ref["amb"])
    have = np.isin(rk[need], kk)
    assert have.all(), f"{(~have).sum()} unambiguous exact nuggets missing, e.g. ray {ref['ray'][need[~have][:4]]} cell {ref['cell'][need[~have][:4]]}"
    en, ex = ref["entry"][row], ref["exit"][row]
    r_en, r_ex = ref["r_entry"][row], ref["r_exit"][row]
    e_en = np.abs(depth[:, 0] - en)
    inf_ex = np.isinf(ex)
    assert (depth[inf_ex, 1] == ex[inf_ex]).all()
    e_ex = np.abs(depth[~inf_ex, 1] - ex[~inf_ex])
    ratio = max(float((e_en / r_en).max(initial=0.0)), float((e_ex / r_ex[~inf_ex]).max(initial=0.0)))
    assert ratio <= 1.0, f"depth outside the rounding radius: {ratio}"
    same = ridx[1:] == ridx[:-1]
    assert (np.diff(ridx) >= 0).all(), "nuggets not grouped by ray"
    dec = same & (depth[1:, 0] < depth[:-1, 0]) & ~ref["amb"][row[:-1]]
    assert not dec.any(), f"entries decrease along ray {ridx[1:][dec][:4]}"
    return kk.shape[0], int(ref["amb"].sum()), ratio


def hit_matrix_from_mask(hitmask, n):
    """[R, nw] int32 words of the marcher -> [R, n] bool."""
    w = np.asarray(hitmask).view(np.uint32)
    bits = (w[:, :, None] >> np.arange(32, dtype=np.uint32)) & 1
    return bits.reshape(w.shape[0], -1)[:, :n].astype(bool)
