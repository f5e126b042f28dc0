"""ctypes front-end of the CPU oracle (TEST INFRASTRUCTURE, NOT PRODUCT CODE).

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference leg may import
this module.  Nothing under kaolin-wisp_b200/ imports it.

It wraps oracle/wisp_oracle.c (the C restatement of the reference hot path; each C function cites
the reference file:line it follows) and adds the small numpy helpers the oracle needs on the host:
an independent SPC (octree) builder, the synthetic "lego-like" occupancy of SURVEY.md section 8(d),
the look-at camera of wisp/trainers/tracker/offline_renderer.py:23-89 and parameter packing.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
from dataclasses import dataclass, field
from typing import List, Optional, Sequence

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "libwisp_oracle.so")
_lib = None


def build(force: bool = False) -> str:
    """Compile oracle/wisp_oracle.c with the committed Makefile (gcc, OpenMP)."""
    src = os.path.join(_HERE, "wisp_oracle.c")
    if force or not os.path.exists(_LIB_PATH) or os.path.getmtime(_LIB_PATH) < os.path.getmtime(src):
        subprocess.run(["make", "-C", _HERE, "-B", "libwisp_oracle.so"], check=True, capture_output=True)
    return _LIB_PATH


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        build()
        _lib = C.CDLL(_LIB_PATH)
        _lib.wo_rf_step.restype = C.c_double
        _lib.wo_rf_trace_fwd.restype = C.c_int64
        _lib.wo_raymarch_ray_count.restype = C.c_int64
        _lib.wo_jitter_export.restype = C.c_float
        _lib.wo_jitter_export.argtypes = [C.c_uint32, C.c_uint32, C.c_uint32]
        _lib.wo_num_threads.restype = C.c_int
    return _lib


def num_threads() -> int:
    return int(lib().wo_num_threads())


def set_num_threads(n: int) -> None:
    lib().wo_set_num_threads(C.c_int(n))


def _p(a: Optional[np.ndarray]):
    if a is None:
        return None
    assert a.flags["C_CONTIGUOUS"], "oracle arrays must be contiguous"
    return a.ctypes.data_as(C.c_void_p)


def _f32(a) -> np.ndarray:
    return np.ascontiguousarray(a, dtype=np.float32)


# ----------------------------------------------------------------------------------------------
# SPC host helpers  [KAOLIN-EXT: unbatched_points_to_octree, SURVEY.md Appendix A]
# ----------------------------------------------------------------------------------------------
def morton3(points: np.ndarray, level: int) -> np.ndarray:
    """morton = sum_i (x_i << (3i+2)) | (y_i << (3i+1)) | (z_i << 3i); child index c = 4x+2y+z."""
    p = points.astype(np.int64)
    m = np.zeros(p.shape[0], dtype=np.int64)
    for i in range(level):
        m |= ((p[:, 0] >> i) & 1) << (3 * i + 2)
        m |= ((p[:, 1] >> i) & 1) << (3 * i + 1)
        m |= ((p[:, 2] >> i) & 1) << (3 * i)
    return m


def points_to_octree(points: np.ndarray, level: int) -> np.ndarray:
    """Quantised integer points [N,3] in [0, 2^level) -> SPC octree bytes (breadth first, root first).
    Mirrors spc_ops.unbatched_points_to_octree(points, level, sorted=False) (octree_as.py:132)."""
    m = np.unique(morton3(np.asarray(points), level))
    levels = []
    cur = m
    for _ in range(level):
        parent = cur >> 3
        child = (cur & 7).astype(np.uint8)
        up, inv = np.unique(parent, return_inverse=True)
        byte = np.zeros(up.shape[0], dtype=np.uint8)
        np.bitwise_or.at(byte, inv, (1 << child).astype(np.uint8))
        levels.append(byte)
        cur = up
    return np.concatenate(levels[::-1]) if levels else np.zeros(0, dtype=np.uint8)


def dense_octree(level: int) -> np.ndarray:
    """wisp.ops.spc.create_dense_octree (constructors.py:14-28): every byte 0xff."""
    n = sum(8 ** l for l in range(level))
    return np.full(n, 255, dtype=np.uint8)


@dataclass
class SPC:
    octree: np.ndarray
    prefix: np.ndarray       # int32 [nbytes+1]
    pyramid: np.ndarray      # int64 [2, max_level+2]
    points: np.ndarray       # int16 [total, 3]
    max_level: int


def octree_to_spc(octree: np.ndarray) -> SPC:
    """wisp.ops.spc.octree_to_spc (conversions.py:72-88)."""
    octree = np.ascontiguousarray(octree, dtype=np.uint8)
    n = octree.shape[0]
    prefix = np.zeros(n + 1, dtype=np.int32)
    pyr = np.zeros(2 * 64, dtype=np.int64)
    ml = lib().wo_scan_octree(_p(octree), C.c_int64(n), _p(prefix), _p(pyr), C.c_int(64))
    assert ml >= 0, "malformed octree"
    pyramid = np.stack([pyr[: ml + 2], pyr[ml + 2: 2 * (ml + 2)]]).copy()
    total = int(pyramid[1, ml + 1])
    points = np.zeros((total, 3), dtype=np.int16)
    lib().wo_generate_points(_p(octree), C.c_int64(n), _p(prefix), _p(points), C.c_int64(total))
    return SPC(octree, prefix, pyramid, points, ml)


def lego_like_points(level: int = 7) -> np.ndarray:
    """Synthetic 'lego-like' occupancy (SURVEY.md 8(d)): level-`level` cells whose centre lies in a
    3-cell-thick shell of the box |x|<0.6,|y|<0.35,|z|<0.8 or in one of 4 vertical cylinders."""
    n = 1 << level
    c = (np.arange(n, dtype=np.float64) + 0.5) / n * 2.0 - 1.0
    x, y, z = np.meshgrid(c, c, c, indexing="ij")
    cell = 2.0 / n
    inside = (np.abs(x) < 0.6) & (np.abs(y) < 0.35) & (np.abs(z) < 0.8)
    t = 3 * cell
    inner = (np.abs(x) < 0.6 - t) & (np.abs(y) < 0.35 - t) & (np.abs(z) < 0.8 - t)
    occ = inside & ~inner
    for cx, cz in ((-0.3, -0.4), (0.3, -0.4), (-0.3, 0.4), (0.3, 0.4)):
        occ |= (((x - cx) ** 2 + (z - cz) ** 2) < 0.12 ** 2) & (np.abs(y - 0.45) < 0.12)
    idx = np.argwhere(occ)
    return idx.astype(np.int16)


# ----------------------------------------------------------------------------------------------
# Rays: offline_renderer.py:23-89 (_look_at/_generate_rays) + ops/geometric.py:65-99 (normalized_grid)
# ----------------------------------------------------------------------------------------------
def look_at_rays(origin, target, height: int, width: int, fov: float = 30.0):
    f = np.asarray(origin, dtype=np.float32)
    t = np.asarray(target, dtype=np.float32)

    def nrm(v):
        return v / max(np.linalg.norm(v), 1e-12)

    view = nrm(t - f)
    right = nrm(np.cross(view, np.array([0, 1, 0], dtype=np.float32)))
    up = nrm(np.cross(right, view))
    wx = np.linspace(-1, 1, width, dtype=np.float32)
    wy = np.linspace(1, -1, height, dtype=np.float32)
    if width > height:
        wx = wx * (width / height)
    elif height > width:
        wy = wy * (height / width)
    gx, gy = np.meshgrid(wx, wy, indexing="xy")          # [H, W]
    tanf = np.float32(np.tan(np.radians(fov / 2)))
    po = (right[None, None] * gx[..., None] * tanf + up[None, None] * gy[..., None] * tanf + f + view)
    d = po.reshape(-1, 3) - f
    d = d / np.maximum(np.linalg.norm(d, axis=-1, keepdims=True), 1e-12)
    o = np.broadcast_to(f, d.shape).copy()
    return o.astype(np.float32), d.astype(np.float32)


# ----------------------------------------------------------------------------------------------
# Neural-field description shared with the C side
# ----------------------------------------------------------------------------------------------
def geometric_resolutions(num_lods: int, min_res: int, max_res: int) -> List[int]:
    """HashGrid.from_geometric (hash_grid.py:160-161)."""
    b = np.exp((np.log(max_res) - np.log(min_res)) / (num_lods - 1))
    return [int(np.floor(min_res * (b ** l))) for l in range(num_lods)]


def table_layout(resolutions: Sequence[int], codebook_bitwidth: int):
    """MultiTable (grids/utils.py:47-59): rows/level = min(2^bw, res^3)."""
    T = 2 ** codebook_bitwidth
    begin = [0]
    for r in resolutions:
        begin.append(begin[-1] + min(T, r ** 3))
    return np.asarray(begin, dtype=np.int64)


@dataclass
class Nef:
    """NeuralRadianceField(HashGrid, ...) parameters as flat numpy arrays (nerf.py:151-173)."""
    resolutions: List[int]
    feature_dim: int
    codebook_bitwidth: int
    table: np.ndarray                     # [rows, F] float32
    dens_W: List[np.ndarray]              # per linear layer [out, in]
    dens_b: Optional[List[np.ndarray]]
    col_W: List[np.ndarray]
    col_b: Optional[List[np.ndarray]]
    multiscale: str = "cat"
    lod_idx: Optional[int] = None
    pos_mode: int = 0
    pos_freq: int = 0
    view_mode: int = 3                    # positional + input (include_input=True, nerf.py:105-106)
    view_freq: int = 4
    begin: np.ndarray = field(init=False)

    def __post_init__(self):
        self.begin = table_layout(self.resolutions, self.codebook_bitwidth)
        assert self.table.shape == (int(self.begin[-1]), self.feature_dim)

    @property
    def L(self):
        return len(self.resolutions)

    def pack(self):
        L, F = self.L, self.feature_dim
        lod = (L - 1) if self.lod_idx is None else self.lod_idx
        has_bias = 1 if self.dens_b is not None else 0
        dd = [self.dens_W[0].shape[1]] + [w.shape[0] for w in self.dens_W]
        dc = [self.col_W[0].shape[1]] + [w.shape[0] for w in self.col_W]
        icfg = [L, F, 2 ** self.codebook_bitwidth, 0 if self.multiscale == "cat" else 1, lod,
                self.pos_mode, self.pos_freq, self.view_mode, self.view_freq, has_bias,
                len(self.dens_W)] + dd + [len(self.col_W)] + dc
        icfg = np.asarray(icfg, dtype=np.int32)
        res = np.asarray(self.resolutions, dtype=np.int32)

        def flat(Ws, bs):
            parts = []
            for i, w in enumerate(Ws):
                parts.append(_f32(w).reshape(-1))
                if bs is not None:
                    parts.append(_f32(bs[i]).reshape(-1))
            return np.concatenate(parts).astype(np.float32)

        return icfg, res, np.ascontiguousarray(self.begin), _f32(self.table), flat(self.dens_W, self.dens_b), flat(self.col_W, self.col_b)

    def unflatten(self, flat_d: np.ndarray, flat_c: np.ndarray):
        """Split packed parameter(-gradient) vectors back into per-layer (W, b) lists."""
        def split(flat, Ws, has_b):
            out_w, out_b, o = [], [], 0
            for w in Ws:
                n = w.size
                out_w.append(flat[o:o + n].reshape(w.shape)); o += n
                if has_b:
                    out_b.append(flat[o:o + w.shape[0]]); o += w.shape[0]
            return out_w, (out_b if has_b else None)
        hb = self.dens_b is not None
        return split(flat_d, self.dens_W, hb), split(flat_c, self.col_W, hb)


def make_nef(num_lods=16, feature_dim=2, codebook_bitwidth=19, min_res=16, max_res=512, hidden_dim=64,
             num_layers=1, bias=True, multiscale="cat", view_freq=4, seed=0, feature_std=1e-4,
             table_scale: Optional[float] = None, pos_mode=0, pos_freq=0, view_mode=3) -> Nef:
    """Random-init NeuralRadianceField in the shape of app/nerf/configs/nerf_hash.yaml.
    nn.Linear default init (kaiming-uniform, bound 1/sqrt(fan_in)); density lout.bias[0]=1 (nerf.py:162-163).
    Embedders (nerf.py:103-106): pos_mode 0 none, 1 identity, 2 positional, 3 positional + input (pos_freq bands);
    view_mode 0 none, 1 identity, 3 positional + input (view_freq bands)."""
    rng = np.random.default_rng(seed)
    res = geometric_resolutions(num_lods, min_res, max_res)
    begin = table_layout(res, codebook_bitwidth)
    std = feature_std if table_scale is None else table_scale
    table = (rng.standard_normal((int(begin[-1]), feature_dim)) * std).astype(np.float32)
    embed_dim = lambda mode, freq: 0 if mode == 0 else 3 if mode == 1 else 6 * freq if mode == 2 else 3 + 6 * freq
    feat = (num_lods * feature_dim if multiscale == "cat" else feature_dim) + embed_dim(pos_mode, pos_freq)
    view_dim = embed_dim(view_mode, view_freq)

    def linear(i, o):
        bound = 1.0 / np.sqrt(i)
        W = rng.uniform(-bound, bound, (o, i)).astype(np.float32)
        b = rng.uniform(-bound, bound, (o,)).astype(np.float32)
        return W, b

    def mlp(i, o, nl):
        Ws, bs = [], []
        d = i
        for _ in range(nl):
            W, b = linear(d, hidden_dim); Ws.append(W); bs.append(b); d = hidden_dim
        W, b = linear(d, o); Ws.append(W); bs.append(b)
        return Ws, bs

    dW, db = mlp(feat, 16, num_layers)
    db[-1][0] = 1.0
    cW, cb = mlp(15 + view_dim, 3, num_layers + 1)
    return Nef(res, feature_dim, codebook_bitwidth, table, dW, db if bias else None, cW, cb if bias else None,
               multiscale=multiscale, pos_mode=pos_mode, pos_freq=pos_freq, view_mode=view_mode, view_freq=view_freq)


# ----------------------------------------------------------------------------------------------
# C entry points
# ----------------------------------------------------------------------------------------------
def jitter(seed: int, ray: int, step: int) -> float:
    return float(lib().wo_jitter_export(seed, ray, step))


def query(spc: SPC, coords: np.ndarray, level: Optional[int] = None, with_parents: bool = False) -> np.ndarray:
    level = spc.max_level if level is None else level
    coords = _f32(coords)
    N = coords.shape[0]
    out = np.empty((N, level + 1) if with_parents else (N,), dtype=np.int32)
    lib().wo_query(_p(spc.octree), _p(spc.prefix), _p(coords), C.c_int64(N), C.c_int(level), C.c_int(int(with_parents)), _p(out))
    return out


def _ray_args(origins, dirs, near, far):
    origins, dirs = _f32(origins), _f32(dirs)
    if np.ndim(near) == 0:
        return origins, dirs, C.c_float(float(near)), C.c_float(float(far)), None, None
    nv, fv = _f32(np.reshape(near, -1)), _f32(np.reshape(far, -1))
    return origins, dirs, C.c_float(0.0), C.c_float(0.0), nv, fv


def raymarch_ray(spc: SPC, origins, dirs, near, far, num_samples: int, level: Optional[int] = None,
                 jitter_arr: Optional[np.ndarray] = None, seed: int = 0):
    """OctreeAS._raymarch_ray (octree_as.py:247-309) -> dict of ASRaymarchResults fields (+ step index, counts)."""
    level = spc.max_level if level is None else level
    o, d, ns, fs, nv, fv = _ray_args(origins, dirs, near, far)
    R = o.shape[0]
    jit = None if jitter_arr is None else _f32(jitter_arr)
    counts = np.zeros(R, dtype=np.int32)
    total = lib().wo_raymarch_ray_count(_p(spc.octree), _p(spc.prefix), C.c_int(level), _p(o), _p(d), C.c_int64(R), ns, fs,
                                        _p(nv), _p(fv), C.c_int(num_samples), _p(jit), C.c_uint32(seed), _p(counts))
    offsets = np.zeros(R, dtype=np.int64)
    np.cumsum(counts[:-1], out=offsets[1:])
    S = int(total)
    ridx = np.zeros(S, dtype=np.int64); samples = np.zeros((S, 3), dtype=np.float32)
    depth = np.zeros(S, dtype=np.float32); deltas = np.zeros(S, dtype=np.float32)
    boundary = np.zeros(S, dtype=np.uint8); step_idx = np.zeros(S, dtype=np.int32)
    lib().wo_raymarch_ray_fill(_p(spc.octree), _p(spc.prefix), C.c_int(level), _p(o), _p(d), C.c_int64(R), ns, fs, _p(nv), _p(fv),
                               C.c_int(num_samples), _p(jit), C.c_uint32(seed), _p(offsets), _p(ridx), _p(samples), _p(depth),
                               _p(deltas), _p(boundary), _p(step_idx))
    return dict(ridx=ridx, samples=samples, depth_samples=depth[:, None], deltas=deltas[:, None],
                boundary=boundary.astype(bool), step_idx=step_idx, counts=counts)


def hashgrid_fwd(coords, table, resolutions, codebook_bitwidth, return_corners=False):
    """wisp_C.ops.hashgrid_interpolate_cuda (hashgrid_interpolate.cpp:46-65): raw [N, L*F] features."""
    coords, table = _f32(coords), _f32(table)
    N, L, F = coords.shape[0], len(resolutions), table.shape[1]
    res = np.asarray(resolutions, dtype=np.int32)
    begin = table_layout(resolutions, codebook_bitwidth)
    feats = np.zeros((N, L * F), dtype=np.float32)
    corners = np.zeros((N, L, 8), dtype=np.int32) if return_corners else None
    lib().wo_hashgrid_fwd(_p(coords), C.c_int64(N), _p(table), C.c_int(L), C.c_int(F), C.c_int32(2 ** codebook_bitwidth),
                          _p(res), _p(begin), _p(feats), _p(corners))
    return (feats, corners) if return_corners else feats


def hashgrid_bwd(coords, grad_feats, n_rows, resolutions, codebook_bitwidth):
    """wisp_C.ops.hashgrid_interpolate_backward_cuda (hashgrid_interpolate.cpp:71-105), fp32 branch."""
    coords, grad_feats = _f32(coords), _f32(grad_feats)
    N, L = coords.shape[0], len(resolutions)
    F = grad_feats.shape[1] // L
    res = np.asarray(resolutions, dtype=np.int32)
    begin = table_layout(resolutions, codebook_bitwidth)
    gt = np.zeros((n_rows, F), dtype=np.float32)
    lib().wo_hashgrid_bwd(_p(coords), C.c_int64(N), _p(grad_feats), C.c_int(L), C.c_int(F), C.c_int32(2 ** codebook_bitwidth),
                          _p(res), _p(begin), _p(gt))
    return gt


def nef_rgba(nef: Nef, coords, dirs):
    icfg, res, begin, table, pd, pc = nef.pack()
    coords, dirs = _f32(coords), _f32(dirs)
    S = coords.shape[0]
    rgb = np.zeros((S, 3), dtype=np.float32); dens = np.zeros((S, 1), dtype=np.float32)
    lib().wo_nef_rgba(_p(icfg), _p(res), _p(begin), _p(table), _p(pd), _p(pc), _p(coords), _p(dirs), C.c_int64(S), _p(rgb), _p(dens))
    return rgb, dens


def exponential_integration(feats, tau, boundary):
    feats, tau = _f32(feats), _f32(np.reshape(tau, -1))
    b = np.ascontiguousarray(boundary, dtype=np.uint8)
    S, Cn = feats.shape
    P = int(b.sum())
    out = np.zeros((P, Cn), dtype=np.float32); w = np.zeros(S, dtype=np.float32)
    lib().wo_exponential_integration(_p(feats), C.c_int(Cn), _p(tau), _p(b), C.c_int64(S), _p(out), _p(w))
    return out, w[:, None]


def sum_reduce(feats, boundary):
    feats = _f32(feats)
    b = np.ascontiguousarray(boundary, dtype=np.uint8)
    S, Cn = feats.shape
    out = np.zeros((int(b.sum()), Cn), dtype=np.float32)
    lib().wo_sum_reduce(_p(feats), C.c_int(Cn), _p(b), C.c_int64(S), _p(out))
    return out


def _scene_args(spc, level, origins, dirs, near, far, n, jitter_arr, seed, nef, bg):
    level = spc.max_level if level is None else level
    o, d, ns, fs, nv, fv = _ray_args(origins, dirs, near, far)
    jit = None if jitter_arr is None else _f32(jitter_arr)
    icfg, res, begin, table, pd, pc = nef.pack()
    bgv = _f32(bg)
    keep = (o, d, nv, fv, jit, icfg, res, begin, table, pd, pc, bgv)
    args = [_p(spc.octree), _p(spc.prefix), C.c_int(level), _p(o), _p(d), C.c_int64(o.shape[0]), ns, fs, _p(nv), _p(fv),
            C.c_int(n), _p(jit), C.c_uint32(seed), _p(icfg), _p(res), _p(begin), _p(table), _p(pd), _p(pc), _p(bgv)]
    return args, keep, o.shape[0], pd.size, pc.size


def rf_trace_fwd(spc, nef: Nef, origins, dirs, near, far, num_steps, bg=(1, 1, 1), level=None, jitter_arr=None, seed=0):
    """PackedRFTracer.trace forward (packed_rf_tracer.py:84-181) -> rgb, depth, alpha, hit, counts."""
    args, keep, R, _, _ = _scene_args(spc, level, origins, dirs, near, far, num_steps, jitter_arr, seed, nef, bg)
    rgb = np.zeros((R, 3), np.float32); depth = np.zeros((R, 1), np.float32); alpha = np.zeros((R, 1), np.float32)
    hit = np.zeros(R, np.uint8); counts = np.zeros(R, np.int32)
    total = lib().wo_rf_trace_fwd(*args, _p(rgb), _p(depth), _p(alpha), _p(hit), _p(counts))
    return dict(rgb=rgb, depth=depth, alpha=alpha, hit=hit.astype(bool), counts=counts, num_samples=int(total))


def rf_trace_bwd(spc, nef: Nef, origins, dirs, near, far, num_steps, g_rgb, g_depth=None, g_alpha=None,
                 bg=(1, 1, 1), level=None, jitter_arr=None, seed=0):
    args, keep, R, nd, nc = _scene_args(spc, level, origins, dirs, near, far, num_steps, jitter_arr, seed, nef, bg)
    g_rgb = _f32(g_rgb)
    gd = None if g_depth is None else _f32(np.reshape(g_depth, -1))
    ga = None if g_alpha is None else _f32(np.reshape(g_alpha, -1))
    gt = np.zeros_like(nef.table, dtype=np.float32); gdens = np.zeros(nd, np.float32); gcol = np.zeros(nc, np.float32)
    lib().wo_rf_trace_bwd(*args, _p(g_rgb), _p(gd), _p(ga), _p(gt), _p(gdens), _p(gcol))
    return dict(table=gt, dens=gdens, col=gcol)


def rf_step(spc, nef: Nef, origins, dirs, near, far, num_steps, target, loss="huber", bg=(1, 1, 1), level=None,
            jitter_arr=None, seed=0):
    """One fused fwd+bwd pass with the trainer loss (multiview_trainer.py:140-154)."""
    args, keep, R, nd, nc = _scene_args(spc, level, origins, dirs, near, far, num_steps, jitter_arr, seed, nef, bg)
    target = _f32(target)
    rgb = np.zeros((R, 3), np.float32)
    gt = np.zeros_like(nef.table, dtype=np.float32); gdens = np.zeros(nd, np.float32); gcol = np.zeros(nc, np.float32)
    total = C.c_int64(0)
    lt = {"l2": 0, "l1": 1, "huber": 2}[loss]
    val = lib().wo_rf_step(*args, _p(target), C.c_int(lt), _p(rgb), _p(gt), _p(gdens), _p(gcol), C.byref(total))
    return dict(loss=float(val), rgb=rgb, table=gt, dens=gdens, col=gcol, num_samples=int(total.value))


# ----------------------------------------------------------------------------------------------
# raytrace + 'voxel' / 'uniform' marching
# ----------------------------------------------------------------------------------------------
def raytrace(spc: SPC, origins, dirs, level: Optional[int] = None):
    """OctreeAS.raytrace(with_exit=True) (octree_as.py:165-186) -> ridx i32[Ng], pidx i32[Ng], depth f32[Ng,2], counts i32[R]."""
    level = spc.max_level if level is None else level
    o, d = _f32(origins), _f32(dirs)
    R = o.shape[0]
    lib().wo_raytrace_count.restype = C.c_int64
    counts = np.zeros(R, dtype=np.int32)
    total = int(lib().wo_raytrace_count(_p(spc.octree), _p(spc.prefix), C.c_int(level), _p(o), _p(d), C.c_int64(R), _p(counts)))
    offsets = np.zeros(R, dtype=np.int64)
    np.cumsum(counts[:-1], out=offsets[1:])
    ridx = np.zeros(total, np.int32); pidx = np.zeros(total, np.int32); depth = np.zeros((total, 2), np.float32)
    lib().wo_raytrace_fill(_p(spc.octree), _p(spc.prefix), C.c_int(level), _p(o), _p(d), C.c_int64(R), _p(offsets), _p(ridx), _p(pidx), _p(depth))
    return dict(ridx=ridx, pidx=pidx, depth=depth, counts=counts)


def raymarch_voxel(spc: SPC, origins, dirs, num_samples: int, level: Optional[int] = None, jitter_arr=None, seed: int = 0):
    """OctreeAS._raymarch_voxel (octree_as.py:188-245)."""
    o, d = _f32(origins), _f32(dirs)
    rt = raytrace(spc, o, d, level)
    Ng = rt["ridx"].shape[0]
    S = Ng * num_samples
    jit = None if jitter_arr is None else _f32(jitter_arr)
    ridx = np.zeros(S, np.int64); samples = np.zeros((S, 3), np.float32); depth = np.zeros(S, np.float32)
    deltas = np.zeros(S, np.float32); boundary = np.zeros(S, np.uint8)
    lib().wo_raymarch_voxel(_p(o), _p(d), _p(rt["ridx"]), _p(rt["depth"]), C.c_int64(Ng), C.c_int(num_samples), _p(jit), C.c_uint32(seed),
                            _p(ridx), _p(samples), _p(depth), _p(deltas), _p(boundary))
    return dict(ridx=ridx, samples=samples, depth_samples=depth[:, None], deltas=deltas[:, None], boundary=boundary.astype(bool), nuggets=rt)


def raymarch_uniform(spc: SPC, origins, dirs, num_samples: int, level: Optional[int] = None):
    """OctreeAS._raymarch_uniform (octree_as.py:311-374)."""
    o, d = _f32(origins), _f32(dirs)
    rt = raytrace(spc, o, d, level)
    Ng = rt["ridx"].shape[0]
    scale = int(lib().wo_uniform_scale(C.c_int(num_samples)))
    lib().wo_raymarch_uniform_count.restype = C.c_int64
    cnt = np.zeros(Ng, np.int32)
    S = int(lib().wo_raymarch_uniform_count(_p(rt["depth"]), C.c_int64(Ng), C.c_int(scale), _p(cnt)))
    offsets = np.zeros(max(Ng, 1), np.int64)
    if Ng > 1:
        np.cumsum(cnt[:-1], out=offsets[1:Ng])
    ridx = np.zeros(S, np.int64); samples = np.zeros((S, 3), np.float32); depth = np.zeros(S, np.float32)
    deltas = np.zeros(S, np.float32); boundary = np.zeros(S, np.uint8)
    lib().wo_raymarch_uniform_fill(_p(o), _p(d), _p(rt["ridx"]), _p(rt["depth"]), C.c_int64(Ng), C.c_int(scale), _p(cnt), _p(offsets),
                                   _p(ridx), _p(samples), _p(depth), _p(deltas), _p(boundary))
    return dict(ridx=ridx, samples=samples, depth_samples=depth[:, None], deltas=deltas[:, None], boundary=boundary.astype(bool), nuggets=rt, scale=scale)
