#!/usr/bin/env python
"""Generate tests/golden/spc_trace.npz: renders of the reference's own SPCField (wisp/models/nefs/spc_field.py) through its own
PackedSPCTracer (wisp/tracers/packed_spc_tracer.py), run on CPU from an UNMODIFIED kaolin-wisp checkout (TEST INFRASTRUCTURE).

    python tools/make_spc_golden.py

oracle/ref_import.py answers the Kaolin calls (scan_octrees, generate_points, unbatched_raytrace, mark_pack_boundaries) with the
oracle's definitions, so the nuggets are the oracle's, bit for bit what wb_raytrace_fill gives.

Octrees: 'octa5' (level 5, every cell whose centre lies in |x| + |y| + |z| <= 0.8) and 'rand7' (level 7, 1 % of the cells, seeded).
Colour sources (spc_field.py:69-114), one field each: 'rgba' uint8 RGBA colours, 'normals' float32 unit normals (float64 ones fail
the reference's own rgb index put, packed_spc_tracer.py:87) and 'coords' (no features: the finest level's point coordinates / 2^level).
Rays (the same for every field of an octree): four 32 x 32 look-at cameras (outside hitting, outside missing, inside the cube, past
the cube looking away) and axis-aligned rays running along cell faces and edges of the finest level (zero direction components).
Recorded: the octree bytes, features and rays, and per field the depth [R, 1], hit [R], rgb [R, 3], alpha [R, 1] of trace() at the
finest level (lod_idx None) and, for octa5, at level 3 (lod_idx 3: the reference indexes the colours with negative rows)."""
from __future__ import annotations

import os
import sys
import warnings

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
OUT = os.path.join(ROOT, "tests", "golden", "spc_trace.npz")
f32 = np.float32


def octree_points(name):
    if name == "octa5":
        n = 32
        c = (np.arange(n) + 0.5) / n * 2.0 - 1.0
        x, y, z = np.meshgrid(c, c, c, indexing="ij")
        return np.argwhere(np.abs(x) + np.abs(y) + np.abs(z) <= 0.8).astype(np.int16), 5
    rng = np.random.default_rng(7)
    n = 128
    return rng.integers(0, n, (int(0.01 * n ** 3), 3)).astype(np.int16), 7


def rays(level, seed):
    from oracle import oracle as O
    rng = np.random.default_rng(seed)
    os_, ds = [], []
    for origin, target, fov in (([2.6, 1.1, -3.0], [0.05, -0.02, 0.03], 40.0),       # outside, hitting
                                ([2.5, 2.5, 2.5], [4.0, 3.0, 5.0], 30.0),            # outside, looking away: misses
                                ([0.11, 0.23, -0.31], [0.5, -0.2, 0.9], 90.0),       # origin inside the cube
                                ([0.0, 0.0, 1.7], [0.3, 0.1, 3.0], 60.0)):           # past the cube, looking away
        o, d = O.look_at_rays(origin, target, 32, 32, fov)
        os_.append(o); ds.append(d)
    n, h = 1 << level, 2.0 ** (level - 1)
    oa = rng.uniform(-1, 1, (128, 3))
    ax = rng.integers(0, 3, 128)
    for i in range(128):
        for a in range(3):
            if a != ax[i] and (i < 64 or a == (ax[i] + 1) % 3):             # one coordinate on a cell face (an edge for i >= 64)
                oa[i, a] = rng.integers(0, n + 1) / h - 1.0
        oa[i, ax[i]] = rng.choice([-1.5, 1.5])
    da = np.zeros((128, 3), f32)
    da[np.arange(128), ax] = np.where(oa[np.arange(128), ax] < 0, 1.0, -1.0)
    da[1::4] = -da[1::4] + 0.0                                              # a quarter point away from the cube
    os_.append(oa.astype(f32)); ds.append(da)
    return np.concatenate(os_).astype(f32), np.concatenate(ds).astype(f32)


def main():
    warnings.filterwarnings("ignore")
    from oracle import oracle as O, ref_import
    ref_import.install()
    from wisp.core import Rays
    from wisp.models.nefs import SPCField
    from wisp.tracers import PackedSPCTracer
    out = {}
    tracer = PackedSPCTracer()
    for oi, name in enumerate(("octa5", "rand7")):
        pts, level = octree_points(name)
        octree = O.points_to_octree(pts, level)
        M = int(O.octree_to_spc(octree).pyramid[0, level])
        rng = np.random.default_rng(100 + oi)
        colors = rng.integers(0, 256, (M, 4)).astype(np.uint8)
        normals = rng.standard_normal((M, 3))
        normals = (normals / np.linalg.norm(normals, axis=1, keepdims=True)).astype(f32)
        o, d = rays(level, 200 + oi)
        out.update({f"{name}_octree": octree, f"{name}_level": np.int32(level), f"{name}_colors": colors, f"{name}_normals": normals,
                    f"{name}_origins": o, f"{name}_dirs": d})
        r = Rays(origins=torch.from_numpy(o), dirs=torch.from_numpy(d))
        for src, feats in (("rgba", {"colors": torch.from_numpy(colors)}), ("normals", {"normals": torch.from_numpy(normals)}), ("coords", None)):
            nef = SPCField(torch.from_numpy(octree), features_dict=feats, device="cpu")
            out[f"{name}_{src}_field_colors"] = nef.colors.numpy()
            for lod in ((None, 3) if name == "octa5" else (None,)):
                rb = tracer(nef, r, lod_idx=lod)
                key = f"{name}_{src}" + ("" if lod is None else f"_lod{lod}")
                for ch in ("depth", "hit", "rgb", "alpha"):
                    out[f"{key}_{ch}"] = getattr(rb, ch).numpy()
                print(f"{key}: rays={o.shape[0]} hits={int(rb.hit.sum())}")
    np.savez_compressed(OUT, **out)
    print(f"wrote {OUT}")


if __name__ == "__main__":
    main()
