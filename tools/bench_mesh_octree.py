#!/usr/bin/env python
"""Time wisp.ops.spc.mesh_to_octree (OctreeAS.from_mesh's octree, app/nglod's nglod_octree / nglod_hash blas) at level 7 and 10^8
surface samples on procedural noisy-sphere meshes (oracle/mesh_shapes.py) of about 20 k, 330 k and 1.3 M triangles:
  native     wisp_b200.mesh_to_octree: one wb_mesh_octree_bits launch into a dense bitmask, then spc.points_to_octree of the set cells
  reference  the reference's algorithm restated op by op in torch on the device (sample_surface's area_weighted_distribution /
             Categorical sample, its two host torch.rand calls copied to the device, the V[F[idx]] gathers, the jittered copies and the
             cat, quantize_points), with this package's spc.points_to_octree in place of Kaolin's
The arms alternate call by call (CUDA events, median over --reps calls after a warm-up call of each).  Each arm's peak device memory
and both arms' finest-level cell counts are printed, one JSON line per mesh, with the device name and power limit read in the same run.

    python tools/bench_mesh_octree.py [--reps 3] [--samples 100000000] [--level 7] [--out FILE]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()
        name, power = [s.strip() for s in out[0].split(",")]
        return name, power
    except Exception:                                   # noqa: BLE001 -- the numbers stand without it
        return torch.cuda.get_device_name(), "unknown"


def timed(fn):
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    out = fn()
    e1.record()
    torch.cuda.synchronize()
    return out, e0.elapsed_time(e1), torch.cuda.max_memory_allocated() - base


def reference(V, F, level, n):
    """conversions.py:91-109 with sample_surface (sample_surface.py, random_face.py, area_weighted_distribution.py) written out."""
    from wisp_b200 import spc as S
    mesh = V[F]
    normals = torch.cross(mesh[:, 0] - mesh[:, 1], mesh[:, 1] - mesh[:, 2], dim=1)
    areas = torch.norm(normals, p=2, dim=1) * 0.5
    areas /= torch.sum(areas) + 1e-10
    idx = torch.distributions.Categorical(areas.view(-1)).sample([n])
    f = V[F[idx]]
    u = torch.sqrt(torch.rand(n)).to(V.device).unsqueeze(-1)
    v = torch.rand(n).to(V.device).unsqueeze(-1)
    samples = (1 - u) * f[:, 0, :] + (u * (1 - v)) * f[:, 1, :] + u * v * f[:, 2, :]
    del f
    samples = torch.cat([samples, samples + (torch.rand_like(samples) * 2.0 - 1.0) * (1.0 / (2 ** (level + 1)))], dim=0)
    return S.points_to_octree(S.quantize_points(samples, level), level)


def cells(octree, level):
    from wisp_b200 import spc as S
    _, pyramid, _ = S.scan_octree(octree)
    return int(pyramid[0, level])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--samples", type=int, default=10 ** 8)
    ap.add_argument("--level", type=int, default=7)
    ap.add_argument("--subdiv", type=int, nargs="+", default=[5, 7, 8])
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_mesh_octree needs a CUDA device"
    import wisp_b200 as W
    from oracle import mesh_shapes as MS
    name, power = _gpu_info()
    print(json.dumps({"device": name, "power_limit": power}), flush=True)
    n, level = args.samples, args.level
    for sd in args.subdiv:
        V, F = MS.noisy_sphere(sd, seed=11)
        Vt, Ft = torch.from_numpy(V.astype(np.float32)).cuda(), torch.from_numpy(F).cuda()
        nat = lambda: W.mesh_to_octree(Vt, Ft, level, n)
        ref = lambda: reference(Vt, Ft, level, n)
        nat_out, _, nat_mem = timed(nat)                  # warm-up
        ref_out, _, ref_mem = timed(ref)
        nat_ms, ref_ms = [], []
        for _ in range(args.reps):
            nat_ms.append(timed(nat)[1])
            ref_ms.append(timed(ref)[1])
        rec = {"triangles": F.shape[0], "level": level, "samples": n,
               "native_ms": float(np.median(nat_ms)), "native_ms_all": nat_ms, "native_peak_mem_mb": nat_mem / 2 ** 20,
               "native_cells": cells(nat_out, level),
               "ref_ms": float(np.median(ref_ms)), "ref_ms_all": ref_ms, "ref_peak_mem_mb": ref_mem / 2 ** 20,
               "ref_cells": cells(ref_out, level),
               "speedup": float(np.median(ref_ms)) / float(np.median(nat_ms)), "device": name, "power_limit": power}
        print(json.dumps(rec), flush=True)
        if args.out:
            with open(args.out, "a") as f:
                f.write(json.dumps(rec) + "\n")
        del nat_out, ref_out
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
