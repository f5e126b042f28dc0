#!/usr/bin/env python
"""Time PackedSPCTracer.trace over a 1024^2 pinhole frame (wb_raygen_pinhole) of procedural sphere-shell SPCs at levels 8 and 10:
  native     ops.spc_trace: one wb_spc_trace launch (first nugget per ray, colour gather, background)
  reference  the reference's algorithm on this package's kernels: OctreeAS.raytrace (count + scan + fill, packed_spc_tracer.py:56) and
             the torch first-hit selection, colour gather and scatters of packed_spc_tracer.py:62-90
on the same rays, the arms alternated window by window (CUDA events, median of the windows).  Exits 1 if the two arms' depth, hit,
rgb or alpha differ.  Prints one JSON line per level with the device name and power limit read in the same run.

    python tools/bench_spc_trace.py [--steps 50] [--warmup 5] [--windows 7]
"""
from __future__ import annotations

import argparse
import json
import math
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SIDE = 1024


def _gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()
        name, power = [s.strip() for s in out[0].split(",")]
        return name, power
    except Exception:                                   # noqa: BLE001 -- the numbers stand without it
        return torch.cuda.get_device_name(), "unknown"


def sphere_shell(W, level, radius=0.7, seed=0):
    """Cells of `level` within about one cell of the sphere |x| = radius, from 24 random surface samples per cell of the shell."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    n = 1 << level
    N = int(24 * 4 * math.pi * (radius * n / 2) ** 2)
    p = torch.nn.functional.normalize(torch.randn(N, 3, device="cuda", generator=g), dim=-1)
    p = p * (radius + (torch.rand(N, 1, device="cuda", generator=g) * 2 - 1) / n)
    return W.spc.points_to_octree(W.spc.quantize_points(p, level), level)


def reference_trace(W, blas, rays, colors, offset):
    """packed_spc_tracer.py:50-90 with OctreeAS.raytrace on this package's kernels and SPCField.rgba's gather."""
    N = rays.origins.shape[0]
    rt = blas.raytrace(rays, blas.max_level, with_exit=False)
    ridx, pidx, depths = rt.ridx, rt.pidx, rt.depth
    first = torch.ones_like(ridx, dtype=torch.bool)
    first[1:] = ridx[1:] != ridx[:-1]
    fp, fr, fd = pidx[first], ridx[first].long(), depths[first]
    color = colors[fp.long() - offset, :3]
    depth = torch.zeros(N, 1, device=fd.device)
    depth[fr, :] = fd
    alpha = torch.ones([color.shape[0], 1], device=color.device)
    hit = torch.zeros(N, device=color.device).bool()
    rgb = torch.zeros(N, 3, device=color.device)
    out_alpha = torch.zeros(N, 1, device=color.device)
    hit[fr] = alpha[..., 0] > 0.0
    rgb[fr, :3] = alpha * color
    out_alpha[fr] = alpha
    return W.RenderBuffer(depth=depth, hit=hit, rgb=rgb, alpha=out_alpha)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--windows", type=int, default=7)
    args = ap.parse_args()
    import wisp_b200 as W
    name, power = _gpu_info()
    pos = np.array([0.0, 0.0, 2.6], np.float32)
    Rm = np.eye(3, dtype=np.float32)
    rays = W.raygen.pinhole_rays(pos, Rm, 45.0, SIDE, SIDE)
    if float(rays.dirs[:, 2].mean()) > 0:                     # the camera looks along +z in its frame: turn it towards the SPC
        rays = W.raygen.pinhole_rays(pos, np.diag([-1.0, 1.0, -1.0]).astype(np.float32), 45.0, SIDE, SIDE)
    ok = True
    for level in (8, 10):
        blas = W.OctreeAS(sphere_shell(W, level))
        M, offset = int(blas.pyramid[0, level]), int(blas.pyramid[1, level])
        colors = torch.rand(M, 3, device="cuda", generator=torch.Generator(device="cuda").manual_seed(level))
        oct = blas.tensors()
        arms = {"native": lambda: W.ops.spc_trace(oct, rays.origins, rays.dirs, level, colors, offset),
                "reference": lambda: reference_trace(W, blas, rays, colors, offset)}
        outs = {k: f() for k, f in arms.items()}
        same = all(torch.equal(getattr(outs["native"], c), getattr(outs["reference"], c)) for c in ("depth", "hit", "rgb", "alpha"))
        ok &= same
        n0 = W._cabi.launch_count()
        arms["native"]()
        launches = {"native": W._cabi.launch_count() - n0}
        n0 = W._cabi.launch_count()
        arms["reference"]()
        launches["reference"] = W._cabi.launch_count() - n0
        for f in arms.values():
            for _ in range(args.warmup):
                f()
        torch.cuda.synchronize()
        ms = {k: [] for k in arms}
        for _ in range(args.windows):
            for k, f in arms.items():
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(args.steps):
                    f()
                e1.record()
                e1.synchronize()
                ms[k].append(e0.elapsed_time(e1) / args.steps)
        nuggets = int(blas.raytrace(rays, level).ridx.shape[0])
        med = {k: float(np.median(v)) for k, v in ms.items()}
        print(json.dumps(dict(workload=f"spc_trace_sphere_shell_level{level}", device=name, power_limit=power, rays=SIDE * SIDE,
                              points=M, hits=int(outs["native"].hit.sum()), nuggets=nuggets, outputs_equal=same,
                              native_ms=round(med["native"], 4), reference_ms=round(med["reference"], 4),
                              speedup=round(med["reference"] / med["native"], 2), library_launches=launches,
                              native_ms_windows=[round(x, 4) for x in ms["native"]],
                              reference_ms_windows=[round(x, 4) for x in ms["reference"]],
                              steps=args.steps, warmup=args.warmup, windows=args.windows)), flush=True)
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
