#!/usr/bin/env python
"""Time wisp.ops.mesh.compute_sdf on procedural noisy-sphere meshes (oracle/mesh_shapes.py) of about 20 k, 330 k and 1.3 M triangles,
each with 1 M and 2.5 M points drawn as the SDF datasets draw them (uniform, near-surface and surface points, 1 : 2 : 2):
  native     wisp_b200.compute_sdf: one wb_mesh_sdf call (LBVH build + culled query)
  reference  the reference's kernel (mesh2sdf_gpu_fast_nopre, oracle/_ref/libwisp_ref_mesh2sdf.so from build_ref_mesh.py) when present.
             Its cost is O(N T); above --ref-max-pairs it is timed on a seeded prefix of the points and its per-point time is also
             stated scaled to all N ("ref_ms_scaled", an extrapolation, marked as such).
The arms alternate call by call (CUDA events, median over --reps calls after a warm-up call).  Each arm's peak device memory and the
largest difference between the arms' distances (|sdf|) and the number of sign differences (on the reference's points) are printed.  One JSON line per workload, with the device
name and power limit read in the same run.

    python tools/bench_mesh_sdf.py [--reps 3] [--ref-max-pairs 5e10] [--out FILE]
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
REF_LIB = os.path.join(ROOT, "oracle", "_ref", "libwisp_ref_mesh2sdf.so")
REF_SPLIT = 10 ** 6          # compute_sdf's split_size default


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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--ref-max-pairs", type=float, default=5e10)
    ap.add_argument("--subdiv", type=int, nargs="+", default=[5, 7, 8])
    ap.add_argument("--points", type=int, nargs="+", default=[1_000_000, 2_500_000])
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_mesh_sdf needs a CUDA device"
    import wisp_b200 as W
    from oracle import mesh_shapes as MS
    name, power = _gpu_info()
    print(json.dumps({"device": name, "power_limit": power}), flush=True)
    ref = None
    if os.path.exists(REF_LIB):
        ref = C.CDLL(REF_LIB)
        ref.ref_mesh_last_error.restype = C.c_char_p
    for sd in args.subdiv:
        V, F = MS.noisy_sphere(sd, seed=11)
        Vt, Ft = torch.from_numpy(V).cuda(), torch.from_numpy(F).cuda()
        tris = Vt[Ft].reshape(-1, 9).contiguous()
        T = F.shape[0]
        for N in args.points:
            P = torch.from_numpy(MS.dataset_points(V, F, N, np.random.default_rng(N + sd))).cuda()
            P = P[torch.randperm(N, generator=torch.Generator().manual_seed(1)).cuda()].contiguous()
            n_ref = int(min(N, max(1, args.ref_max_pairs // T)))
            Pr = P[:n_ref].contiguous()

            def native():
                return W.compute_sdf(Vt, Ft, P)

            def reference():
                # in splits of compute_sdf's default split_size: the kernel's int offsets (64 x N x 26 stab bytes) overflow past ~1.3 M
                out = torch.empty(n_ref, dtype=torch.float64, device="cuda")
                for a in range(0, n_ref, REF_SPLIT):
                    n = min(REF_SPLIT, n_ref - a)
                    rc = ref.ref_mesh2sdf(0, C.c_void_p(Pr[a:].data_ptr()), C.c_int64(n), C.c_void_p(tris.data_ptr()), C.c_int64(T),
                                          C.c_void_p(out[a:].data_ptr()))
                    assert rc == 0, ref.ref_mesh_last_error().decode()
                return out

            nat_out, _, nat_mem = timed(native)                  # warm-up
            if ref is not None:
                ref_out, _, ref_mem = timed(reference)
            nat_ms, ref_ms = [], []
            for _ in range(args.reps):
                nat_ms.append(timed(native)[1])
                if ref is not None:
                    ref_ms.append(timed(reference)[1])
            rec = {"triangles": T, "points": N, "native_ms": float(np.median(nat_ms)), "native_ms_all": nat_ms,
                   "native_peak_mem_mb": nat_mem / 2 ** 20, "native_points_per_s": N / (np.median(nat_ms) / 1e3)}
            if ref is not None:
                a, b = nat_out[:n_ref, 0], ref_out
                finite = torch.isfinite(a) & torch.isfinite(b)
                rec.update({"ref_points": n_ref, "ref_ms": float(np.median(ref_ms)), "ref_ms_all": ref_ms,
                            "ref_peak_mem_mb": ref_mem / 2 ** 20,
                            "max_abs_diff_of_distance": float((a.abs() - b.abs())[finite].abs().max()) if finite.any() else 0.0,
                            "inf_mismatch": int((torch.isfinite(a) != torch.isfinite(b)).sum()),
                            "sign_mismatch": int(((a < 0) != (b < 0)).sum()),
                            "bit_identical_frac": float((a == b).double().mean())})
                if n_ref < N:
                    rec["ref_ms_scaled"] = rec["ref_ms"] * N / n_ref
                    rec["ref_ms_scaled_note"] = "extrapolated from ref_points points (the kernel's cost is linear in N)"
                rec["speedup"] = (rec.get("ref_ms_scaled", rec["ref_ms"])) / rec["native_ms"]
            rec.update({"device": name, "power_limit": power})
            print(json.dumps(rec), flush=True)
            if args.out:
                with open(args.out, "a") as f:
                    f.write(json.dumps(rec) + "\n")
            del P, Pr, nat_out
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
