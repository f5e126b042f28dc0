"""The recipe that stores what the reference's OWN mesh-to-SDF kernel (mesh2sdf_gpu_fast_nopre, behind wisp.ops.mesh.compute_sdf)
returns on the procedural meshes and seeded points of oracle/mesh_shapes.py.

    python -m oracle.make_ref_golden_mesh [OUT]   (needs oracle/_ref/libwisp_ref_mesh2sdf.so from oracle/ref_kernels/build_ref_mesh.py
                                                   and a CUDA device)

writes tests/golden/ref_mesh_sdf.npz (or OUT): per case <name>_V (float64), <name>_F (uint16), <name>_points (float64, the only
dtype the reference takes) and <name>_sdf (its result: +-sqrtf of an fp32 minimum or inf, so stored exactly as float32); plus
f32_error, the message the reference raises when it is given the float32 tensors wisp's SDF datasets pass it (empty when it accepts
them).  The reference runs on every point golden_points draws; a seeded subset of KEEP points per case is stored, which keeps the file
under 1 MB (each point's result depends on that point alone).
"""
import ctypes as C
import os

import numpy as np

from . import mesh_shapes as MS

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_LIB = os.path.join(ROOT, "oracle", "_ref", "libwisp_ref_mesh2sdf.so")
GOLDEN = os.path.join(ROOT, "tests", "golden", "ref_mesh_sdf.npz")
KEEP = {"noisy_sphere": 4000}           # stored points per case (2000 for the others)


def store(out, name, case_seed, V, F, pts, sdf):
    """Put one case's seeded subset of points, compacted without loss, into `out`."""
    keep = np.sort(np.random.default_rng(1000 + case_seed).choice(pts.shape[0], KEEP.get(name, 2000), replace=False))
    sdf32 = sdf[keep].astype(np.float32)
    assert np.array_equal(sdf32.astype(np.float64), sdf[keep]) and F.max() < 2 ** 16
    out[f"{name}_V"], out[f"{name}_F"], out[f"{name}_points"], out[f"{name}_sdf"] = V, F.astype(np.uint16), pts[keep], sdf32


def main(path=GOLDEN):
    import torch
    L = C.CDLL(REF_LIB)
    L.ref_mesh_last_error.restype = C.c_char_p
    p = lambda t: C.c_void_p(t.data_ptr())
    out = {}
    for seed, (name, ((V, F), counts)) in enumerate(MS.golden_cases().items()):
        pts = MS.golden_points(name, V, F, counts, seed=100 + seed)
        tris = torch.from_numpy(V[F].reshape(-1, 9)).cuda().contiguous()
        pt = torch.from_numpy(pts).cuda().contiguous()
        sdf = torch.empty(pts.shape[0], dtype=torch.float64, device="cuda")
        rc = L.ref_mesh2sdf(0, p(pt), C.c_int64(pt.shape[0]), p(tris), C.c_int64(tris.shape[0]), p(sdf))
        assert rc == 0, L.ref_mesh_last_error().decode()
        store(out, name, seed, V, F, pts, sdf.cpu().numpy())
        print(name, F.shape[0], "triangles", pts.shape[0], "points", "inside", int((sdf < 0).sum()), "stored", out[f"{name}_sdf"].size)
    V, F = MS.icosphere(1)
    tris32 = torch.from_numpy(V[F].reshape(-1, 9)).float().cuda().contiguous()
    pts32 = torch.zeros(4, 3, device="cuda")
    rc = L.ref_mesh2sdf_f32(0, p(pts32), C.c_int64(4), p(tris32), C.c_int64(tris32.shape[0]))
    out["f32_error"] = np.array(L.ref_mesh_last_error().decode().splitlines()[0] if rc != 0 else "")
    print("float32 inputs:", "refused: " + str(out["f32_error"]) if rc != 0 else "accepted")
    os.makedirs(os.path.dirname(os.path.abspath(path)), exist_ok=True)
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    import sys
    main(*sys.argv[1:2])
