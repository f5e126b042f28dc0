"""The recipe that stores what the reference's OWN wisp.ops.spc.mesh_to_octree (conversions.py:91-109: sample_surface, the jittered
copies, quantize_points, unbatched_points_to_octree) returns on the procedural meshes of oracle/mesh_shapes.py.

    python -m oracle.make_ref_golden_mesh_octree [OUT]      (needs the reference checkout; runs on the CPU)

The unmodified reference function runs through oracle/ref_import.py.  During each call Tensor.cuda is the identity (the sampler runs on
the CPU with torch's CPU generator), Kaolin's quantize_points is this package's spc.quantize_points (Kaolin's rule), and
unbatched_points_to_octree is the oracle's.  Vertices are float32, as OctreeAS.from_mesh passes them.

Writes tests/golden/ref_mesh_octree.npz (or OUT): per mesh <mesh>_V (float32) and <mesh>_F (uint16); per case <mesh>_L<level> the
octree bytes of torch seeds 0..3 at num_samples N[level] (uint8 arrays <case>_s<seed>).
"""
import os
import sys
import time

import numpy as np

from . import mesh_shapes as MS

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "ref_mesh_octree.npz")
SEEDS = (0, 1, 2, 3)
N = {5: 2 * 10 ** 5, 7: 10 ** 6}                   # num_samples per level


def meshes():
    return {"noisy_sphere": MS.noisy_sphere(3), "torus": MS.torus(), "cube": MS.cube(), "open": MS.open_mesh()}


def reference_mesh_to_octree():
    """-> f(vertices, faces, level, num_samples, seed): the reference's mesh_to_octree on the CPU after torch.manual_seed(seed)."""
    import torch
    from . import ref_import
    ref_import.install()
    sys.path.insert(0, ROOT)
    import kaolin.ops.spc as kaolin_spc
    import wisp.ops.spc as wisp_spc
    from wisp_b200 import spc as S

    def run(V, F, level, n, seed):
        cuda, quant = torch.Tensor.cuda, getattr(kaolin_spc, "quantize_points", None)
        torch.Tensor.cuda = lambda self, *a, **k: self
        kaolin_spc.quantize_points = S.quantize_points
        try:
            torch.manual_seed(seed)
            return wisp_spc.mesh_to_octree(torch.from_numpy(V), torch.from_numpy(F), level, n).numpy().astype(np.uint8)
        finally:
            torch.Tensor.cuda = cuda
            kaolin_spc.quantize_points = quant
    return run


def main(path=GOLDEN):
    run = reference_mesh_to_octree()
    out = {}
    for name, (V, F) in meshes().items():
        V32 = V.astype(np.float32)
        out[f"{name}_V"], out[f"{name}_F"] = V32, F.astype(np.uint16)
        for level, n in N.items():
            t = time.time()
            for seed in SEEDS:
                out[f"{name}_L{level}_s{seed}"] = run(V32, F.astype(np.int64), level, n, seed)
            print(name, "level", level, "n", n, "octree bytes", [out[f"{name}_L{level}_s{s}"].size for s in SEEDS],
                  f"{time.time() - t:.1f} s", flush=True)
    os.makedirs(os.path.dirname(os.path.abspath(path)), exist_ok=True)
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main(*sys.argv[1:2])
