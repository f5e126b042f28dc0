"""Inputs of tests/test_gpu_ref_kernels.py, and the recipe that stores what the reference's OWN CUDA operators return for them.

    python -m oracle.make_ref_golden [OUT]   (needs oracle/_ref/libwisp_ref_kernels.so from oracle/ref_kernels/build_ref.py and a CUDA device)

writes tests/golden/ref_kernels.npz (or OUT).  The tests then compare the product's kernels with those stored results and need neither the
reference checkout nor its library.  Outputs that the tests compare bit for bit are stored as SHA-256 digests of their bytes; the
hash-grid results (compared within a tolerance) as a fixed, seeded sample of entries, which keeps the file small.
"""
import ctypes as C
import hashlib
import os

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_LIB = os.path.join(ROOT, "oracle", "_ref", "libwisp_ref_kernels.so")
GOLDEN = os.path.join(ROOT, "tests", "golden", "ref_kernels.npz")
HASHGRID_N = 200_000
SAMPLE = 8192           # stored entries of each hash-grid output


def digest(*arrays) -> str:
    h = hashlib.sha256()
    for a in arrays:
        h.update(np.ascontiguousarray(a).tobytes())
    return h.hexdigest()


def sample_index(size: int, seed: int) -> np.ndarray:
    return np.sort(np.random.default_rng(seed).choice(size, size=min(SAMPLE, size), replace=False))


def hashgrid_case(W, F):
    """Dense and hashed levels, points on cell faces and at the +-1 borders; inputs drawn on the host from fixed seeds."""
    import torch
    torch.manual_seed(0)
    blas = W.OctreeAS.make_dense(3, device="cuda")
    grid = W.HashGrid.from_geometric(blas, feature_dim=F, num_lods=12, multiscale_type='cat', feature_std=1.0, codebook_bitwidth=14,
                                     min_grid_res=8, max_grid_res=300).cuda()
    g = torch.Generator().manual_seed(1)
    coords = torch.rand(HASHGRID_N, 3, generator=g) * 2 - 1
    coords[:1000] = torch.round(coords[:1000] * 8) / 8                    # exact cell faces of the coarse levels
    coords[1000:1100] = torch.sign(coords[1000:1100])                     # corners / borders of the unit cube
    go = torch.randn(HASHGRID_N, len(grid.resolutions) * F, generator=g)
    return grid, coords.cuda(), go.cuda()


def uniform_case(W):
    """OctreeAS._raymarch_uniform inputs fed as octree_as.py:340-357 feeds uniform_sample_cuda (zero-count nuggets filtered, inclusive sum)."""
    import torch
    from oracle import oracle as O
    blas = W.OctreeAS.from_quantized_points(torch.from_numpy(O.lego_like_points(6)).cuda(), 6)
    o, d = O.look_at_rays([-3.0, 0.65, -3.0], [0, 0, 0], 96, 96, 30.0)
    rays = W.Rays(torch.from_numpy(o).cuda(), torch.from_numpy(d).cuda(), 0.0, 10.0)
    n = 256
    mr = blas.raymarch(rays, 'uniform', n, 6)
    rt = blas.raytrace(rays, 6, with_exit=True)
    scale = W.ops.uniform_scale(n)
    depth = rt.depth.contiguous()
    cnt = (torch.ceil(scale * depth[:, 1]) - torch.ceil(scale * depth[:, 0])).int()          # octree_as.py:343-345
    nz = cnt > 0
    ridx_f, depth_f = rt.ridx[nz].contiguous(), depth[nz].contiguous()
    insum = torch.cumsum(cnt[nz], 0).int().contiguous()
    return mr, scale, ridx_f, depth_f, insum


def depth_bound_case():
    rng = np.random.default_rng(3)
    P = 5000
    counts = rng.integers(1, 6, P); offs = np.concatenate([[0], np.cumsum(counts)]).astype(np.int32)
    Ng = int(offs[-1])
    en = np.sort(rng.random(Ng) * 5).astype(np.float32); depth = np.stack([en, en + 0.01 + rng.random(Ng).astype(np.float32) * 0.05], -1).astype(np.float32)
    curr = offs[:-1].copy(); curr[::13] = -1
    q = (rng.random(P) * 5).astype(np.float32)
    return q, curr, depth


def main(path=GOLDEN):
    import torch
    import wisp_b200 as W
    L = C.CDLL(REF_LIB)
    L.ref_last_error.restype = C.c_char_p
    p = lambda t: C.c_void_p(t.data_ptr())

    def chk(rc):
        assert rc == 0, L.ref_last_error().decode()
    out = {}
    for F in (2, 4):
        grid, coords, go = hashgrid_case(W, F)
        table = grid.codebook.feats.detach().contiguous()
        L_, bw = len(grid.resolutions), grid.codebook_bitwidth
        first = grid.codebook.begin_idxes.to("cuda").contiguous()
        res_host = (C.c_int64 * L_)(*grid.resolutions)
        feats = torch.empty(HASHGRID_N, L_ * F, device="cuda")
        chk(L.ref_hashgrid_fwd(0, p(coords), C.c_int64(HASHGRID_N), p(table), C.c_int64(table.shape[0]), F, p(first), L_, res_host, bw, p(feats)))
        gt = torch.zeros_like(table)
        chk(L.ref_hashgrid_bwd(0, p(coords), C.c_int64(HASHGRID_N), p(go), p(table), C.c_int64(table.shape[0]), F, p(first), L_, res_host, bw, p(gt)))
        torch.cuda.synchronize()
        feats, gt = feats.cpu().numpy().reshape(-1), gt.cpu().numpy().reshape(-1)
        out[f"hashgrid{F}_feats"] = feats[sample_index(feats.size, 10 + F)]
        out[f"hashgrid{F}_feats_absmax"] = np.float32(np.abs(feats).max())
        out[f"hashgrid{F}_grad"] = gt[sample_index(gt.size, 20 + F)]
        out[f"hashgrid{F}_grad_absmax"] = np.float32(np.abs(gt).max())
    mr, scale, ridx_f, depth_f, insum = uniform_case(W)
    V, total = int(ridx_f.shape[0]), int(insum[-1])
    r_ridx = torch.empty(total, dtype=torch.int64, device="cuda"); r_depth = torch.empty(total, device="cuda"); r_b = torch.empty(total, dtype=torch.bool, device="cuda")
    chk(L.ref_uniform_sample(0, scale, p(ridx_f), p(depth_f), p(insum), C.c_int64(V), C.c_int64(total), p(r_ridx), p(r_depth), p(r_b)))
    torch.cuda.synchronize()
    out["uniform_total"] = np.int64(total)
    out["uniform_sha256"] = np.array(digest(r_ridx.cpu().numpy(), r_depth.cpu().numpy(), r_b.cpu().numpy()))
    q, curr, depth = depth_bound_case()
    tq, tc, td = torch.from_numpy(q).cuda(), torch.from_numpy(curr).cuda(), torch.from_numpy(depth).cuda()
    ob = torch.empty(q.shape[0], dtype=torch.int32, device="cuda")
    chk(L.ref_find_depth_bound(0, p(tq), p(tc), p(td), C.c_int64(q.shape[0]), C.c_int64(depth.shape[0]), p(ob)))
    torch.cuda.synchronize()
    out["depth_bound"] = ob.cpu().numpy()
    os.makedirs(os.path.dirname(os.path.abspath(path)), exist_ok=True)
    np.savez_compressed(path, **out)
    print("wrote", path, {k: v.shape for k, v in out.items()})


if __name__ == "__main__":
    import sys
    main(*sys.argv[1:2])
