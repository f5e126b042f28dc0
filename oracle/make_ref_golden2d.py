"""Inputs of tests/test_gpu_ref_hashgrid2d.py, and the recipe that stores what the reference's OWN 2-D hash-grid kernels (app/image)
return for them.

    python -m oracle.make_ref_golden2d [OUT]   (needs oracle/_ref/libwisp_ref_hashgrid2d.so from oracle/ref_kernels/build_ref2d.py and a
                                                CUDA device)

writes tests/golden/ref_hashgrid2d.npz (or OUT): for each case a fixed, seeded sample of the features and of the table gradient
(oracle/make_ref_golden.py's sampling), with their largest magnitudes.
"""
import ctypes as C
import os

import numpy as np

from .make_ref_golden import HASHGRID_N, ROOT, sample_index

REF_LIB = os.path.join(ROOT, "oracle", "_ref", "libwisp_ref_hashgrid2d.so")
GOLDEN = os.path.join(ROOT, "tests", "golden", "ref_hashgrid2d.npz")
CASES = ((2, 3), (4, 2))          # (F, coord_dim): image_hash.yaml's table layout, and a coord_dim = 2 table


def hashgrid2d_case(W, F, coord_dim):
    """[N, 2] coordinates over a 'cat' grid whose table has coord_dim-shaped levels (min(res^coord_dim, T) rows): dense levels below
    res 128 (res^2 < 2^14), hashed above, points on the cell lines of the coarse levels and at the +-1 borders."""
    import torch
    torch.manual_seed(0)
    grid = W.HashGrid.from_geometric(None, feature_dim=F, num_lods=10, multiscale_type='cat', feature_std=1.0, codebook_bitwidth=14,
                                     min_grid_res=8, max_grid_res=600, coord_dim=coord_dim).cuda()
    g = torch.Generator().manual_seed(2)
    coords = torch.rand(HASHGRID_N, 2, generator=g) * 2 - 1
    coords[:1000] = torch.round(coords[:1000] * 8) / 8
    coords[1000:1100] = torch.sign(coords[1000:1100])
    go = torch.randn(HASHGRID_N, len(grid.resolutions) * F, generator=g)
    return grid, coords.cuda(), go.cuda()


def main(path=GOLDEN):
    import torch
    import wisp_b200 as W
    L = C.CDLL(REF_LIB)
    L.ref2d_last_error.restype = C.c_char_p
    p = lambda t: C.c_void_p(t.data_ptr())

    def chk(rc):
        assert rc == 0, L.ref2d_last_error().decode()
    out = {}
    for F, cd in CASES:
        grid, coords, go = hashgrid2d_case(W, F, cd)
        table = grid.codebook.feats.detach().contiguous()
        L_, bw = len(grid.resolutions), grid.codebook_bitwidth
        first = grid.codebook.begin_idxes.to("cuda").contiguous()
        res_host = (C.c_int64 * L_)(*grid.resolutions)
        feats = torch.empty(HASHGRID_N, L_ * F, device="cuda")
        chk(L.ref_hashgrid2d_fwd(0, p(coords), C.c_int64(HASHGRID_N), p(table), C.c_int64(table.shape[0]), F, p(first), L_, res_host, bw, p(feats)))
        gt = torch.zeros_like(table)
        chk(L.ref_hashgrid2d_bwd(0, p(coords), C.c_int64(HASHGRID_N), p(go), p(table), C.c_int64(table.shape[0]), F, p(first), L_, res_host, bw, p(gt)))
        torch.cuda.synchronize()
        feats, gt = feats.cpu().numpy().reshape(-1), gt.cpu().numpy().reshape(-1)
        k = f"hashgrid2d_F{F}_cd{cd}"
        out[f"{k}_feats"] = feats[sample_index(feats.size, 30 + F)]
        out[f"{k}_feats_absmax"] = np.float32(np.abs(feats).max())
        out[f"{k}_grad"] = gt[sample_index(gt.size, 40 + F)]
        out[f"{k}_grad_absmax"] = np.float32(np.abs(gt).max())
    os.makedirs(os.path.dirname(os.path.abspath(path)), exist_ok=True)
    np.savez_compressed(path, **out)
    print("wrote", path, {k: v.shape for k, v in out.items()})


if __name__ == "__main__":
    import sys
    main(*sys.argv[1:2])
