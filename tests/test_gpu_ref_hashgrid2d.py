"""GPU tests (-m gpu) of the 2-D hash-grid kernels (wb_hashgrid2d_fwd / _bwd, app/image) against the REFERENCE's OWN 2-D CUDA kernels
(hashgrid_interpolate_2d_cuda_kernel and its backward, hashgrid_interpolate_cuda.cu:214-339).  Their results on the inputs built by
oracle/make_ref_golden2d.py (hashgrid2d_case) were stored once in tests/golden/ref_hashgrid2d.npz (python -m oracle.make_ref_golden2d, on
the GPU, with the kernels compiled from a kaolin-wisp checkout by oracle/ref_kernels/build_ref.py and build_ref2d.py)."""
import os

import numpy as np
import pytest
import torch

from oracle import make_ref_golden2d as RG2
from oracle.make_ref_golden import sample_index

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def golden():
    return dict(np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_hashgrid2d.npz")))


@pytest.fixture(scope="module")
def W():
    import wisp_b200
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return wisp_b200


@pytest.mark.parametrize("F,cd", RG2.CASES)
def test_hashgrid2d_kernels_vs_reference_cuda(W, golden, F, cd):
    """ops.hashgrid on [N, 2] (what install() patches into wisp.ops.grid) vs the reference's 2-D kernels, one launch per LOD: dense and
    hashed levels, cell lines and the +-1 borders, tables of coord_dim 3 (image_hash.yaml) and 2.  Forward: the same arithmetic
    (prints how many sampled features are bit-identical); backward: the same products in another atomic order."""
    grid, coords, go = RG2.hashgrid2d_case(W, F, cd)
    L_, bw = len(grid.resolutions), grid.codebook_bitwidth
    k = f"hashgrid2d_F{F}_cd{cd}"
    mine = W.ops.hashgrid(coords, bw, L_ - 1, grid.codebook)
    got = mine.detach().cpu().numpy().reshape(-1)[sample_index(mine.numel(), 30 + F)]
    ref = golden[f"{k}_feats"]
    err = float(np.abs(got - ref).max())
    print(f"REFHASH2D F={F} coord_dim={cd}: {int((got == ref).sum())}/{ref.size} sampled features bit-identical, max err {err:.3e}")
    assert err <= 2e-6 * float(golden[f"{k}_feats_absmax"]), err
    grid.codebook.feats.grad = None
    mine.backward(go)
    gt = grid.codebook.feats.grad.cpu().numpy().reshape(-1)
    gerr = float(np.abs(gt[sample_index(gt.size, 40 + F)] - golden[f"{k}_grad"]).max())
    assert gerr <= 2e-5 * float(golden[f"{k}_grad_absmax"]), gerr
