"""GPU tests (-m gpu) against the REFERENCE's OWN CUDA kernels:
    hashgrid_interpolate_cuda / _backward_cuda  (A14)      uniform_sample_cuda  (A8)      find_depth_bound_cuda  (B1)
Their results on the inputs built by oracle/make_ref_golden.py were stored once in tests/golden/ref_kernels.npz (the recipe compiles the
kernels from a kaolin-wisp checkout with oracle/ref_kernels/build_ref.py and runs them on the GPU).  This pins those three operators to
the code they replace, not to a restatement of it."""
import os

import numpy as np
import pytest
import torch

from oracle import make_ref_golden as RG

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def golden(golden_dir):
    return dict(np.load(os.path.join(golden_dir, "ref_kernels.npz")))


@pytest.fixture(scope="module")
def W():
    import wisp_b200
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    return wisp_b200


@pytest.mark.parametrize("F", [2, 4])
def test_hashgrid_kernels_vs_reference_cuda(W, golden, F):
    """wb_hashgrid_fwd / _bwd (one launch, all LODs) vs wisp._C.ops.hashgrid_interpolate_cuda / _backward_cuda (one launch per LOD):
    dense and hashed levels, points on cell faces and at the +-1 borders.  Forward: same arithmetic -> 2 ulp-level agreement;
    backward: same products, different atomic order."""
    grid, coords, go = RG.hashgrid_case(W, F)
    L_, bw = len(grid.resolutions), grid.codebook_bitwidth
    mine = W.ops.hashgrid(coords, bw, L_ - 1, grid.codebook)
    got = mine.detach().cpu().numpy().reshape(-1)
    ref = golden[f"hashgrid{F}_feats"]
    err = float(np.abs(got[RG.sample_index(got.size, 10 + F)] - ref).max())
    assert err <= 2e-6 * float(golden[f"hashgrid{F}_feats_absmax"]), err
    grid.codebook.feats.grad = None
    mine.backward(go)
    gt = grid.codebook.feats.grad.cpu().numpy().reshape(-1)
    gerr = float(np.abs(gt[RG.sample_index(gt.size, 20 + F)] - golden[f"hashgrid{F}_grad"]).max())
    assert gerr <= 2e-5 * float(golden[f"hashgrid{F}_grad_absmax"]), gerr


def test_uniform_sampler_vs_reference_cuda(W, golden):
    """OctreeAS._raymarch_uniform: wb_raymarch_uniform_{count,fill} vs the reference's uniform_sample_cuda kernel fed as
    octree_as.py:340-357 feeds it (zero-count nuggets filtered, inclusive sum): ridx, depth samples and boundary bit-exact."""
    mr, scale, ridx_f, depth_f, insum = RG.uniform_case(W)
    total = int(insum[-1])
    assert total == mr.ridx.shape[0] == int(golden["uniform_total"]) > 1000
    got = RG.digest(mr.ridx.cpu().numpy(), mr.depth_samples[:, 0].contiguous().cpu().numpy(), mr.boundary.cpu().numpy())
    assert got == str(golden["uniform_sha256"])


def test_find_depth_bound_vs_reference_cuda(W, golden):
    """wb_find_depth_bound vs find_depth_bound_cuda (cursor kernel of the SDF tracer), quirks included."""
    q, curr, depth = RG.depth_bound_case()
    tq, tc, td = torch.from_numpy(q).cuda(), torch.from_numpy(curr).cuda(), torch.from_numpy(depth).cuda()
    mine = W.ops.find_depth_bound(tq[:, None], td, curr_idxes=tc)
    assert np.array_equal(mine.cpu().numpy(), golden["depth_bound"])
