"""NeuralSDF(HashGrid) on the native SDF route, host side: ops.sdf_field describes hash fields of 4 or 8 features per LOD through
wb_sdf_desc.hash (and declines the others), the library validates that description with wb_make_grid, wb_sdf_train's footprint
query covers hash fields, and wb_sdf_trace refuses them before launching anything.  No device is touched."""
import ctypes as C

import numpy as np
import pytest
import torch

import wisp_b200 as W
from wisp_b200 import _cabi as A
from wisp_b200 import ops


def _hash_sdf(F=8, ms='cat', L=4, bw=10, rmin=4, rmax=32, pos='none', pin=True, H=32, nh=1):
    blas = W.OctreeAS.make_dense(3, device="cpu")
    torch.manual_seed(0)
    grid = W.HashGrid.from_geometric(blas, feature_dim=F, num_lods=L, multiscale_type=ms, feature_std=0.1, codebook_bitwidth=bw,
                                     min_grid_res=rmin, max_grid_res=rmax)
    return W.NeuralSDF(grid, pos_embedder=pos, pos_multires=4, position_input=pin, hidden_dim=H, num_layers=nh)


@pytest.mark.parametrize("F,ms", [(8, 'cat'), (4, 'sum'), (4, 'cat'), (8, 'sum')])
def test_sdf_field_describes_hash_fields(F, ms):
    nef = _hash_sdf(F=F, ms=ms)
    fd = ops.sdf_field(nef)
    assert fd is not None
    d, oct, keep = fd
    assert oct is None and not d.points and not d.trinkets and not d.feats
    assert (d.feature_dim, d.num_lods, d.multiscale, d.base_lod, d.pos_mode) == (F, 4, int(ms == 'sum'), 0, 1)
    h = d.hash.contents
    g = nef.grid
    assert (h.num_lods, h.feature_dim, h.codebook_size, h.multiscale, h.grid_kind) == (4, F, 2 ** 10, int(ms == 'sum'), 0)
    assert [h.resolutions[l] for l in range(4)] == [int(r) for r in g.resolutions]
    assert [h.begin_idxes[l] for l in range(5)] == g.codebook.begin_idxes.tolist()
    assert h.table == g.codebook.feats.data_ptr()                  # the parameter itself: SDFStep trains it in place
    assert d.params == keep[-1].data_ptr()
    assert ops.sdf_train_smem_bytes(fd) > 0


def test_sdf_field_declines_hash_fields_outside_the_native_range():
    assert ops.sdf_field(_hash_sdf(F=2)) is None                  # 8-byte rows: the nglod_nerf-style table keeps autograd
    blas = W.OctreeAS.make_dense(3, device="cpu")
    grid = W.HashGrid.from_geometric(blas, feature_dim=16, num_lods=2, multiscale_type='sum', codebook_bitwidth=10, min_grid_res=4, max_grid_res=8)
    assert ops.sdf_field(W.NeuralSDF(grid, hidden_dim=16)) is None


def test_hash_training_footprint_boundary():
    """The one formula of wb_sdf_train_smem_bytes covers hash fields: 2 layers of 64 fit, 3 layers of 128 do not."""
    assert ops.sdf_train_smem_bytes(ops.sdf_field(_hash_sdf(H=64, nh=2))) > 0
    assert ops.sdf_train_smem_bytes(ops.sdf_field(_hash_sdf(H=128, nh=3))) < 0


def _refused_eval(d) -> str:
    """wb_sdf_eval of the description fails with WB_ERR_INVALID: -> its message."""
    c = torch.zeros(4, 3)
    out = torch.zeros(4, 1)
    with pytest.raises(A.WispB200Error) as e:
        A.lib().wb_sdf_eval(None, d, d.num_lods - 1, A.ptr(c), 4, A.ptr(out), None)
    assert e.value.status == -1
    return str(e.value)


def test_hash_description_refusals_raise():
    d, _, keep = ops.sdf_field(_hash_sdf())
    bad = A.make_grid_desc(keep[1], [4, 8, 16, 32], [0] * 5, 1000)        # not a power of two: wb_make_grid refuses it
    d.hash = C.pointer(bad)
    assert "power of two" in _refused_eval(d)
    d, _, keep = ops.sdf_field(_hash_sdf())
    d.feature_dim = 4                                              # disagrees with the hash description
    assert "hash field" in _refused_eval(d)
    d, _, keep = ops.sdf_field(_hash_sdf())
    h2 = A.make_grid_desc(torch.zeros(64, 2), [4, 8, 16, 32], [0, 16, 32, 48, 64], 2 ** 10)
    d.hash, d.feature_dim = C.pointer(h2), 2                       # F = 2: outside the native range
    assert "4 or 8" in _refused_eval(d)


def test_sdf_trace_raises_on_hash_fields():
    d, _, keep = ops.sdf_field(_hash_sdf())
    rays = A.RaysDesc()
    rays.num_rays = 1
    st = A.SdfState()
    with pytest.raises(A.WispB200Error, match="phase by phase") as e:
        A.lib().wb_sdf_trace(None, d, 3, rays, None, 1, None, 8, 1.0, 1e-4, 0, st, None, None, None, None, None, None, None)
    assert e.value.status == -1


def test_sdf_step_hash_needs_a_device():
    with pytest.raises(W.WispB200Error):
        W.SDFStep(W.Pipeline(_hash_sdf()))
