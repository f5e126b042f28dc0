"""SDFStep without a GPU: the numpy restatement of NeuralSDF.sdf reproduces the reference trainer's step-1 loss
(tests/golden/sdf_train.npz), and SDFStep refuses host tensors (there is no CPU fallback)."""
import os

import numpy as np
import pytest
import torch

from oracle import octree_grid as OG
from oracle import oracle as O


@pytest.mark.parametrize("case", ["sum", "cat", "sum_all"])
def test_neural_sdf_oracle_reproduces_golden_loss(golden_dir, case):
    g = np.load(os.path.join(golden_dir, "sdf_train.npz"))
    level = int(g["level"])
    spc = O.octree_to_spc(g["octree"])
    _, pyr, trinkets, _ = OG.make_trilinear_spc(spc)
    sdf_case = dict(spc=spc, trinkets=trinkets, active_lods=[level - 2, level - 1, level], multiscale=str(g[f"{case}_multiscale"]),
                    feats=[g[f"{case}_init_grid.features.{k}"] for k in range(3)],
                    W=[g[f"{case}_init_decoder.layers.0.weight"], g[f"{case}_init_decoder.lout.weight"]],
                    b=[g[f"{case}_init_decoder.layers.0.bias"], g[f"{case}_init_decoder.lout.bias"]])
    coords, sdf = g["coords"], g["sdf"]
    loss = sum(float(((OG.neural_sdf(sdf_case, coords, int(lod)).astype(np.float64) - sdf) ** 2).sum()) for lod in g[f"{case}_loss_lods"])
    loss /= coords.shape[0]
    assert abs(loss - g[f"{case}_losses"][0]) <= 1e-5 * g[f"{case}_losses"][0], (loss, g[f"{case}_losses"][0])


def test_sdf_step_needs_a_device():
    import wisp_b200 as W
    from oracle.make_golden import octahedron_points
    blas = W.OctreeAS(torch.from_numpy(O.points_to_octree(octahedron_points(4), 4)))
    grid = W.OctreeGrid(blas, feature_dim=4, num_lods=2, multiscale_type='sum', feature_std=0.1)
    nef = W.NeuralSDF(grid, pos_embedder='none', position_input=True, hidden_dim=8, num_layers=1)
    with pytest.raises(W.WispB200Error):
        W.SDFStep(W.Pipeline(nef))
