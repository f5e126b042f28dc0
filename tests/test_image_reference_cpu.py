"""CPU checks of the app/image reference (tests/image_reference.py) and of the host side of the app/image route: the float64 chain
equals torch float64 autograd, fp32 torch autograd lies inside the intervals, the 2-D rows never leave their level, and the mirror
classes accept what the reference accepts (HashGrid coord_dim 2, ImageNeuralField's names and widths), and the restatement reproduces
the reference trainer's first step (tests/golden/image_step.npz)."""
import os

import numpy as np
import pytest
import torch

import image_reference as IR
import wisp_b200 as W


def make_case(coord_dim=3, F=2, L=4, bw=10, min_res=4, max_res=48, H=16, multiscale="cat", N=300, seed=0, std=0.5):
    rng = np.random.default_rng(seed)
    b = np.exp((np.log(max_res) - np.log(min_res)) / (L - 1)) if L > 1 else 1.0
    res = [int(np.floor(min_res * b ** l)) for l in range(L)]
    begin = IR.table_layout(res, bw, coord_dim)
    table = (rng.standard_normal((int(begin[-1]), F)) * std).astype(np.float32)
    FW = F * L if multiscale == "cat" else F
    IN = FW + 14
    params = (rng.standard_normal(H * IN + H + 3 * H + 3) * 0.3).astype(np.float32)
    coords = rng.uniform(-1, 1, (N, 2)).astype(np.float32)
    coords[:4] = [[1, 1], [-1, -1], [1, -1], [0, 0]]
    gt = rng.uniform(0, 1, (N, 3)).astype(np.float32)
    return dict(res=res, bw=bw, begin=begin, table=table, params=params, coords=coords, gt=gt, F=F, L=L, H=H, IN=IN, ms=multiscale)


def torch_model(c, dtype, lod):
    """ImageNeuralField.rgb + F.mse_loss in torch autograd over the emulated rows and coefficients, in `dtype`."""
    table = torch.tensor(c["table"], dtype=dtype, requires_grad=True)
    params = torch.tensor(c["params"], dtype=dtype, requires_grad=True)
    coords = torch.tensor(c["coords"], dtype=dtype)
    feats = []
    for l, r in enumerate(c["res"]):
        rows, cf = IR.corners(c["coords"], r, c["bw"])
        rows = torch.from_numpy(rows + c["begin"][l]); cf = torch.tensor(cf, dtype=dtype)
        feats.append(sum(table[rows[:, j]] * cf[:, j:j + 1] for j in range(4)))
    if c["ms"] == "cat":
        f = torch.cat(feats, 1)
        f = torch.cat([f[:, :lod * c["F"]], torch.zeros_like(f[:, lod * c["F"]:])], 1)
    else:
        f = torch.stack(feats, 1).sum(1)
    w = torch.cat([coords * b for b in IR.BANDS], 1)
    x = torch.cat([f, coords, torch.sin(w), torch.cos(w)], 1)
    H, IN = c["H"], c["IN"]
    W0 = params[:H * IN].view(H, IN); b0 = params[H * IN:H * IN + H]
    Wo = params[H * IN + H:H * IN + 4 * H].view(3, H); bo = params[H * IN + 4 * H:]
    y = torch.sigmoid(torch.relu(x @ W0.T + b0) @ Wo.T + bo)
    loss = torch.nn.functional.mse_loss(y, torch.tensor(c["gt"], dtype=dtype))
    loss.backward()
    return y.detach().numpy(), float(loss.detach()), table.grad.numpy(), params.grad.numpy()


@pytest.mark.parametrize("ms,coord_dim,F", [("cat", 3, 2), ("sum", 2, 4), ("cat", 2, 8)])
def test_float64_chain_equals_torch_autograd(ms, coord_dim, F):
    c = make_case(coord_dim=coord_dim, F=F, multiscale=ms)
    lod = c["L"] - 1
    y, loss, gt, gp = torch_model(c, torch.float64, lod)
    r = IR.train(c["coords"], c["gt"], c["table"], c["params"], c["res"], c["bw"], c["begin"], ms, lod, c["H"], rounding=False)
    assert abs(r["loss"] - loss) <= 1e-12 * loss
    assert np.abs(r["y"] - y).max() <= 1e-12
    assert np.abs(r["gtable"] - gt).max() <= 1e-12 * np.abs(gt).max()
    assert np.abs(r["gparams"] - gp).max() <= 1e-12 * np.abs(gp).max()


@pytest.mark.parametrize("ms,lod", [("cat", 3), ("cat", 1), ("sum", 3)])
def test_fp32_autograd_inside_intervals(ms, lod):
    """fp32 torch (other summation orders than the kernels') lands inside the a-priori radii: they bound any order."""
    c = make_case(multiscale=ms, F=4, H=32, N=500, seed=3)
    y, loss, gt, gp = torch_model(c, torch.float32, lod)
    r = IR.train(c["coords"], c["gt"], c["table"], c["params"], c["res"], c["bw"], c["begin"], ms, lod, c["H"])
    assert np.all(np.abs(y - r["y"]) <= r["ry"])
    assert abs(loss - r["loss"]) <= r["rloss"]
    assert np.all(np.abs(gt - r["gtable"]) <= r["rgtable"] + 1e-30)
    assert np.all(np.abs(gp - r["gparams"]) <= r["rgparams"] + 1e-30)
    # the radii are informative: well below the values they bound
    assert np.median(r["rgparams"] / np.maximum(np.abs(r["gparams"]), 1e-30)) < 1e-3


@pytest.mark.parametrize("coord_dim", [2, 3])
def test_rows_stay_inside_their_level(coord_dim):
    """Dense levels with res >= 258 at coordinates exactly +-1: the clamp puts +1 on the last cell, whose +1 corner (weight 0) keeps
    the cell's own row; the reference's unclamped row lies past the level (past the table for a coord_dim = 2 table's last level)."""
    bw = 19
    res = [258, 400, 724]
    assert all(IR.is_dense(r, bw) for r in res)
    edge = np.array([[1, 1], [-1, 1], [1, -1], [-1, -1], [1, 0.3], [0.2, 1], [np.nan, 1]], np.float32)
    for r in res:
        rows, cf = IR.corners(edge, r, bw)
        assert rows.min() >= 0 and rows.max() < IR.level_rows(r, bw, coord_dim)
        raw, _ = IR.corners(edge, r, bw, top_clamp=False)
        moved = rows != raw
        assert np.all(cf[moved] == 0)                                 # only weight-0 corners move
        if coord_dim == 2:
            assert raw.max() >= r * r                                 # the reference's row past the level
    # res^2 == T: hashed, every row below T
    rows, _ = IR.corners(np.random.default_rng(0).uniform(-1.2, 1.2, (1000, 2)).astype(np.float32), 2 ** 6, 12)
    assert not IR.is_dense(2 ** 6, 12) and rows.max() < 2 ** 12


def test_hashgrid_mirror_accepts_2d_and_rejects_other_widths():
    g = W.HashGrid.from_geometric(None, feature_dim=2, num_lods=4, multiscale_type='cat', codebook_bitwidth=10, min_grid_res=4,
                                  max_grid_res=48, coord_dim=2)
    assert g.codebook.feats.shape[0] == int(IR.table_layout(g.resolutions, 10, 2)[-1])
    with pytest.raises(AssertionError):
        W.HashGrid.from_geometric(None, 2, 4, 'cat', codebook_bitwidth=10, min_grid_res=4, max_grid_res=48, coord_dim=4)
    with pytest.raises(ValueError):
        W.ops.hashgrid(torch.zeros(5, 4), 10, 3, g.codebook)
    with pytest.raises(W.WispB200Error):                              # 2-D is accepted, and has no CPU fallback
        W.ops.hashgrid(torch.zeros(5, 2), 10, 3, g.codebook)


def test_image_field_mirror_names_and_route():
    g = W.HashGrid.from_geometric(None, feature_dim=2, num_lods=16, multiscale_type='cat', feature_std=1e-9, codebook_bitwidth=19,
                                  min_grid_res=16, max_grid_res=1024)
    nef = W.ImageNeuralField(g, activation_type='relu', layer_type='linear', hidden_dim=64, num_layers=1)
    names = dict(nef.named_parameters())
    assert set(names) == {"grid.codebook.feats", "embedder.bands", "decoder.layers.0.weight", "decoder.layers.0.bias",
                          "decoder.lout.weight", "decoder.lout.bias"}
    assert names["decoder.layers.0.weight"].shape == (64, 46) and names["decoder.lout.weight"].shape == (3, 64)
    assert nef.embed_dim == 14 and nef.embedder.out_dim == 21 and not names["embedder.bands"].requires_grad
    assert W.ops.image_field(nef) is None                             # CPU parameters: not the native route
    with pytest.raises(NotImplementedError):
        W.ImageNeuralField(g, activation_type='sin')


GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "image_step.npz")
DEC = ("decoder.layers.0.weight", "decoder.layers.0.bias", "decoder.lout.weight", "decoder.lout.bias")


def golden_case(z, name):
    res = [int(r) for r in z[f"{name}_resolutions"]]
    bw, cd = int(z[f"{name}_codebook_bitwidth"]), int(z[f"{name}_coord_dim"])
    params = np.concatenate([z[f"{name}_init_{k}"].reshape(-1) for k in DEC])
    return res, bw, IR.table_layout(res, bw, cd), z[f"{name}_init_grid.codebook.feats"], params, str(z[f"{name}_multiscale"])


@pytest.mark.parametrize("name", ["cat3", "sum2"])
def test_reference_golden_first_step(name):
    """tests/golden/image_step.npz (the reference's own ImageTrainer.step, ImageNeuralField and HashGrid, tools/make_image_golden.py):
    the loss and the step-1 gradients lie inside the intervals of the restatement (plus 1e-6 of the largest value for the golden's own
    fp32 rounding of the features)."""
    z = np.load(GOLDEN)
    res, bw, begin, table, params, ms = golden_case(z, name)
    assert table.shape[0] == begin[-1]
    H = int(z["hidden_dim"])
    r = IR.train(z["coords"], z["rgb"], table, params, res, bw, begin, ms, len(res) - 1, H)
    assert abs(z[f"{name}_losses"][0] - r["loss"]) <= r["rloss"] + 1e-6 * r["loss"]
    gp = np.concatenate([z[f"{name}_grad1_{k}"].reshape(-1) for k in DEC])
    assert np.all(np.abs(gp - r["gparams"]) <= r["rgparams"] + 1e-6 * np.abs(gp).max())
    gt = z[f"{name}_grad1_grid.codebook.feats"]
    assert np.all(np.abs(gt - r["gtable"]) <= r["rgtable"] + 1e-6 * np.abs(gt).max())


def test_install_routes_the_reference_image_field():
    """install() against the UNMODIFIED reference ImageNeuralField (imported on CPU through oracle/ref_import.py, in a subprocess: the
    import stubs are process-wide): rgb keeps its signature, ops.image_field reads the reference's own field (declined on CPU tensors),
    the patched rgb falls back to the original body on CPU, the reference's HashGrid accepts [N, 2] through the patched hashgrid only
    with its kernels (no CPU fallback), and uninstall() restores the original."""
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    code = r"""
import inspect, sys, warnings
warnings.filterwarnings("ignore")
sys.path.insert(0, ROOT)
import torch
from oracle import ref_import
ref_import.install()
from wisp.models.grids import HashGrid
from wisp.models.nefs.image_nef import ImageNeuralField
orig = ImageNeuralField.rgb
from wisp_b200 import install as I, ops
import wisp_b200 as W
assert I.install() is True
assert ImageNeuralField.rgb is not orig and list(inspect.signature(ImageNeuralField.rgb).parameters) == list(inspect.signature(orig).parameters)
torch.manual_seed(0)
g = HashGrid.from_geometric(None, feature_dim=2, num_lods=4, multiscale_type='cat', feature_std=0.1, codebook_bitwidth=10, min_grid_res=4, max_grid_res=64)
nef = ImageNeuralField(g, activation_type='relu', layer_type='linear', hidden_dim=16, num_layers=1)
assert ops.image_field(nef) is None                      # CPU tensors
deep = ImageNeuralField(g, activation_type='relu', layer_type='linear', hidden_dim=16, num_layers=2)
assert ops.image_field(deep.cuda() if torch.cuda.is_available() else deep) is None
try:
    with torch.no_grad():
        nef.rgb(torch.zeros(4, 2))
    raise SystemExit("expected the hash-grid kernels to refuse CPU tensors")
except W.WispB200Error:
    pass
I.uninstall()
assert ImageNeuralField.rgb is orig
print("ok")
""".replace("ROOT", repr(root))
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and "ok" in r.stdout, r.stdout[-2000:] + r.stderr[-4000:]
