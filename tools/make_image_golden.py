#!/usr/bin/env python
"""Generate tests/golden/image_step.npz: three optimisation steps of the reference's own ImageTrainer.step
(wisp/trainers/image_trainer.py:51-80) over its own ImageNeuralField (wisp/models/nefs/image_nef.py) and HashGrid.from_geometric, with
the optimiser and MultiStepLR of its BaseTrainer.init_optimizer (wisp/trainers/base_trainer.py:205-246), run on CPU from an UNMODIFIED
kaolin-wisp checkout (TEST INFRASTRUCTURE).

    python tools/make_image_golden.py [path/to/kaolin-wisp]

oracle/ref_import.py answers the 3-D hash-grid kernels; this tool adds the 2-D case to its stand-in for wisp._C.ops
(install_hashgrid2d: the reference's 2-D kernel restated in numpy, picked from the coordinate width as hashgrid_interpolate_cuda.cu:374
picks it).  The trainer modules are loaded from their files; the trainer object is created without its constructor and given what step() and init_optimizer() read.
init_optimizer's `instantiate(cfg.optimizer, params=groups)` (FusedAdam in image_hash.yaml, adam_w_mode) is answered by
torch.optim.AdamW(groups, lr, betas, eps, weight_decay=0): the decoder group carries its weight decay, the grid and rest groups none.
enable_amp is off (fp32); scheduler on with milestones (0.5,) over max_steps = 4, i.e. iteration 2: step 3 runs at lr * gamma.

Cases (16 hidden units, N = 256 pixels including the image corners, grid_lr_weight 5, weight_decay 1e-2):
  cat3  'cat' F = 2, coord_dim 3 (image_hash.yaml's table layout), 4 LODs of 4 .. 64 at bitwidth 10: dense 4, 10, 25, hashed 64
  sum2  'sum' F = 4, coord_dim 2 (min(res^2, T) rows per level), the same resolutions
Recorded per case: the initial parameters, the loss of each step, the gradients of step 1 and the parameters after step 3."""
from __future__ import annotations

import importlib.util
import os
import sys
import warnings
from types import SimpleNamespace

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

LR, EPS, WD, GRID_LR_WEIGHT, GAMMA, STEPS, N, H = 1e-3, 1e-15, 1e-2, 5.0, 0.333, 3, 256, 16
CASES = {"cat3": ("cat", 2, 3), "sum2": ("sum", 4, 2)}


def _load(name, path):
    spec = importlib.util.spec_from_file_location(name, path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _params(nef):
    return {k: p.detach().numpy().copy() for k, p in nef.named_parameters() if p.requires_grad}


def _hashgrid2d_corners(coords, res, codebook_bitwidth):
    """The 2-D path of the reference kernel (hashgrid_interpolate_2d_cuda_kernel, hashgrid_interpolate_cuda.cu:214-339, hash_index_2d
    in hash_utils.cuh:65-84) for one level, as written: x = clamp(res * (c * 0.5 + 0.5), 0, res - 1 - 1e-5) in double, rounded to
    float; corner j = (x + (j>>1 & 1), y + (j & 1)); dense rows x + y*res when res < T and res^2 < T, else (x ^ y*2654435761) % T.
    -> (rows int64 [N, 4] level-local, coefficients fp32 [N, 4])."""
    c = np.asarray(coords, np.float32).astype(np.float64)
    T = 2 ** codebook_bitwidth
    with np.errstate(invalid="ignore"):
        x = np.clip(res * (c * 0.5 + 0.5), 0.0, res - 1 - 1e-5).astype(np.float32)
    p = np.floor(x)
    w = (x - p).astype(np.float32)
    iw = (1.0 - w.astype(np.float64)).astype(np.float32)
    p = p.astype(np.int64)
    cf = np.stack([iw[:, 0] * iw[:, 1], iw[:, 0] * w[:, 1], w[:, 0] * iw[:, 1], w[:, 0] * w[:, 1]], 1).astype(np.float32)
    rows = np.zeros((c.shape[0], 4), np.int64)
    for j in range(4):
        px, py = p[:, 0] + ((j >> 1) & 1), p[:, 1] + (j & 1)
        rows[:, j] = px + py * res if (res < T and res * res < T) else (px ^ ((py * 2654435761) & 0xFFFFFFFF)) % T
    return rows, cf


def install_hashgrid2d():
    """Route [N, 2] calls of the stubbed wisp._C.ops.hashgrid_interpolate_cuda / _backward_cuda to the 2-D restatement above; [N, 3]
    calls keep oracle/ref_import.py's answers."""
    ops = sys.modules["wisp._C.ops"]
    fwd3, bwd3 = ops.hashgrid_interpolate_cuda, ops.hashgrid_interpolate_backward_cuda

    def fwd(coords, codebook, codebook_first_idx, resolution, codebook_bitwidth):
        if coords.shape[-1] != 2:
            return fwd3(coords, codebook, codebook_first_idx, resolution, codebook_bitwidth)
        res = [int(r) for r in resolution.reshape(-1)]
        table, begin = codebook.detach().numpy().astype(np.float32), codebook_first_idx.numpy().astype(np.int64)
        out = []
        for l, r in enumerate(res):
            rows, cf = _hashgrid2d_corners(coords.detach().numpy(), r, codebook_bitwidth)
            v = table[begin[l] + rows].astype(np.float64)                      # [N, 4, F]
            out.append((v * cf[:, :, None].astype(np.float64)).sum(1).astype(np.float32))
        return torch.from_numpy(np.concatenate(out, 1))

    def bwd(coords, grad_output, codebook, codebook_first_idx, resolution, codebook_bitwidth, feature_dim, require_grad_coords):
        if coords.shape[-1] != 2:
            return bwd3(coords, grad_output, codebook, codebook_first_idx, resolution, codebook_bitwidth, feature_dim, require_grad_coords)
        res = [int(r) for r in resolution.reshape(-1)]
        begin = codebook_first_idx.numpy().astype(np.int64)
        go = grad_output.detach().numpy().astype(np.float64).reshape(coords.shape[0], len(res), -1)
        g = np.zeros(tuple(codebook.shape), np.float64)
        for l, r in enumerate(res):
            rows, cf = _hashgrid2d_corners(coords.detach().numpy(), r, codebook_bitwidth)
            for j in range(4):
                np.add.at(g, begin[l] + rows[:, j], go[:, l] * cf[:, j:j + 1].astype(np.float64))
        return [torch.empty(0), torch.from_numpy(g.astype(np.float32))]

    ops.hashgrid_interpolate_cuda, ops.hashgrid_interpolate_backward_cuda = fwd, bwd


def batch():
    rng = np.random.default_rng(23)
    coords = rng.uniform(-1, 1, (N, 2)).astype(np.float32)
    coords[:4] = [[1, 1], [-1, -1], [1, -1], [-1, 1]]
    rgb = rng.uniform(0, 1, (N, 3)).astype(np.float32)
    return coords, rgb


def main():
    from oracle import ref_import
    if len(sys.argv) > 1:
        ref_import.REF_ROOT = sys.argv[1]
    warnings.filterwarnings("ignore")
    ref_import.install()
    install_hashgrid2d()
    import wisp.models, wisp.models.pipeline, wisp.framework, wisp.datasets, wisp.trainers     # noqa: F401
    from wisp.models.grids import HashGrid
    from wisp.models import Pipeline
    nef_mod = _load("ref_image_nef", os.path.join(ref_import.REF_ROOT, "wisp/models/nefs/image_nef.py"))
    it = _load("ref_image_trainer", os.path.join(ref_import.REF_ROOT, "wisp/trainers/image_trainer.py"))
    bt = _load("ref_base_trainer", os.path.join(ref_import.REF_ROOT, "wisp/trainers/base_trainer.py"))
    bt.instantiate = lambda cfg, params: torch.optim.AdamW(params, lr=cfg.lr, betas=cfg.betas, eps=cfg.eps, weight_decay=0.0)
    coords, rgb = batch()
    out = dict(coords=coords, rgb=rgb, lr=LR, eps=EPS, weight_decay=WD, grid_lr_weight=GRID_LR_WEIGHT, gamma=GAMMA,
               milestones=np.asarray([2]), hidden_dim=H)
    for name, (ms, F, cd) in CASES.items():
        torch.manual_seed(11)
        grid = HashGrid.from_geometric(None, feature_dim=F, num_lods=4, multiscale_type=ms, feature_std=0.1, feature_bias=0.0,
                                       codebook_bitwidth=10, min_grid_res=4, max_grid_res=64, coord_dim=cd)
        nef = nef_mod.ImageNeuralField(grid, activation_type='relu', layer_type='linear', hidden_dim=H, num_layers=1)
        t = object.__new__(it.ImageTrainer)
        t.pipeline = Pipeline(nef=nef, tracer=None)
        t.device = 'cpu'
        t.tracker = SimpleNamespace(metrics=SimpleNamespace(total_loss=0., rgb_loss=0.))
        t.train_dataset = [None] * 4
        t.cfg = SimpleNamespace(optimizer=SimpleNamespace(lr=LR, eps=EPS, weight_decay=WD, betas=(0.9, 0.999)), grid_lr_weight=GRID_LR_WEIGHT,
                                max_epochs=1, scheduler_milestones=[0.5], scheduler_gamma=GAMMA, scheduler=True, enable_amp=False)
        bt.BaseTrainer.init_optimizer(t)
        grads = {}

        def record_first_grads(opt, args, kwargs):
            if not grads:
                grads.update({n: p.grad.numpy().copy() for n, p in nef.named_parameters() if p.grad is not None})
        t.optimizer.register_step_pre_hook(record_first_grads)
        d = {f"{name}_multiscale": ms, f"{name}_feature_dim": F, f"{name}_coord_dim": cd, f"{name}_resolutions": np.asarray(grid.resolutions),
             f"{name}_codebook_bitwidth": 10}
        d.update({f"{name}_init_{k}": v for k, v in _params(nef).items()})
        losses = []
        for s in range(STEPS):
            before = t.tracker.metrics.total_loss
            t.step((torch.from_numpy(coords)[None], torch.from_numpy(rgb)[None]))
            losses.append(t.tracker.metrics.total_loss - before)
            if s == 0:
                d.update({f"{name}_grad1_{k}": v for k, v in grads.items()})
        d.update({f"{name}_step3_{k}": v for k, v in _params(nef).items()})
        d[f"{name}_losses"] = np.asarray(losses, np.float64)
        out.update(d)
        print(name, "resolutions", grid.resolutions, "losses", losses, "params", sorted(_params(nef)), "grads", sorted(grads))
    path = os.path.join(ROOT, "tests", "golden", "image_step.npz")
    np.savez_compressed(path, **out)
    print("wrote", path)


if __name__ == "__main__":
    main()
