#!/usr/bin/env python
"""Generate tests/golden/sdf_train.npz: three optimisation steps of the reference's own SDFTrainer.step
(wisp/trainers/sdf_trainer.py:65-124) with the optimiser of its BaseTrainer.init_optimizer (wisp/trainers/base_trainer.py:205-239),
run on CPU from an UNMODIFIED kaolin-wisp checkout (TEST INFRASTRUCTURE).

    python tools/make_sdf_train_golden.py [--deep | --hash] [path/to/kaolin-wisp]

Writes only sdf_train.npz, or with --deep only sdf_train_deep.npz, or with --hash only sdf_train_hash.npz.  Kaolin calls are answered by the oracle (oracle/ref_import.py).  The two trainer modules are loaded
from their files; the trainer object is created without its constructor and given what step() and init_optimizer() read.
init_optimizer's `instantiate(cfg.optimizer, params=groups)` is answered by torch.optim.Adam(groups, lr, betas, eps): the decoder
group carries its weight decay, the grid and rest groups Adam's default of none (the reference's instantiate would also pass
cfg.optimizer.weight_decay as that default; the nglod configs train with weight_decay 0, where the two agree).

Cases (the octahedron model of oracle/make_golden.py:gen_sdf at level 5, 3 LODs, F = 8, H = 16): 'sum' and 'cat' with only_last,
and 'sum' over all LODs, with one hidden layer; --deep: 'sum' only_last with 2 hidden layers, 'cat' only_last with 3, and 'sum'
over all LODs with 2 (the deeper layers pass the six |x|-units through unchanged, as oracle.sdf_reference.random_decoder);
--hash: the reference's NeuralSDF(HashGrid.from_geometric(4 LODs, 4 .. 32, codebook_bitwidth 10: dense levels 4 and 8, hashed
levels 16 and 32 with collisions)), 'cat' F = 8 only_last, 'sum' F = 4 only_last, 'cat' F = 8 over all LODs, and 'cat' F = 8 with
2 hidden layers (the hash kernels answered by the oracle).  grid_lr_weight = 5 and weight_decay = 1e-2 so that every group is pinned.  Recorded per case: the initial
parameters, the loss of each step, the gradients of step 1 (after backward(), before optimizer.step()) and the parameters after
steps 1 and 3."""
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

LR, EPS, WD, GRID_LR_WEIGHT, STEPS, N = 1e-3, 1e-15, 1e-2, 5.0, 3, 256
CASES = {"sum": ("sum", True, 1), "cat": ("cat", True, 1), "sum_all": ("sum", False, 1)}
DEEP_CASES = {"sum": ("sum", True, 2), "cat": ("cat", True, 3), "sum_all": ("sum", False, 2)}
HASH_CASES = {"cat": ("cat", True, 1, 8), "sum": ("sum", True, 1, 4), "cat_all": ("cat", False, 1, 8), "cat_l2": ("cat", True, 2, 8)}


def _load(name, path):
    spec = importlib.util.spec_from_file_location(name, path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _params(nef):
    return {k: p.detach().numpy().copy() for k, p in nef.named_parameters() if p.requires_grad}


def init_decoder(nef):
    """sdf ~ (|x|+|y|+|z|)/sqrt(3) - 0.3 + small learned perturbation (as gen_sdf)."""
    with torch.no_grad():
        W0 = nef.decoder.layers[0].weight; W0.mul_(0.05)
        W0[:6, :3] = torch.tensor([[1, 0, 0], [-1, 0, 0], [0, 1, 0], [0, -1, 0], [0, 0, 1], [0, 0, -1.0]])
        nef.decoder.layers[0].bias.uniform_(-0.05, 0.05)
        for l in list(nef.decoder.layers)[1:]:
            l.weight.mul_(0.05); l.weight[:6, :] = 0.0; l.weight[:6, :6] = torch.eye(6)
            l.bias.uniform_(-0.05, 0.05); l.bias[:6] = 0.0
        nef.decoder.lout.weight.mul_(0.05); nef.decoder.lout.weight[0, :6] = 1.0 / np.sqrt(3.0)
        nef.decoder.lout.bias.fill_(-0.25)


def batch():
    """The training batch of every case: N points around the octahedron with its noisy distance."""
    rng = np.random.default_rng(17)
    coords = rng.uniform(-0.7, 0.7, (N, 3)).astype(np.float32)
    sdf = ((np.abs(coords).sum(-1, keepdims=True) - 0.3) / np.sqrt(3.0) + rng.normal(0.0, 0.01, (N, 1))).astype(np.float32)
    return coords, sdf


def main():
    from oracle import oracle as O
    from oracle import ref_import
    args = sys.argv[1:]
    deep, hashed = "--deep" in args, "--hash" in args
    args = [a for a in args if a not in ("--deep", "--hash")]
    if args:
        ref_import.REF_ROOT = args[0]
    warnings.filterwarnings("ignore")
    ref_import.install()
    import wisp.models, wisp.models.pipeline, wisp.framework, wisp.datasets, wisp.trainers     # noqa: F401
    from wisp.accelstructs import OctreeAS
    from wisp.models.grids import HashGrid, OctreeGrid
    from wisp.models.nefs import NeuralSDF
    from wisp.models import Pipeline
    from oracle.make_golden import octahedron_points
    st = _load("ref_sdf_trainer", os.path.join(ref_import.REF_ROOT, "wisp/trainers/sdf_trainer.py"))
    bt = _load("ref_base_trainer", os.path.join(ref_import.REF_ROOT, "wisp/trainers/base_trainer.py"))
    bt.instantiate = lambda cfg, params: torch.optim.Adam(params, lr=cfg.lr, betas=cfg.betas, eps=cfg.eps)
    level = 5
    oct_np = O.points_to_octree(octahedron_points(level), level)
    coords, sdf = batch()
    out = dict(octree=oct_np, level=level, coords=coords, sdf=sdf, lr=LR, eps=EPS, weight_decay=WD, grid_lr_weight=GRID_LR_WEIGHT)
    cases = HASH_CASES if hashed else {k: v + (8,) for k, v in (DEEP_CASES if deep else CASES).items()}
    for name, (ms, only_last, layers, F) in cases.items():
        torch.manual_seed(7)
        blas = OctreeAS(torch.from_numpy(oct_np))
        if hashed:
            grid = HashGrid.from_geometric(blas, feature_dim=F, num_lods=4, multiscale_type=ms, feature_std=0.05, feature_bias=0.0,
                                           codebook_bitwidth=10, min_grid_res=4, max_grid_res=32)
        else:
            grid = OctreeGrid(blas, feature_dim=8, num_lods=3, interpolation_type='linear', multiscale_type=ms, feature_std=0.05)
        nl = grid.num_lods
        nef = NeuralSDF(grid, pos_embedder='none', position_input=True, hidden_dim=16, num_layers=layers)
        init_decoder(nef)
        t = object.__new__(st.SDFTrainer)
        t.pipeline = Pipeline(nef=nef, tracer=None)
        t.device = 'cpu'
        t.loss_lods = [nl - 1] if only_last else list(range(nl))
        t.tracker = SimpleNamespace(metrics=SimpleNamespace(total_loss=0., l2_loss=0., rgb_loss=0., num_samples=0))
        t.train_dataset = [None]
        t.cfg = SimpleNamespace(optimizer=SimpleNamespace(lr=LR, eps=EPS, weight_decay=WD, betas=(0.9, 0.999)), grid_lr_weight=GRID_LR_WEIGHT,
                                max_epochs=1, scheduler_milestones=[], scheduler=False)
        bt.BaseTrainer.init_optimizer(t)
        grads = {}

        def record_first_grads(opt, args, kwargs):
            if not grads:
                grads.update({n: p.grad.numpy().copy() for n, p in nef.named_parameters() if p.grad is not None})
        t.optimizer.register_step_pre_hook(record_first_grads)
        d = {f"{name}_multiscale": ms, f"{name}_loss_lods": np.asarray(t.loss_lods)}
        if hashed:
            d.update({f"{name}_feature_dim": F, f"{name}_num_layers": layers, f"{name}_resolutions": np.asarray(grid.resolutions),
                      f"{name}_codebook_bitwidth": 10})
        d.update({f"{name}_init_{k}": v for k, v in _params(nef).items()})
        losses = []
        for s in range(STEPS):
            before = t.tracker.metrics.total_loss
            t.step({'coords': torch.from_numpy(coords), 'sdf': torch.from_numpy(sdf)})
            losses.append((t.tracker.metrics.total_loss - before) / N)       # the tracker holds the loss before `loss /= batch_size`
            if s == 0:
                d.update({f"{name}_step1_{k}": v for k, v in _params(nef).items()})
                d.update({f"{name}_grad1_{k}": v for k, v in grads.items()})
        d.update({f"{name}_step3_{k}": v for k, v in _params(nef).items()})
        d[f"{name}_losses"] = np.asarray(losses, np.float64)
        out.update(d)
        print(name, "losses", losses, "params", len(_params(nef)), "grads", len(grads))
    path = os.path.join(ROOT, "tests", "golden", "sdf_train_hash.npz" if hashed else "sdf_train_deep.npz" if deep else "sdf_train.npz")
    np.savez_compressed(path, **out)
    print(path)


if __name__ == "__main__":
    main()
