#!/usr/bin/env python
"""Generate tests/golden/optim_groups.npz: eight optimisation steps of the reference's own SDFTrainer.step
(wisp/trainers/sdf_trainer.py:65-124), each followed by scheduler.step() as MultiviewTrainer.step does
(multiview_trainer.py:179-180), with the optimiser AND the MultiStepLR of its BaseTrainer.init_optimizer
(wisp/trainers/base_trainer.py:205-246), run on CPU from an UNMODIFIED kaolin-wisp checkout (TEST INFRASTRUCTURE).

    python tools/make_optim_golden.py [path/to/kaolin-wisp]

Set up as tools/make_sdf_train_golden.py (same model: its 'sum' case, NeuralSDF(OctreeGrid) with one hidden layer, F = 8, 3 LODs,
H = 16; same batch; the octahedron's octree at level 4 instead of 5, which keeps 3 x 8 steps of gradients and parameters under 1 MB):
Kaolin calls are answered by the oracle, the two trainer modules are loaded from their files, the trainer object is created
without its constructor.  init_optimizer's `instantiate(cfg.optimizer, params=groups)` is answered by the torch class the
config names with the options that config exposes, EXCEPT weight_decay: the decoder group carries its own, the grid and rest
groups get the optimiser's default of none (the reference's instantiate would also pass cfg.optimizer.weight_decay as the
default of those groups; this project's documented choice is explicit group options only).

Cases: 'rmsprop' (ConfigRMSprop, momentum 0), 'rmsprop_m' (momentum 0.9), 'adamw' (ConfigAdamW).  grid_lr_weight = 5 and
weight_decay = 1e-2 pin every group; scheduler = True with the default milestones (0.5, 0.75, 0.9) and gamma 0.333 over
len(train_dataset) * max_epochs = 8 steps: init_optimizer hands MultiStepLR the floats 4.0, 6.0 and 7.2, so the rate drops
after steps 4 and 6 and the third milestone never fires.  Recorded per case: the initial parameters, and for every step the
gradients optimizer.step() consumed, each group's learning rate during that step, and the parameters after it."""
from __future__ import annotations

import os
import sys
import warnings
from types import SimpleNamespace

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

LR, EPS, WD, GRID_LR_WEIGHT, STEPS, LEVEL = 1e-3, 1e-8, 1e-2, 5.0, 8, 4
ALPHA, BETAS, MILESTONES, GAMMA = 0.99, (0.9, 0.999), (0.5, 0.75, 0.9), 0.333
CASES = {"rmsprop": ("RMSprop", 0.0), "rmsprop_m": ("RMSprop", 0.9), "adamw": ("AdamW", 0.0)}


def main():
    import make_sdf_train_golden as G
    from oracle import oracle as O
    from oracle import ref_import
    if sys.argv[1:]:
        ref_import.REF_ROOT = sys.argv[1]
    warnings.filterwarnings("ignore")
    ref_import.install()
    import wisp.models, wisp.models.pipeline, wisp.framework, wisp.datasets, wisp.trainers     # noqa: F401
    from wisp.accelstructs import OctreeAS
    from wisp.models.grids import OctreeGrid
    from wisp.models.nefs import NeuralSDF
    from wisp.models import Pipeline
    from oracle.make_golden import octahedron_points
    st = G._load("ref_sdf_trainer", os.path.join(ref_import.REF_ROOT, "wisp/trainers/sdf_trainer.py"))
    bt = G._load("ref_base_trainer", os.path.join(ref_import.REF_ROOT, "wisp/trainers/base_trainer.py"))

    def instantiate(cfg, params):
        if cfg.constructor == "RMSprop":
            return torch.optim.RMSprop(params, lr=cfg.lr, alpha=cfg.alpha, eps=cfg.eps, momentum=cfg.momentum)
        return torch.optim.AdamW(params, lr=cfg.lr, betas=cfg.betas, eps=cfg.eps, weight_decay=0.0)
    bt.instantiate = instantiate
    level = LEVEL
    oct_np = O.points_to_octree(octahedron_points(level), level)
    coords, sdf = G.batch()
    out = dict(octree=oct_np, level=level, coords=coords, sdf=sdf, lr=LR, eps=EPS, weight_decay=WD, grid_lr_weight=GRID_LR_WEIGHT,
               alpha=ALPHA, betas=np.asarray(BETAS), gamma=GAMMA, steps=STEPS)
    for name, (ctor, momentum) in CASES.items():
        torch.manual_seed(7)
        grid = OctreeGrid(OctreeAS(torch.from_numpy(oct_np)), feature_dim=8, num_lods=3, interpolation_type='linear', multiscale_type='sum',
                          feature_std=0.05)
        nef = NeuralSDF(grid, pos_embedder='none', position_input=True, hidden_dim=16, num_layers=1)
        G.init_decoder(nef)
        t = object.__new__(st.SDFTrainer)
        t.pipeline = Pipeline(nef=nef, tracer=None)
        t.device = 'cpu'
        t.loss_lods = [grid.num_lods - 1]
        t.tracker = SimpleNamespace(metrics=SimpleNamespace(total_loss=0., l2_loss=0., rgb_loss=0., num_samples=0))
        t.train_dataset = [None] * 4
        t.cfg = SimpleNamespace(optimizer=SimpleNamespace(constructor=ctor, lr=LR, eps=EPS, weight_decay=WD, betas=BETAS, alpha=ALPHA, momentum=momentum),
                                grid_lr_weight=GRID_LR_WEIGHT, max_epochs=2, scheduler_milestones=list(MILESTONES), scheduler_gamma=GAMMA, scheduler=True)
        bt.BaseTrainer.init_optimizer(t)
        names = [k for k, p in nef.named_parameters() if p.requires_grad]
        grads = []
        t.optimizer.register_step_pre_hook(
            lambda opt, args, kwargs: grads.append({k: p.grad.numpy().copy() for k, p in nef.named_parameters() if p.grad is not None}))
        d = {f"{name}_momentum": momentum, f"{name}_milestone_iters": np.asarray(sorted(t.scheduler.milestones.elements())),
             f"{name}_names": np.asarray(names)}
        d.update({f"{name}_init_{k}": v for k, v in G._params(nef).items()})
        lrs = []
        for s in range(1, STEPS + 1):
            lrs.append([g["lr"] for g in t.optimizer.param_groups])            # decoder, grid, rest
            t.step({'coords': torch.from_numpy(coords), 'sdf': torch.from_numpy(sdf)})
            t.scheduler.step()
            d.update({f"{name}_step{s}_{k}": v for k, v in G._params(nef).items()})
            d.update({f"{name}_grad{s}_{k}": v for k, v in grads[s - 1].items()})
        d[f"{name}_lrs"] = np.asarray(lrs, np.float64)
        out.update(d)
        print(name, "lrs (decoder)", [l[0] for l in lrs], "params", len(names))
    path = os.path.join(ROOT, "tests", "golden", "optim_groups.npz")
    np.savez_compressed(path, **out)
    print(path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
