#!/usr/bin/env python
"""Time the one-launch optimiser steps over the parameter set of BASELINE config 2 (nerf_hash.yaml: a 5 217 937 x 2 hash table plus
the two 64-wide decoders, 3 152 and 7 107 parameters; seeded values and gradients): NativeAdam / NativeAdamW / NativeRMSprop
(momentum 0 and 0.9), each launch also clearing the gradients, against torch.optim.Adam / AdamW (fused=True) and RMSprop
(foreach=True; torch has no fused RMSprop) each followed by its zero_grad(set_to_none=False), with init_optimizer's groups.
The arms alternate in one process; CUDA events around windows of --steps steps; the median of --rounds windows per arm.

    python tools/bench_optim_step.py [--steps 2000] [--warmup 20] [--rounds 5]

Prints one JSON line: per arm ms/step and the windows; for the native arms the bytes the rule moves per parameter (parameter
read + write, gradient read + clear, every state tensor read + write) and the achieved GB/s over them; library launches per
step; the device name and power limit read in the same run.  Fails without a GPU."""
from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

SHAPES = {"grid": (5217937, 2), "decoder_density": (3152,), "decoder_color": (7107,)}
LR, WD, GRID_LR_WEIGHT, EPS = 1e-3, 1e-6, 100.0, 1e-8
STATE_TENSORS = {"adam": 2, "adamw": 2, "rmsprop": 1, "rmsprop_momentum": 2}


def bytes_per_param(rule: str) -> int:
    return 4 * (2 + 2 + 2 * STATE_TENSORS[rule])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=2000)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_optim_step.py measures on a CUDA device"
    import wisp_b200 as W
    from bench_sdf_step import _gpu_info
    torch.cuda.set_device(0)
    gen = torch.Generator(device="cuda").manual_seed(0)
    total = sum(int(np.prod(s)) for s in SHAPES.values())

    def tensors():
        return {k: torch.randn(s, device="cuda", generator=gen) * 0.1 for k, s in SHAPES.items()}

    def groups(p):
        return [(p["grid"], LR * GRID_LR_WEIGHT, 0.0), (p["decoder_density"], LR, WD), (p["decoder_color"], LR, WD)]

    run = {}
    for rule in STATE_TENSORS:
        p, g = tensors(), tensors()
        if rule == "adam":
            opt = W.NativeAdam(groups(p), eps=EPS)
        elif rule == "adamw":
            opt = W.NativeAdamW(groups(p), eps=EPS)
        else:
            opt = W.NativeRMSprop(groups(p), eps=EPS, momentum=0.9 if rule == "rmsprop_momentum" else 0.0)
        gl = [g["grid"], g["decoder_density"], g["decoder_color"]]
        # every arm clears its gradients, so all but the first step read zeros: the memory traffic is that of any other gradient
        run["native_" + rule] = (lambda opt=opt, gl=gl: opt.step(gl, zero_grad=True))
        p, g = tensors(), tensors()
        for k in p:
            p[k].requires_grad_(True); p[k].grad = g[k]
        tg = [{"params": [p["grid"]], "lr": LR * GRID_LR_WEIGHT, "weight_decay": 0.0},
              {"params": [p["decoder_density"], p["decoder_color"]], "lr": LR, "weight_decay": WD}]
        if rule == "adam":
            topt = torch.optim.Adam(tg, lr=LR, eps=EPS, fused=True)
        elif rule == "adamw":
            topt = torch.optim.AdamW(tg, lr=LR, eps=EPS, fused=True)
        else:
            topt = torch.optim.RMSprop(tg, lr=LR, eps=EPS, momentum=0.9 if rule == "rmsprop_momentum" else 0.0, foreach=True)

        def torch_step(topt=topt):
            topt.step()
            topt.zero_grad(set_to_none=False)
        run["torch_" + rule] = torch_step
    for fn in run.values():
        for _ in range(args.warmup):
            fn()
    torch.cuda.synchronize()
    res = {k: dict(ms=[], launches=0) for k in run}
    for _ in range(args.rounds):                         # alternate the arms
        for k, fn in run.items():
            l0 = W._cabi.launch_count()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(args.steps):
                fn()
            e1.record()
            torch.cuda.synchronize()
            res[k]["ms"].append(e0.elapsed_time(e1) / args.steps)
            res[k]["launches"] += W._cabi.launch_count() - l0
    arms = {}
    for k, v in res.items():
        ms = float(np.median(v["ms"]))
        arms[k] = dict(ms_per_step=ms, ms_per_step_windows=[round(x, 5) for x in v["ms"]], library_launches_per_step=v["launches"] / (args.rounds * args.steps))
        if k.startswith("native_"):
            b = bytes_per_param(k[len("native_"):])
            arms[k].update(bytes_per_param=b, achieved_GB_per_s=b * total / (ms * 1e-3) / 1e9)
    name, power = _gpu_info()
    print(json.dumps(dict(workload="optim_step_config2", parameters=total, device=name, power_limit=power, steps=args.steps, warmup=args.warmup,
                          rounds=args.rounds, arms=arms)))


if __name__ == "__main__":
    main()
