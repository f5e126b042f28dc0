#!/usr/bin/env python
"""Time the app/image training step at image_hash.yaml's shape (HashGrid.from_geometric 'cat', F 2, 16 LODs of 16 .. 1024 for a
2048^2 image, 2^19 rows per level, decoder 46-64-3, 4096 pixels per step, lr 1e-3, eps 1e-16, weight decay 1e-6, grid_lr_weight 500):
  native    ImageStep: wb_image_train + wb_adamw_step
  fp32      autograd (native 2-D grid kernel + torch embedding, decoder, mse_loss) + torch.optim.AdamW(fused) with init_optimizer's groups
  amp       the same under torch.autocast(fp16) with GradScaler (the reference's enable_amp step)
on the same seeded batches, the arms alternated window by window (median of the windows).  Kernel launches per step come from a
separate torch.profiler run of a few steps per arm.  Then ImageNeuralField.rgb over the full 2048^2 frame in 1 M-pixel chunks (the
trainer's validate()): wb_image_eval against the autograd body under no_grad.  Prints one JSON line with the device name and power limit.

    python tools/bench_image_step.py [--steps 200] [--warmup 20] [--windows 5]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

APP = dict(lr=1e-3, eps=1e-16, weight_decay=1e-6, grid_lr_weight=500.0)
SIDE = 2048


def _gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()
        name, power = [s.strip() for s in out[0].split(",")]
        return name, power
    except Exception:                                   # noqa: BLE001 -- the numbers stand without it
        return torch.cuda.get_device_name(), "unknown"


def _field(W, seed):
    torch.manual_seed(seed)
    g = W.HashGrid.from_geometric(None, feature_dim=2, num_lods=16, multiscale_type='cat', feature_std=1e-9, codebook_bitwidth=19,
                                  min_grid_res=16, max_grid_res=SIDE // 2)
    return W.ImageNeuralField(g, activation_type='relu', layer_type='linear', hidden_dim=64, num_layers=1).cuda()


def _torch_opt(nef):
    dec = [p for n, p in nef.named_parameters() if "decoder" in n and p.requires_grad]
    grid = [p for n, p in nef.named_parameters() if "decoder" not in n and "grid" in n and p.requires_grad]
    return torch.optim.AdamW([{"params": dec, "lr": APP["lr"], "weight_decay": APP["weight_decay"]},
                              {"params": grid, "lr": APP["lr"] * APP["grid_lr_weight"], "weight_decay": 0.0}],
                             lr=APP["lr"], eps=APP["eps"], fused=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--windows", type=int, default=5)
    args = ap.parse_args()
    import wisp_b200 as W
    assert torch.cuda.is_available(), "bench_image_step needs a CUDA device"
    y, x = torch.meshgrid(torch.linspace(-1, 1, SIDE, device="cuda"), torch.linspace(-1, 1, SIDE, device="cuda"), indexing="ij")
    coords = torch.stack([x, y], -1).reshape(-1, 2).contiguous()
    img = torch.stack([0.5 + 0.5 * torch.sin(9 * x + 4 * y * y), 0.5 + 0.5 * torch.cos(13 * torch.hypot(x - 0.2, y + 0.1)),
                       ((torch.floor(6 * (x + 1)) + torch.floor(6 * (y + 1))) % 2) * 0.8 + 0.1], -1).reshape(-1, 3).contiguous()
    gen = torch.Generator(device="cuda").manual_seed(0)
    n_batches = 64
    batches = [torch.randint(0, SIDE * SIDE, (4096,), device="cuda", generator=gen) for _ in range(n_batches)]
    batches = [(coords[i].contiguous(), img[i].contiguous()) for i in batches]

    nef_n, nef_f, nef_a = _field(W, 1), _field(W, 1), _field(W, 1)
    native = W.ImageStep(W.Pipeline(nef_n), **APP)
    assert native.fused
    opt_f, opt_a = _torch_opt(nef_f), _torch_opt(nef_a)
    scaler = torch.amp.GradScaler("cuda")

    def step_native(c, g):
        native.step(c, g)

    def step_fp32(c, g):
        opt_f.zero_grad()
        torch.nn.functional.mse_loss(nef_f.rgb(c), g).backward()
        opt_f.step()

    def step_amp(c, g):
        opt_a.zero_grad()
        with torch.autocast("cuda", torch.float16):
            loss = torch.nn.functional.mse_loss(nef_a.rgb(c), g)
        scaler.scale(loss).backward()
        scaler.step(opt_a)
        scaler.update()

    arms = dict(native=step_native, autograd_fp32=step_fp32, autograd_amp=step_amp)
    for fn in arms.values():
        for k in range(args.warmup):
            fn(*batches[k % n_batches])
    torch.cuda.synchronize()
    times = {k: [] for k in arms}
    for w in range(args.windows):
        for name, fn in arms.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for k in range(args.steps):
                fn(*batches[(w * args.steps + k) % n_batches])
            e1.record()
            torch.cuda.synchronize()
            times[name].append(e0.elapsed_time(e1) / args.steps)
    ms = {k: float(np.median(v)) for k, v in times.items()}

    launches = {}
    for name, fn in arms.items():
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            for k in range(10):
                fn(*batches[k])
            torch.cuda.synchronize()
        launches[name] = sum(1 for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and "memcpy" not in e.name.lower()
                             and "memset" not in e.name.lower()) / 10.0
    before = W._cabi.launch_count()
    native.step(*batches[0])
    torch.cuda.synchronize()
    lib_launches = W._cabi.launch_count() - before

    # full-frame evaluation in 1 M-pixel chunks
    def frame(fused):
        out = []
        for c in coords.split(1 << 20):
            if fused:
                with torch.no_grad():
                    out.append(nef_n.rgb(c))
            else:
                with torch.no_grad(), torch.autocast("cuda", enabled=False):
                    b = c.shape[0]
                    f = nef_n.grid.interpolate(c, len(nef_n.grid.resolutions) - 1).reshape(-1, nef_n.feature_dim)
                    out.append(torch.sigmoid(nef_n.decoder(torch.cat([f, nef_n.embedder(c).view(b, nef_n.embed_dim)], -1))))
        return torch.cat(out)

    eval_ms = {"wb_image_eval": [], "autograd_body": []}
    for _ in range(2):
        frame(True); frame(False)
    torch.cuda.synchronize()
    for w in range(args.windows):
        for name, fused in (("wb_image_eval", True), ("autograd_body", False)):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(3):
                out = frame(fused)
            e1.record()
            torch.cuda.synchronize()
            eval_ms[name].append(e0.elapsed_time(e1) / 3)
    err = float((frame(True) - frame(False)).abs().max())
    name, power = _gpu_info()
    print(json.dumps(dict(workload="image_step_image_hash", device=name, power_limit=power, steps=args.steps, warmup=args.warmup,
                          windows=args.windows, batch=4096, ms_per_step=ms,
                          speedup_vs_fp32=ms["autograd_fp32"] / ms["native"], speedup_vs_amp=ms["autograd_amp"] / ms["native"],
                          kernel_launches_per_step=launches, native_library_launches_per_step=lib_launches,
                          eval_frame=f"{SIDE}x{SIDE}", eval_ms={k: float(np.median(v)) for k, v in eval_ms.items()},
                          eval_speedup=float(np.median(eval_ms["autograd_body"]) / np.median(eval_ms["wb_image_eval"])), eval_max_abs_diff=err)))


if __name__ == "__main__":
    main()
