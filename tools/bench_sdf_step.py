#!/usr/bin/env python
"""Time the app/nglod training step at BASELINE config-3 shapes: SDFStep (wb_sdf_train + wb_adam_step) against the autograd route
(grid kernel + torch decoder, torch loss and backward) + fused torch.optim.Adam with the reference's groups, on the same seeded
inputs, alternating the two arms.  Prints one JSON line: ms/step, samples/s and library launches per step of each arm and batch
size, the device name and power limit, and a parity block (SDFStep's gradients against the autograd route at batch 65 536; a
parity failure fails the run).

    python tools/bench_sdf_step.py [--steps 200] [--warmup 20] [--batches 512,65536,1048576] [--num-layers 1] [--hidden-dim 128]
                                   [--grid octree|hash] [--precision 0|1]

--num-layers / --hidden-dim replace config 3's decoder (19-128-1) by one with that many hidden layers of that width
(oracle.sdf_reference.random_decoder, seeded); the grid and the samples stay config 3's.
--grid hash replaces config 3's OctreeGrid by the nglod_hash.yaml grid (HashGrid.from_geometric: 'cat', F = 8, 4 LODs of 16 .. 2048,
2^19 rows per level, feature_std 0.01, seeded) with identity position input and a decoder of --num-layers x --hidden-dim (torch's
default init, seeded); octree and samples stay config 3's.
--precision 1 times SDFStep(precision=1) (wb_sdf_train_tc + wb_adam_step: the reference's enable_amp arithmetic on the tensor
cores) against SDFStep() (precision 0) and against the reference's own enable_amp arm, autograd under torch.autocast(fp16) + fused
torch.optim.Adam; its parity block compares precision 1 with that arm at batch 65 536 (loss 2e-3 relative, gradients 3e-2 of
max, the arm's backward loss-scaled by the same power of two as the kernel's).
"""
from __future__ import annotations

import argparse
import contextlib
import json
import math
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def _gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()
        name, power = [s.strip() for s in out[0].split(",")]
        return name, power
    except Exception:                                   # noqa: BLE001 -- the numbers stand without it
        return torch.cuda.get_device_name(), "unknown"


def _points(case, n, seed):
    rng = np.random.default_rng(seed)
    spc, L = case["spc"], case["level"]
    pts = spc.points[spc.pyramid[1, L]: spc.pyramid[1, L] + spc.pyramid[0, L]].astype(np.float32)
    nn = (n + 1) // 2
    near = (pts[rng.integers(0, pts.shape[0], nn)] + rng.random((nn, 3)).astype(np.float32)) / (2.0 ** (L - 1)) - 1.0
    c = np.concatenate([near, rng.uniform(-1.05, 1.05, (n - nn, 3))]).astype(np.float32)[:n]
    gt = ((np.abs(c).sum(-1, keepdims=True) - 0.5) / np.sqrt(3.0)).astype(np.float32)
    return torch.from_numpy(c).cuda(), torch.from_numpy(gt).cuda()


def _torch_adam(nef, lr, eps):
    dec = [p for n, p in nef.named_parameters() if p.requires_grad and "decoder" in n]
    grd = [p for n, p in nef.named_parameters() if p.requires_grad and "decoder" not in n and "grid" in n]
    return torch.optim.Adam([{"params": dec, "lr": lr, "eps": eps, "weight_decay": 0.0}, {"params": grd, "eps": eps, "lr": lr}],
                            lr=lr, eps=eps, fused=True)


def _autograd_step(nef, opt, coords, gt, update=True, amp=False):
    opt.zero_grad(set_to_none=True)
    with torch.autocast("cuda", torch.float16) if amp else contextlib.nullcontext():
        loss = ((nef(coords=coords, lod_idx=nef.grid.num_lods - 1, channels="sdf") - gt) ** 2).sum() / coords.shape[0]
    loss.backward()
    if update:
        opt.step()
    return loss.detach()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--batches", default="512,65536,1048576")
    ap.add_argument("--num-layers", type=int, default=1)
    ap.add_argument("--hidden-dim", type=int, default=128)
    ap.add_argument("--grid", choices=["octree", "hash"], default="octree")
    ap.add_argument("--precision", type=int, choices=[0, 1], default=0)
    args = ap.parse_args()
    import wisp_b200 as W
    from oracle import octree_grid as OG
    from gpu_util import sdf_nef_from_case
    assert torch.cuda.is_available(), "bench_sdf_step.py measures on a CUDA device"
    torch.cuda.set_device(0)
    case = OG.make_sdf_case(level=7, num_lods=6, feature_dim=16, hidden_dim=128, multiscale="sum", res=4, seed=11, feature_std=0.02)
    if (args.num_layers, args.hidden_dim) != (1, 128):
        from oracle import sdf_reference as S
        case["W"], case["b"] = S.random_decoder(np.random.default_rng(4), 19, 1, args.hidden_dim, args.num_layers, scale=0.2)
    lr, eps = 1e-3, 1e-15

    def make_nef():
        if args.grid == "octree":
            return sdf_nef_from_case(case)
        torch.manual_seed(0)
        blas = W.OctreeAS(torch.from_numpy(case["octree"]).cuda())
        grid = W.HashGrid.from_geometric(blas, feature_dim=8, num_lods=4, multiscale_type='cat', feature_std=0.01, codebook_bitwidth=19,
                                         min_grid_res=16, max_grid_res=2048)
        return W.NeuralSDF(grid, pos_embedder='none', position_input=True, hidden_dim=args.hidden_dim, num_layers=args.num_layers).cuda()

    # parity: SDFStep's gradients and loss against the autograd route at batch 65 536
    nef = make_nef()
    amp = args.precision == 1
    step = W.SDFStep(W.Pipeline(nef), lr=lr, eps=eps, precision=args.precision)
    c, gt = _points(case, 65536, 1)
    loss = float(step.step(c, gt, update=False))
    for p in nef.parameters():
        p.grad = None
    scale = 2.0 ** -math.frexp(1.0 / 65536)[1] if amp else 1.0       # wb_sdf_train_tc's power-of-two loss scale at this batch
    with torch.autocast("cuda", torch.float16) if amp else contextlib.nullcontext():
        ref = ((nef(coords=c, lod_idx=nef.grid.num_lods - 1, channels="sdf") - gt) ** 2).sum() / c.shape[0]
    (ref * scale).backward()
    ref = ref.detach()
    for p in nef.parameters():
        if p.grad is not None:
            p.grad /= scale
    got = list(step.g_feats) + [step.g_dec]
    refs = [f.grad for f in W.SDFStep._grid_tensors(nef.grid)] + [torch.cat([p.grad.reshape(-1) for p in W.ops.decoder_params(nef.decoder)])]
    grad_err = max(float((a - b).abs().max() / b.abs().max().clamp_min(1e-30)) for a, b in zip(got, refs))
    loss_err = abs(loss - float(ref)) / abs(float(ref))
    parity = dict(batch=65536, loss=loss, loss_autograd=float(ref), loss_relerr=loss_err, grad_relerr_of_max=grad_err,
                  ok=bool((step.fused or amp) and loss_err <= (5e-2 if amp else 1e-5) and grad_err <= (3e-2 if amp else 1e-4)))
    step.zero_grads()

    arms = {}
    for B in [int(b) for b in args.batches.split(",")]:
        nef_n, nef_a = make_nef(), make_nef()
        native = W.SDFStep(W.Pipeline(nef_n), lr=lr, eps=eps, precision=args.precision)
        opt = _torch_adam(nef_a, lr, eps)
        coords, gts = _points(case, B, 2)
        run = {"native": lambda: native.step(coords, gts), "autograd": lambda: _autograd_step(nef_a, opt, coords, gts, amp=amp)}
        if amp:                                          # precision 0 on its own copy of the field
            native0 = W.SDFStep(W.Pipeline(make_nef()), lr=lr, eps=eps)
            run["native_precision0"] = lambda: native0.step(coords, gts)
        for fn in run.values():
            for _ in range(args.warmup):
                fn()
        torch.cuda.synchronize()
        res = {k: dict(ms=[], launches=0) for k in run}
        rounds = 4
        per = max(1, args.steps // rounds)
        for _ in range(rounds):                          # alternate the arms
            for k, fn in run.items():
                l0 = W._cabi.launch_count()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(per):
                    fn()
                e1.record()
                torch.cuda.synchronize()
                res[k]["ms"].append(e0.elapsed_time(e1) / per)
                res[k]["launches"] += W._cabi.launch_count() - l0
        arms[str(B)] = {k: dict(ms_per_step=float(np.median(v["ms"])), ms_per_step_runs=[round(x, 4) for x in v["ms"]],
                                samples_per_s=B / (float(np.median(v["ms"])) * 1e-3), library_launches_per_step=v["launches"] / (rounds * per))
                        for k, v in res.items()}
        arms[str(B)]["speedup"] = arms[str(B)]["autograd"]["ms_per_step"] / arms[str(B)]["native"]["ms_per_step"]
        if amp:
            arms[str(B)]["speedup_over_precision0"] = arms[str(B)]["native_precision0"]["ms_per_step"] / arms[str(B)]["native"]["ms_per_step"]
    name, power = _gpu_info()
    print(json.dumps(dict(workload="sdf_step_config3" if args.grid == "octree" else "sdf_step_nglod_hash", num_layers=args.num_layers, hidden_dim=args.hidden_dim, precision=args.precision, fused=step.fused, device=name, power_limit=power, steps=args.steps, warmup=args.warmup,
                          batches=arms, parity=parity)))
    if not parity["ok"]:
        sys.exit(1)


if __name__ == "__main__":
    main()
