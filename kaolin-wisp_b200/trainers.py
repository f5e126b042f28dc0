"""MultiviewStep (below), SDFStep and ImageStep (at the end): the trainers' steps as native sequences.

MultiviewStep: the optimisation step of wisp.trainers.MultiviewTrainer (wisp/trainers/multiview_trainer.py:111-180) with the
optimiser set-up of BaseTrainer.init_optimizer (wisp/trainers/base_trainer.py:205-235), as ONE native sequence without autograd:

    march (count / scan / fill; pre-marched on a side stream when the next batch is known)
    shade forward (gather + decoders) -> composite forward
    composite backward WITH the image loss and its gradient inside (wb_composite_bwd_loss)       [torch: 6 launches + a [R,3] tensor]
    device loss scale -> decoder backward -> grid scatter, into persistent gradient buffers
    [N > 1: NCCL all-reduce(sum) of the gradient buffers; the 1/world is folded into the optimiser]
    Adam / AdamW / RMSprop over grid + decoders in one launch that also clears the gradients        [torch: zero_grad + fused Adam]
    (wb_adam_step / wb_adamw_step / wb_rmsprop_step), at the learning rate MultiStepLR would have reached

What the reference does around it and this keeps: parameter groups by name ('decoder' -> weight decay, 'grid' -> lr * grid_lr_weight),
rgb_loss_type l2 / l1 / huber, rgb_loss_denom rays / samples, tracer.prev_num_samples for the adaptive ray budget.  What it drops:
GradScaler (the fp16 decoder backward carries its own power-of-two loss scale on the device, no inf checks or skipped steps).
Fields outside the fused path (ops.nef_spec is None) fall back to autograd + the same native optimiser.
"""
from __future__ import annotations

import contextlib
import ctypes as C
from typing import Optional

import torch
import torch.distributed as dist

from . import _cabi as A
from . import ops
from .core import Rays

LOSS_TYPES = {"l2": 0, "l1": 1, "huber": 2}


def _fill_segments(segs, entries, grads, lr_scale, **state):
    """Fill the C segment array of one step; state: the two state fields of the segment struct by name, each a list of tensors or
    None.  lr_scale multiplies every learning rate in double before the fp32 conversion (1.0: the rate as constructed)."""
    if entries:
        A.require_device(entries[0][0])                                       # no CPU fallback
    for k, ((p, lr, wd), g) in enumerate(zip(entries, grads)):
        assert g.is_contiguous() and p.is_contiguous() and g.numel() == p.numel() and p.dtype == torch.float32 and g.dtype == torch.float32
        sg = segs[k]
        sg.param, sg.grad, sg.numel, sg.lr, sg.weight_decay = p.data_ptr(), g.data_ptr(), p.numel(), lr * lr_scale, wd
        for name, tensors in state.items():
            setattr(sg, name, tensors[k].data_ptr() if tensors is not None else None)


class NativeAdam:
    """torch.optim.Adam (amsgrad off) over a list of (tensor, lr, weight_decay) in one launch; see wb_adam_step.
    `lr_scale` (an attribute, 1.0 unless set) multiplies every entry's learning rate in the steps that follow: a schedule's factor."""
    _entry = "wb_adam_step"

    def __init__(self, entries, betas=(0.9, 0.999), eps=1e-8):
        self.entries = [(p, float(lr), float(wd)) for p, lr, wd in entries]
        self.betas, self.eps, self.t, self.lr_scale = betas, float(eps), 0, 1.0
        self.exp_avg = [torch.zeros_like(p, dtype=torch.float32) for p, _, _ in self.entries]
        self.exp_avg_sq = [torch.zeros_like(p, dtype=torch.float32) for p, _, _ in self.entries]

    def step(self, grads, grad_scale: float = 1.0, zero_grad: bool = True):
        n = len(self.entries)
        segs = (A.AdamSegment * n)()
        _fill_segments(segs, self.entries, grads, self.lr_scale, exp_avg=self.exp_avg, exp_avg_sq=self.exp_avg_sq)
        self.t += 1
        A.check(getattr(A.lib(), self._entry)(segs, C.c_int32(n), C.c_float(self.betas[0]), C.c_float(self.betas[1]), C.c_float(self.eps), C.c_int32(self.t),
                                              C.c_float(grad_scale), C.c_int32(int(zero_grad)), A.stream()))


class NativeAdamW(NativeAdam):
    """torch.optim.AdamW (amsgrad off; apex FusedAdam's default adam_w_mode) with NativeAdam's interface: the entries' weight decay
    is decoupled, p *= 1 - lr * weight_decay before the Adam update; see wb_adamw_step."""
    _entry = "wb_adamw_step"


class NativeRMSprop:
    """torch.optim.RMSprop (centered off) over a list of (tensor, lr, weight_decay) in one launch, with NativeAdam's step and
    lr_scale; see wb_rmsprop_step.  momentum_buffer is None when momentum == 0."""

    def __init__(self, entries, alpha=0.99, eps=1e-8, momentum=0.0):
        self.entries = [(p, float(lr), float(wd)) for p, lr, wd in entries]
        self.alpha, self.eps, self.momentum, self.t, self.lr_scale = float(alpha), float(eps), float(momentum), 0, 1.0
        if self.momentum < 0.0:
            raise ValueError(f"NativeRMSprop: momentum must be >= 0, got {momentum!r}")
        self.square_avg = [torch.zeros_like(p, dtype=torch.float32) for p, _, _ in self.entries]
        self.momentum_buffer = [torch.zeros_like(p, dtype=torch.float32) for p, _, _ in self.entries] if self.momentum > 0.0 else None

    def step(self, grads, grad_scale: float = 1.0, zero_grad: bool = True):
        n = len(self.entries)
        segs = (A.RMSpropSegment * n)()
        _fill_segments(segs, self.entries, grads, self.lr_scale, square_avg=self.square_avg, momentum_buffer=self.momentum_buffer)
        self.t += 1
        A.check(A.lib().wb_rmsprop_step(segs, C.c_int32(n), C.c_float(self.alpha), C.c_float(self.eps), C.c_float(self.momentum),
                                        C.c_float(grad_scale), C.c_int32(int(zero_grad)), A.stream()))


OPTIMIZERS = ("adam", "adamw", "rmsprop")


def _make_optimizer(optimizer, tensors, betas, eps, alpha, momentum):
    """The native optimiser MultiviewStep / SDFStep step with: cfg.optimizer.constructor 'Adam' | 'AdamW' (and apex 'FusedAdam')
    | 'RMSprop' of the reference's configs (wisp/config/presets/torch.py:37-67) as "adam" | "adamw" | "rmsprop"."""
    if optimizer not in OPTIMIZERS:
        raise ValueError(f"optimizer must be one of {OPTIMIZERS}, got {optimizer!r}")
    if optimizer == "rmsprop":
        return NativeRMSprop(tensors, alpha=alpha, eps=eps, momentum=momentum)
    return (NativeAdamW if optimizer == "adamw" else NativeAdam)(tensors, betas=betas, eps=eps)


def multistep_factor(milestones, gamma: float, t: int) -> float:
    """Learning-rate factor of optimiser step t (1-based) under torch.optim.lr_scheduler.MultiStepLR stepped once after every
    optimiser step: gamma^k, k = the number of milestones <= t - 1 counted with multiplicity, multiplied up in double."""
    f = 1.0
    for m in milestones:
        if m <= t - 1:
            f *= gamma
    return f


def _flatten_in_place(module_params):
    """Re-point the .data of `module_params` at consecutive views of one flat fp32 buffer (as DDP's buckets do): the packed decoder
    parameter vector the C ABI wants then exists without a per-step torch.cat, and one Adam segment covers the whole decoder."""
    flat = torch.cat([p.data.reshape(-1).float() for p in module_params]).contiguous()
    o = 0
    for p in module_params:
        n = p.numel()
        p.data = flat[o:o + n].view_as(p)
        o += n
    return flat


class MultiviewStep:
    def __init__(self, pipeline, lr: float = 1e-3, eps: float = 1e-15, weight_decay: float = 0.0, grid_lr_weight: float = 1.0, betas=(0.9, 0.999),
                 rgb_loss_type: str = "huber", rgb_loss_denom: str = "rays", precision: Optional[int] = None, group=None,
                 optimizer: str = "adam", alpha: float = 0.99, momentum: float = 0.0, scheduler_milestones=(), scheduler_gamma: float = 0.333):
        """`optimizer`: "adam" | "adamw" | "rmsprop", the rule cfg.optimizer.constructor names (apex FusedAdam: "adamw"); `betas`
        belong to the first two, `alpha` and `momentum` to RMSprop.  The parameter groups are the same under every rule.

        `scheduler_milestones` / `scheduler_gamma`: the MultiStepLR the reference steps after every optimiser step
        (multiview_trainer.py:179-180).  The milestones are ITERATION NUMBERS (ints): optimiser step t (1-based) runs at
        lr * gamma^k, k = the number of milestones <= t - 1, a repeated milestone counted each time.  step(update=False) does
        not advance the schedule.  The reference's own milestones are not these numbers: init_optimizer hands MultiStepLR the
        floats max_steps * x (max_steps = len(train_dataset) * max_epochs, x in cfg.scheduler_milestones; base_trainer.py:237-246),
        and MultiStepLR.step tests `last_epoch in milestones`, so a milestone fires only when that product is integer-valued
        (8 steps with (0.5, 0.75, 0.9): 4.0 and 6.0 fire, 7.2 never does).  Pass the iterations that do fire.  Empty: no schedule."""
        if rgb_loss_type not in LOSS_TYPES or rgb_loss_denom not in ("rays", "samples"):
            raise NotImplementedError                                                        # multiview_trainer.py:147,157
        self.pipeline, self.nef, self.tracer = pipeline, pipeline.nef, pipeline.tracer
        self.loss_type, self.loss_denom, self.group = rgb_loss_type, rgb_loss_denom, group
        self.precision = precision
        nef = self.nef
        self.spec = ops.nef_spec(nef, None)
        self.fused = self.spec is not None
        if self.fused:
            self.dens_flat = _flatten_in_place(ops.decoder_params(nef.decoder_density))
            self.col_flat = _flatten_in_place(ops.decoder_params(nef.decoder_color))
            self.grid = ops.grid_tensors(nef, self.spec)             # every LOD: a step renders at the finest LOD (random_lod off, multiview_trainer.py:135-137)
            tensors = [(g.data, lr * grid_lr_weight, 0.0) for g in self.grid] + [(self.dens_flat, lr, weight_decay), (self.col_flat, lr, weight_decay)]
            rest = [p for n, p in nef.named_parameters() if p.requires_grad and "decoder" not in n and "grid" not in n]
            tensors += [(p.data, lr, 0.0) for p in rest]
            self.rest = rest
            self.g_grid = [torch.zeros_like(g.data, dtype=torch.float32) for g in self.grid]
            self.g_dens, self.g_col = torch.zeros_like(self.dens_flat), torch.zeros_like(self.col_flat)
            self.g_rest = [torch.zeros_like(p.data) for p in rest]
        else:
            named = list(nef.named_parameters())
            tensors = [(p.data, lr * grid_lr_weight if ("grid" in n and "decoder" not in n) else lr, weight_decay if "decoder" in n else 0.0)
                       for n, p in named if p.requires_grad]
            self.params = [p for _, p in named if p.requires_grad]
        self.opt = _make_optimizer(optimizer, tensors, betas, eps, alpha, momentum)
        self.milestones, self.gamma = [int(m) for m in scheduler_milestones], float(scheduler_gamma)
        if any(m != f for m, f in zip(self.milestones, scheduler_milestones)):
            raise ValueError(f"scheduler_milestones are iteration numbers (ints), got {scheduler_milestones!r}")
        dev = tensors[0][0].device
        self._scalars = torch.zeros(2, dtype=torch.float32, device=dev)       # loss accumulator | max |g_shaded|: cleared by ONE fill per step
        self.loss_buf, self.absmax = self._scalars[0:1], self._scalars[1:2]
        self.scale = torch.ones(1, dtype=torch.float32, device=dev)
        self.last_stage = {}
        self._cl = None                                                        # triplanar planes: channel-last copies + gradient accumulators

    # ---- helpers -------------------------------------------------------------------------------------------------------
    def _world(self) -> int:
        return dist.get_world_size(self.group) if (dist.is_available() and dist.is_initialized()) else 1

    def _march(self, rays: Rays, seed: int):
        grid, tr = self.nef.grid, self.tracer
        pm = tr._pending.pop(tr._march_key(rays, seed, tr.num_steps, grid.blas), None) if (tr.raymarch_type == 'ray' and tr._pending) else None
        return pm.finalize() if pm is not None else ops.march(grid, len(grid.active_lods) - 1, rays, tr.raymarch_type, tr.num_steps, seed=seed)

    # ---- the step ------------------------------------------------------------------------------------------------------
    def step(self, rays: Rays, img_gts: torch.Tensor, seed: Optional[int] = None, next_rays: Optional[Rays] = None, next_seed: Optional[int] = None,
             next_ready=None, zero_grad: bool = True, local_only: bool = False, update: bool = True) -> torch.Tensor:
        """One optimisation step on (rays, img_gts [R,3]); returns the loss as a device scalar (no host sync).  `next_rays` (+ seed)
        lets the march of the following batch overlap this step (PackedRFTracer.premarch).  `update=False` stops after the backward
        (gradients left in g_grid / g_dens / g_col, parameters and optimiser state untouched: gradient checks, bench.py's parity leg)."""
        tr = self.tracer
        if seed is None:
            seed = tr.seed
            tr.seed = (tr.seed + 1) & 0x7FFFFFFF
        if next_rays is not None and tr.raymarch_type == 'ray':
            tr.premarch(self.nef, next_rays, tr.seed if next_seed is None else next_seed, ready=next_ready)
        world = 1 if local_only else self._world()      # local_only: no collective, loss normalised by this rank's rays (diagnostics)
        if not self.fused:
            return self._step_autograd(rays, img_gts, seed, world)
        L = A.lib()
        nef, spec = self.nef, self.spec
        dev = self.dens_flat.device
        ms = self._march(rays, seed)
        tr.prev_num_samples = ms.total
        S, R = ms.total, ms.rays.num_rays
        precision = ops.resolve_precision(self.precision if self.precision is not None else tr.precision, spec, nef, True)
        gt = [t.data for t in self.grid]
        g_used = self.g_grid
        layout = 1 if ops.triplane_wants_channel_last(spec) else 0
        if layout:          # channel-last copies of the planes for this step; their gradients are accumulated channel-last and converted back below
            if self._cl is None:
                self._cl = ([torch.empty((t.shape[2], t.shape[3], t.shape[1]), dtype=torch.float32, device=dev) for t in gt],
                            [torch.zeros((t.shape[2], t.shape[3], t.shape[1]), dtype=torch.float32, device=dev) for t in gt])
            gt = ops.triplane_relayout(gt, True, out=self._cl[0])
            g_used = self._cl[1]
        oct, trinkets = ops._grid_context(nef, spec)
        desc, keep = spec.desc(gt, self.dens_flat, self.col_flat, oct, trinkets, grads=g_used, layout=layout)
        blob = torch.empty(int(L.wb_rf_param_blob_floats(C.byref(desc), C.c_int32(precision))), dtype=torch.float32, device=dev)
        A.check(L.wb_rf_pack_params(C.byref(desc), C.c_int32(precision), A.ptr(blob), A.stream()))
        rec_t, rec_delta, rec_ray = ops.march_fill_records(ms, dev)
        Scap = ops._bucket(S)
        shaded = ops._empty_s(S, (4,), torch.float32, dev)
        g_sh = ops._empty_s(S, (4,), torch.float32, dev)
        wsb = int(L.wb_rf_workspace_bytes(C.byref(desc), C.c_int32(precision), C.c_int64(R), C.c_int64(Scap), C.c_int32(1)))
        fb = int(L.wb_rf_feat_bytes(C.byref(desc), C.c_int32(precision), C.c_int64(Scap)))
        if wsb < 0 or fb < 0:
            raise A.WispB200Error(L.wb_last_error().decode())
        ws = torch.empty(wsb, dtype=torch.uint8, device=dev) if wsb > 0 else None
        feat = torch.empty(fb, dtype=torch.uint8, device=dev) if fb > 0 else None
        rgb = torch.empty((R, 3), dtype=torch.float32, device=dev)
        alpha = torch.empty((R, 1), dtype=torch.float32, device=dev)
        hit = torch.empty(R, dtype=torch.bool, device=dev)
        tr.bg_color = tr.bg_color.to(dev)
        bgv = ops._bg3(tr.bg_color)
        tgt = A.f32c(img_gts)
        with ops._stage("shade_fwd"):
            A.check(L.wb_rf_shade_fwd(C.byref(desc), A.ptr(blob), C.c_int32(precision), C.byref(ms.rays), A.ptr(rec_t), A.ptr(rec_ray), C.c_int64(S),
                                      A.ptr(shaded), A.ptr(feat), A.ptr(ws), A.stream()))
        with ops._stage("composite_fwd"):
            A.check(L.wb_composite_fwd(A.ptr(shaded), A.ptr(rec_t), A.ptr(rec_delta), A.ptr(ms.offsets), C.c_int64(R), bgv, A.ptr(rgb), None, A.ptr(alpha),
                                       A.ptr(hit), A.stream()))
        self._scalars.zero_()
        # rgb_loss.mean() over the GLOBAL batch (SURVEY 8(e)): every rank contributes sum / (3 * R * world); 'samples' divides by the local count
        inv = 1.0 / (3.0 * R * world) if self.loss_denom == "rays" else 1.0 / (max(S, 1) * world)
        with ops._stage("composite_bwd"):
            A.check(L.wb_composite_bwd_loss(A.ptr(shaded), A.ptr(rec_t), A.ptr(rec_delta), A.ptr(ms.offsets), C.c_int64(R), bgv, A.ptr(rgb), A.ptr(tgt),
                                            C.c_int32(LOSS_TYPES[self.loss_type]), C.c_float(inv), A.ptr(g_sh), A.ptr(self.absmax), A.ptr(self.loss_buf), A.stream()))
        g_table = g_used[0] if spec.kind == "hash" else None
        if S > 0:
            if precision == 1:
                A.check(L.wb_rf_loss_scale(A.ptr(self.absmax), A.ptr(self.scale), A.stream()))
                L.wb_rf_workspace_holds_ray_rows(C.c_int32(1))      # same workspace, same rays as the forward above
            with ops._stage("shade_bwd"):      # precision 1: decoder backward + table scatter in one kernel where the shape allows
                A.check(L.wb_rf_shade_bwd(C.byref(desc), A.ptr(blob), C.c_int32(precision), C.byref(ms.rays), A.ptr(rec_t), A.ptr(rec_ray), C.c_int64(S), A.ptr(g_sh),
                                          A.ptr(self.scale) if precision == 1 else None, A.ptr(feat), A.ptr(ws), A.ptr(g_table), A.ptr(self.g_dens), A.ptr(self.g_col), A.stream()))
        if layout:          # -> self.g_grid (reference layout, overwritten with the accumulated channel-last gradients)
            ops.triplane_relayout(g_used, False, out=self.g_grid)
        self.last_rgb, self.last_alpha, self.last_hit = rgb, alpha, hit
        loss = self.loss_buf.clone()
        if world > 1:
            with ops._stage("all_reduce"):
                self._all_reduce(loss)
        if update:
            self.opt.lr_scale = multistep_factor(self.milestones, self.gamma, self.opt.t + 1)
            with ops._stage("adam"):
                self.opt.step(self.g_grid + [self.g_dens, self.g_col] + self.g_rest, grad_scale=1.0, zero_grad=zero_grad)
            if layout and zero_grad:
                torch._foreach_zero_(g_used)
        return loss[0]

    def zero_grads(self) -> None:
        """Clear every gradient accumulator (after a step(update=False) whose gradients were only inspected)."""
        for g in self.g_grid + [self.g_dens, self.g_col] + self.g_rest + (self._cl[1] if self._cl is not None else []):
            g.zero_()

    def _all_reduce(self, loss):
        """Gradient exchange of data-parallel training (SURVEY 8(e)): sum over ranks (the mean's 1/world is already in the loss
        gradient: inv_count uses the global ray count).  Decoder gradients + the loss share one small collective."""
        small = torch.cat([self.g_dens, self.g_col, loss] + [g.reshape(-1) for g in self.g_rest])
        dist.all_reduce(small, op=dist.ReduceOp.SUM, group=self.group)
        for g in self.g_grid:
            dist.all_reduce(g, op=dist.ReduceOp.SUM, group=self.group)
        o = 0
        for t in [self.g_dens, self.g_col, loss] + [g.reshape(-1) for g in self.g_rest]:
            t.copy_(small[o:o + t.numel()].view_as(t)); o += t.numel()

    def _step_autograd(self, rays, img_gts, seed, world):
        for p in self.params:
            p.grad = None
        self.tracer.seed = seed
        rb = self.pipeline(rays=rays, lod_idx=None, channels=["rgb"])
        d = rb.rgb - img_gts
        if self.loss_type == "l2":
            l = torch.nn.functional.mse_loss(rb.rgb, img_gts, reduction='none')
        elif self.loss_type == "l1":
            l = torch.abs(d)
        else:
            l = torch.nn.functional.smooth_l1_loss(rb.rgb, img_gts, reduction='none')
        loss = l.mean() if self.loss_denom == "rays" else l.sum() / max(self.tracer.prev_num_samples, 1)
        loss.backward()
        grads = [p.grad if p.grad is not None else torch.zeros_like(p) for p in self.params]
        grads = [g.contiguous() for g in grads]
        if world > 1:
            for g in grads:
                dist.all_reduce(g, op=dist.ReduceOp.SUM, group=self.group)
        self.opt.lr_scale = multistep_factor(self.milestones, self.gamma, self.opt.t + 1)
        self.opt.step(grads, grad_scale=1.0 / world, zero_grad=False)
        return loss.detach()


class SDFStep:
    """The optimisation step of wisp.trainers.SDFTrainer (wisp/trainers/sdf_trainer.py:65-124) with the optimiser of
    BaseTrainer.init_optimizer (wisp/trainers/base_trainer.py:205-239): parameter groups by name ('decoder' -> weight decay,
    'grid' -> lr * grid_lr_weight, the rest -> lr; parameters with requires_grad=False are skipped, as torch.optim.Adam skips
    them), loss = sum over loss_lods of sum((pred - gt)^2), divided by the batch size.  loss_lods is the last LOD when
    `only_last` (nglod_octree.yaml), otherwise every LOD.

    A NeuralSDF with 1 to 4 hidden layers over an OctreeGrid (every app/nglod octree config, with any nef.num_layers up to 4) or
    over a 3D HashGrid of 4 or 8 features per LOD (nglod_hash.yaml) trains natively: per loss LOD one wb_sdf_train launch
    (forward, loss and backward, no autograd), then NativeAdam over every parameter in one launch.  The decoder's parameters are
    flattened in place into one buffer [W0, b0, W1, b1, ..., Wout, bout], which the kernel reads, whose gradient it writes and
    which is one Adam segment; the grid's tensors (OctreeGrid.features, or the one HashGrid codebook.feats table) are the other
    segments.  Every other field (NeuralSDF over a TriplanarGrid, a hash grid of F = 2 or over 8 features, a deeper decoder whose
    weights, weight-gradient accumulators and smallest sample tile exceed an SM's shared memory: wb_sdf_train_smem_bytes < 0)
    takes autograd plus the same NativeAdam.

    `precision` picks the arithmetic, whatever the autocast state:
      0  fp32 decoder (wb_sdf_train; autograd in fp32); the reference's enable_amp fp16 nn.Linear is not reproduced.
      1  the reference's enable_amp arithmetic (every app/nglod config sets enable_amp: True; BaseTrainer runs the step under
         torch.cuda.amp.autocast, base_trainer.py:338): hash fields the native route trains whose tensor-core footprint fits
         (wb_sdf_train_tc_smem_bytes >= 0: one or two hidden layers of 128, any 1-4 layers narrower) take one wb_sdf_train_tc
         launch per loss LOD (fp16 decoder operands and outputs on the tensor cores, fp32 gradients), then the same NativeAdam;
         the hash table stays fp32 (the reference casts it to fp16).  Every other field, octree fields included (the kernel
         trains them through ops.sdf_train, but measured slower than autocast autograd at large batches), takes autograd inside
         torch.autocast("cuda", torch.float16) plus NativeAdam.
    `optimizer`: "adam" | "adamw" | "rmsprop" replaces NativeAdam by NativeAdamW or NativeRMSprop(alpha, momentum) on either route,
    with the same parameter groups.  No learning-rate schedule: SDFTrainer.step never steps one.
    `fused` tells which route was chosen."""

    def __init__(self, pipeline, lr: float = 1e-3, eps: float = 1e-15, weight_decay: float = 0.0, grid_lr_weight: float = 1.0,
                 betas=(0.9, 0.999), only_last: bool = True, precision: int = 0, optimizer: str = "adam", alpha: float = 0.99,
                 momentum: float = 0.0):
        if precision not in (0, 1) or isinstance(precision, bool):
            raise ValueError(f"SDFStep: precision must be 0 (fp32) or 1 (fp16 autocast arithmetic), got {precision!r}")
        self.precision = int(precision)
        self.pipeline, self.nef = pipeline, pipeline.nef
        nef = self.nef
        n = int(nef.grid.num_lods)
        self.loss_lods = [n - 1] if only_last else list(range(n))            # sdf_trainer.py:55-58
        named = [(k, p) for k, p in nef.named_parameters() if p.requires_grad]
        if not named:
            raise A.WispB200Error("SDFStep: the field has no trainable parameters")
        A.require_device(named[0][1])                                         # no CPU fallback
        self.device = named[0][1].device
        self.fd = self._fused_field(nef, [p for _, p in named])
        self.fused = self.fd is not None
        if self.fused:
            feats = self._grid_tensors(nef.grid)
            tensors = [(f.data, lr * grid_lr_weight, 0.0) for f in feats] + [(self.dec_flat, lr, weight_decay)]
            self.g_feats = [torch.zeros_like(f.data) for f in feats]
            self.g_dec = torch.zeros_like(self.dec_flat)
        else:
            tensors = [(p.data, lr if "decoder" in k or "grid" not in k else lr * grid_lr_weight, weight_decay if "decoder" in k else 0.0)
                       for k, p in named]
            self.params = [p for _, p in named]
        self.opt = _make_optimizer(optimizer, tensors, betas, eps, alpha, momentum)
        self.loss_buf = torch.zeros(1, dtype=torch.float32, device=self.device)

    @staticmethod
    def _grid_tensors(grid):
        """The grid tensors wb_sdf_train writes gradients for: OctreeGrid.features, or HashGrid's one codebook.feats table."""
        cb = getattr(grid, "codebook", None)
        if hasattr(cb, "feats") and not hasattr(grid, "features"):
            return [cb.feats]
        return list(getattr(grid, "features", []))

    def _fused_field(self, nef, params):
        """ops.sdf_field of the field with the decoder flattened in place and the description aimed at that buffer, or None when
        the field is outside wb_sdf_train (precision 1: wb_sdf_train_tc): neither an OctreeGrid nor a hash grid in ops.sdf_field's
        range, a decoder whose training footprint exceeds shared memory, or trainable parameters beyond grid and decoder."""
        grid, dec = getattr(nef, "grid", None), getattr(nef, "decoder", None)
        if grid is None or dec is None or getattr(grid, "dictionary", None) is not None:
            return None
        feats = self._grid_tensors(grid)
        if not feats or any(not isinstance(f, torch.Tensor) or f.dim() != 2 or f.shape[1] != grid.feature_dim or f.dtype != torch.float32 or not f.is_contiguous() for f in feats):
            return None
        dparams = ops.decoder_params(dec)
        if {id(p) for p in params} != {id(p) for p in feats + dparams} or any(p.dtype != torch.float32 for p in dparams):
            return None
        fd = ops.sdf_field(nef)
        smem = ops.sdf_train_tc_smem_bytes if self.precision == 1 else ops.sdf_train_smem_bytes
        if fd is None or smem(fd) < 0:
            return None
        if self.precision == 1 and not fd[0].hash:
            return None               # octree fields: wb_sdf_train_tc is slower than autograd under autocast (DESIGN section 7)
        self.dec_flat = _flatten_in_place(dparams)
        fd = ops.sdf_field(nef)
        d, oct, keep = fd
        if (d.hash.contents.table != feats[0].data_ptr()) if d.hash else any(d.feats[k] != f.data_ptr() for k, f in enumerate(feats)):
            return None
        d.params = self.dec_flat.data_ptr()
        return d, oct, keep + [self.dec_flat]

    def _lod_check(self, N: int) -> None:
        g = self.nef.grid
        # an octree 'cat' grid feeds the decoder only LODs 0..lod_idx; a hash 'cat' grid keeps its width and zeroes LODs >= lod_idx
        if self.fused and not self.fd[0].hash and g.multiscale_type == 'cat' and min(self.loss_lods) < g.num_lods - 1:
            lin = self.nef.decoder.layers[0]
            pd = lin.in_features - g.feature_dim * g.num_lods
            k = min(self.loss_lods)
            raise RuntimeError(f"mat1 and mat2 shapes cannot be multiplied ({N}x{pd + g.feature_dim * (k + 1)} and "
                               f"{lin.in_features}x{lin.out_features})")      # what nn.Linear raises on a lower LOD of a 'cat' grid

    def step(self, coords: torch.Tensor, sdf_gt: torch.Tensor, zero_grad: bool = True, update: bool = True) -> torch.Tensor:
        """One optimisation step on (coords [N,3], sdf_gt [N,1]); returns the loss as a device scalar (no host sync).  Host tensors
        are copied to the device (`.to(self.device)`, sdf_trainer.py:69-70).  `update=False` stops after the backward: the
        gradients stay in g_feats / g_dec (autograd route: in the parameters' .grad), parameters and optimiser state untouched."""
        pts, gts = coords.to(self.device), sdf_gt.to(self.device)
        N = int(pts.shape[0])
        if N == 0:
            raise A.WispB200Error("SDFStep.step: empty batch (the reference divides the loss by the batch size)")
        self._lod_check(N)
        if not self.fused:
            return self._step_autograd(pts, gts, N, update)
        c, g = A.f32c(pts).reshape(-1, 3), A.f32c(gts).reshape(-1)
        self.loss_buf.zero_()
        for lod in self.loss_lods:
            ops.sdf_train(self.fd, c, g, lod, 1.0 / N, self.g_feats, self.g_dec, self.loss_buf, precision=self.precision)
        loss = self.loss_buf.clone()
        if update:
            with ops._stage("adam"):
                self.opt.step(self.g_feats + [self.g_dec], grad_scale=1.0, zero_grad=zero_grad)
        return loss[0]

    def zero_grads(self) -> None:
        """Clear every gradient accumulator (after a step(update=False) whose gradients were only inspected)."""
        if self.fused:
            for t in self.g_feats + [self.g_dec]:
                t.zero_()
        else:
            for p in self.params:
                p.grad = None

    def _step_autograd(self, pts, gts, N, update):
        for p in self.params:
            p.grad = None                                                     # self.pipeline.zero_grad() (:77)
        loss = 0.0
        amp = torch.autocast("cuda", torch.float16) if self.precision == 1 else contextlib.nullcontext()
        with amp:                                                             # base_trainer.py:338 with enable_amp
            for lod in self.loss_lods:
                pred = self.nef(coords=pts, lod_idx=lod, channels="sdf")
                loss = loss + ((pred - 1.0 * gts) ** 2).sum()
            loss = loss / N
        loss.backward()
        if update:
            grads = [(p.grad if p.grad is not None else torch.zeros_like(p)).contiguous() for p in self.params]
            self.opt.step(grads, grad_scale=1.0, zero_grad=False)
        return loss.detach()


class ImageStep:
    """The optimisation step of wisp.trainers.ImageTrainer (wisp/trainers/image_trainer.py:51-80): loss = F.mse_loss(nef.rgb(coords),
    rgb), the mean over N * 3, one optimiser step, then the MultiStepLR step of `scheduler: True`.  Parameter groups of
    BaseTrainer.init_optimizer (base_trainer.py:205-246): 'decoder' -> lr and weight_decay, 'grid' -> lr * grid_lr_weight, the rest -> lr;
    parameters with requires_grad=False (embedder.bands) are skipped.

    An ImageNeuralField over a hash grid of 2, 4 or 8 features per LOD with one hidden layer (image_hash.yaml) trains natively in two
    launches per step: wb_image_train (forward, loss and backward, no autograd) and the optimiser (wb_adamw_step by default: apex
    FusedAdam's adam_w_mode), which also clears the gradients and applies the schedule's factor.  The decoder's parameters are flattened
    in place into one buffer [W0, b0, Wout, bout], which the kernels read, whose gradient wb_image_train writes and which is one
    optimiser segment; grid.codebook.feats is the other.  Every other field (deeper decoders, other grids or embedders, a decoder input
    wider than the kernel's shared-memory image: ops.image_field is None) takes autograd plus the same native optimiser.

    `precision`: 0 fp32 (the native route above); 1 the reference's enable_amp arithmetic, which runs the autograd route inside
    torch.autocast("cuda", torch.float16) (no tensor-core image kernel) with the same native optimiser and no GradScaler.
    `optimizer`: "adamw" (FusedAdam), "adam" or "rmsprop".
    `scheduler_milestones` / `scheduler_gamma`: MultiStepLR stepped after every optimiser step, as MultiviewStep takes them: iteration
    numbers; step t (1-based) runs at lr * gamma^k, k = the number of milestones <= t - 1.  The reference hands MultiStepLR
    max_steps * (0.5, 0.75, 0.9), which fire only where that product is integer-valued.  `fused` tells which route was chosen."""

    def __init__(self, pipeline, lr: float = 1e-3, eps: float = 1e-15, weight_decay: float = 0.0, grid_lr_weight: float = 1.0,
                 betas=(0.9, 0.999), optimizer: str = "adamw", scheduler_milestones=(), scheduler_gamma: float = 0.333, precision: int = 0):
        if precision not in (0, 1) or isinstance(precision, bool):
            raise ValueError(f"ImageStep: precision must be 0 (fp32) or 1 (fp16 autocast arithmetic), got {precision!r}")
        self.precision = int(precision)
        self.pipeline, self.nef = pipeline, pipeline.nef
        nef = self.nef
        named = [(k, p) for k, p in nef.named_parameters() if p.requires_grad]
        if not named:
            raise A.WispB200Error("ImageStep: the field has no trainable parameters")
        A.require_device(named[0][1])                                         # no CPU fallback
        self.device = named[0][1].device
        self.fd = self._fused_field(nef, [p for _, p in named]) if self.precision == 0 else None
        self.fused = self.fd is not None
        if self.fused:
            table = nef.grid.codebook.feats
            tensors = [(table.data, lr * grid_lr_weight, 0.0), (self.dec_flat, lr, weight_decay)]
            self.g_table = torch.zeros_like(table.data)
            self.g_dec = torch.zeros_like(self.dec_flat)
        else:
            tensors = [(p.data, lr if "decoder" in k or "grid" not in k else lr * grid_lr_weight, weight_decay if "decoder" in k else 0.0)
                       for k, p in named]
            self.params = [p for _, p in named]
        self.opt = _make_optimizer(optimizer, tensors, betas, eps, 0.99, 0.0)
        self.milestones, self.gamma = [int(m) for m in scheduler_milestones], float(scheduler_gamma)
        if any(m != f for m, f in zip(self.milestones, scheduler_milestones)):
            raise ValueError(f"scheduler_milestones are iteration numbers (ints), got {scheduler_milestones!r}")

    def _fused_field(self, nef, params):
        """ops.image_field of the field with the decoder flattened in place, or None when wb_image_train does not take the field or the
        field has trainable parameters beyond codebook.feats and the decoder."""
        if ops.image_field(nef) is None:
            return None
        dparams = ops.decoder_params(nef.decoder)
        if {id(p) for p in params} != {id(p) for p in [nef.grid.codebook.feats] + dparams}:
            return None
        self.dec_flat = _flatten_in_place(dparams)
        fd = ops.image_field(nef)
        if fd is None or fd[2][0] != self.dec_flat.data_ptr():
            return None
        return fd

    def step(self, coords: torch.Tensor, rgb: torch.Tensor, zero_grad: bool = True, update: bool = True) -> torch.Tensor:
        """One optimisation step on (coords [N, 2], rgb [N, 3]); returns the loss as a device scalar (no host sync).  Host tensors are
        copied to the device (image_trainer.py:53-54).  `update=False` stops after the backward: the gradients stay in g_table / g_dec
        (autograd route: in the parameters' .grad), parameters, optimiser state and schedule untouched."""
        pts, gts = coords.to(self.device), rgb.to(self.device)
        if int(pts.shape[0]) == 0:
            raise A.WispB200Error("ImageStep.step: empty batch (mse_loss averages over it)")
        if not self.fused:
            return self._step_autograd(pts, gts, update)
        loss = torch.zeros(1, dtype=torch.float32, device=self.device)
        ops.image_train(self.fd, A.f32c(pts).reshape(-1, 2), A.f32c(gts).reshape(-1, 3), len(self.nef.grid.resolutions) - 1,
                        self.g_table, self.g_dec, loss)
        if update:
            self.opt.lr_scale = multistep_factor(self.milestones, self.gamma, self.opt.t + 1)
            with ops._stage("adam"):
                self.opt.step([self.g_table, self.g_dec], grad_scale=1.0, zero_grad=zero_grad)
        return loss[0]

    def zero_grads(self) -> None:
        """Clear every gradient accumulator (after a step(update=False) whose gradients were only inspected)."""
        if self.fused:
            self.g_table.zero_()
            self.g_dec.zero_()
        else:
            for p in self.params:
                p.grad = None

    def _step_autograd(self, pts, gts, update):
        for p in self.params:
            p.grad = None                                                     # self.optimizer.zero_grad() (:61)
        amp = torch.autocast("cuda", torch.float16) if self.precision == 1 else contextlib.nullcontext()
        with amp:                                                             # image_trainer.py:64 with enable_amp
            loss = torch.nn.functional.mse_loss(self.nef.rgb(pts), gts)
        loss.backward()
        if update:
            grads = [(p.grad if p.grad is not None else torch.zeros_like(p)).float().contiguous() for p in self.params]
            self.opt.lr_scale = multistep_factor(self.milestones, self.gamma, self.opt.t + 1)
            self.opt.step(grads, grad_scale=1.0, zero_grad=False)
        return loss.detach().float()
