"""PackedRFTracer / PackedSDFTracer: host-side mirrors of wisp.tracers.PackedRFTracer (wisp/tracers/packed_rf_tracer.py:20-181),
wisp.tracers.PackedSDFTracer (wisp/tracers/packed_sdf_tracer.py:20-174) and wisp.tracers.BaseTracer.forward
(wisp/tracers/base_tracer.py:99-162).  PackedRFTracer.trace() runs the fused native pipeline when the neural field is a
NeuralRadianceField(HashGrid) with the 'ray' sampler, and otherwise the unfused route (native raymarch + nef forward + native
compositing)."""
from __future__ import annotations

import inspect
from typing import Optional

import torch
import torch.nn as nn

from . import ops
from .core import RenderBuffer


class BaseTracer(nn.Module):
    def forward(self, nef, rays, channels=None, **kwargs):
        """base_tracer.py:99-162: channel negotiation, kwargs default to tracer attributes of the same name."""
        nef_channels = nef.get_supported_channels()
        unsupported_inputs = self.get_required_nef_channels() - nef_channels
        if unsupported_inputs:
            raise Exception(f"The neural field class {type(nef)} does not output the required channels {unsupported_inputs}.")
        requested = self.get_supported_channels() if channels is None else {channels} if isinstance(channels, str) else set(channels)
        extra = requested - self.get_supported_channels()
        unsupported_outputs = extra - nef_channels
        if unsupported_outputs:
            raise Exception(f"Channels {unsupported_outputs} are not supported in the tracer {type(self)} or neural field {type(nef)}.")
        input_args = {}
        for a in list(inspect.signature(self.trace).parameters)[4:]:
            if a in kwargs:
                input_args[a] = kwargs[a]
            else:
                d = getattr(self, a, None)
                if d is not None:
                    input_args[a] = d
        return self.trace(nef, rays, requested, extra, **input_args)


class PackedRFTracer(BaseTracer):
    def __init__(self, raymarch_type='ray', num_steps=1024, step_size=1.0, bg_color=(1.0, 1.0, 1.0)):
        super().__init__()
        self.raymarch_type, self.num_steps, self.step_size = raymarch_type, num_steps, step_size
        self.bg_color = torch.tensor(bg_color, dtype=torch.float32)
        self.prev_num_samples = None
        # decoder arithmetic of the fused path: 0 = fp32 (autocast off), 1 = fp16 tensor cores with fp32 accumulation (what the
        # reference runs under `enable_amp: True`, base_trainer.py autocast); None = follow torch.is_autocast_enabled()
        self.precision = None
        self.seed = 0               # base of the counter-based jitter stream; advanced once per trace() call
        self.jitter = None          # optional explicit [R, num_steps] jitter (parity tests)
        self._pending = {}          # pre-marched batches (premarch), keyed by (origins ptr, dirs ptr, num rays, seed, num_steps)
        self._march_stream = None

    def __getstate__(self):                                  # deepcopy / pickle: streams and in-flight marches are not state
        d = self.__dict__.copy()
        d["_pending"], d["_march_stream"] = {}, None
        return d

    def premarch(self, nef, rays, seed: int, num_steps: Optional[int] = None, ready=None):
        """Enqueue the ray march of a FUTURE batch on a side stream.  Sample selection depends only on the rays, the occupancy
        structure and the jitter seed -- not on the weights -- so the march (and its sample-count read-back, the one host sync
        of the path) of batch i+1 can overlap the shading / backward / optimiser step of batch i.  The matching trace() call
        (same ray tensors, same seed, 'ray' marching) picks the result up; anything else ignores it.  Do not prune() in between."""
        blas = nef.grid.blas
        n = self.num_steps if num_steps is None else num_steps
        dev = rays.origins.device
        if self._march_stream is None:
            self._march_stream = torch.cuda.Stream(device=dev)
        cur = torch.cuda.current_stream(dev)
        level = ops.raymarch_level(nef.grid, nef.grid.num_lods - 1)
        oct = ops.octree_tensors(blas)
        oct.ensure_bits(level)                              # built on the caller's stream BEFORE the side stream starts waiting on it
        self._march_stream.wait_stream(cur)                 # the rays (and octree masks) are ready on the caller's stream ...
        if ready is not None:
            self._march_stream.wait_event(ready)            # ... or when `ready` fires (e.g. HostPrefetcher.staged_event)
        with torch.cuda.stream(self._march_stream):
            key = (rays.origins.shape[0], n)
            if getattr(self, "_primed", None) != key:
                # first pre-march of this shape: reserve four sets of march buffers in the side stream's allocator pool, so that
                # the steady state (one set being filled, one consumed, up to two waiting for their cross-stream events to retire)
                # never calls cudaMalloc (three sets left an occasional cudaMalloc in a timed step, BENCH_r01)
                R, nw = key[0], (n + 31) // 32
                spare = [(torch.empty((R, nw), dtype=torch.int32, device=dev), torch.empty(R, dtype=torch.int32, device=dev),
                          torch.empty(R + 1, dtype=torch.int64, device=dev)) for _ in range(4)]
                del spare
                self._primed = key
            pm = ops.march_count(oct, rays.origins, rays.dirs, rays.dist_min, rays.dist_max, n, level,
                                 seed=seed, defer_total=True)
        for t in (rays.origins, rays.dirs):
            t.record_stream(self._march_stream)
        if len(self._pending) >= 4:
            self._pending.clear()
        self._pending[self._march_key(rays, seed, n, blas)] = pm

    @staticmethod
    def _march_key(rays, seed, n, blas):
        """Identity of a pre-marched batch: the ray tensors (storage + version: an in-place overwrite invalidates it), the ray
        interval, the jitter seed, the step count and the occupancy structure (object + its octree storage, which prune() replaces)."""
        nf = tuple((x.data_ptr(), x._version) if torch.is_tensor(x) else float(x) for x in (rays.dist_min, rays.dist_max))
        return (rays.origins.data_ptr(), rays.dirs.data_ptr(), rays.origins._version, rays.dirs._version, rays.origins.shape[0], nf,
                seed & 0xFFFFFFFF, n, id(blas), blas.octree.data_ptr())

    def get_prev_num_samples(self):
        return self.prev_num_samples

    def get_supported_channels(self):
        return {"depth", "hit", "rgb", "alpha"}

    def get_required_nef_channels(self):
        return {"rgb", "density"}

    def trace(self, nef, rays, channels, extra_channels, lod_idx=None, raymarch_type='voxel', num_steps=64, step_size=1.0, bg_color='white'):
        """packed_rf_tracer.py:84-181.  Like the reference, the body reads self.bg_color, not the bg_color argument."""
        assert nef.grid is not None and "this tracer requires a grid"
        N = rays.origins.shape[0]
        if lod_idx is None:
            lod_idx = nef.grid.num_lods - 1
        dev = rays.origins.device
        self.bg_color = self.bg_color.to(dev)
        jitter, seed = self.jitter, self.seed
        self.seed = (self.seed + 1) & 0x7FFFFFFF
        spec = nef.fused_spec(lod_idx) if hasattr(nef, "fused_spec") else None
        if raymarch_type not in ('ray', 'voxel', 'uniform'):
            raise TypeError(f"Raymarch sampler type: {raymarch_type} is not supported by OctreeAS.")       # octree_as.py:427
        if spec is not None and not extra_channels:
            pm = None
            if raymarch_type == 'ray' and self._pending and jitter is None:
                pm = self._pending.pop(self._march_key(rays, seed, num_steps, nef.grid.blas), None)
            ms = pm.finalize() if pm is not None else ops.march(nef.grid, lod_idx, rays, raymarch_type, num_steps, jitter=jitter, seed=seed)
            self.prev_num_samples = ms.total
            # read by resolve_precision only when it follows autocast: the parameter scan runs only then
            need_bwd = self.precision is None and torch.is_autocast_enabled() and torch.is_grad_enabled() and any(p.requires_grad for p in nef.parameters())
            rgb, depth, alpha, hit = ops.rf_trace_nef(ms, spec, nef, self.bg_color, precision=ops.resolve_precision(self.precision, spec, nef, need_bwd))
            return RenderBuffer(depth=depth if "depth" in channels else None, hit=hit, rgb=rgb, alpha=alpha)

        # ---- unfused route: same operators, nef evaluated through its own forward() ----
        mr = nef.grid.raymarch(rays, level=nef.grid.active_lods[lod_idx], num_samples=num_steps, raymarch_type=raymarch_type,
                               jitter=jitter, seed=seed)
        ridx, samples, deltas, depths, boundary = mr.ridx, mr.samples, mr.deltas, mr.depth_samples, mr.boundary
        self.prev_num_samples = samples.shape[0]
        num_samples = samples.shape[0]
        hit_ray_d = rays.dirs.index_select(0, ridx)
        color, density = nef(coords=samples, ray_d=hit_ray_d, lod_idx=lod_idx, channels=["rgb", "density"])
        density = density.reshape(num_samples, 1)
        counts = torch.bincount(ridx, minlength=N)
        offsets = torch.zeros(N + 1, dtype=torch.int64, device=dev)
        offsets[1:] = torch.cumsum(counts, 0)
        shaded = torch.cat([color.float(), density.float()], -1)
        rgb, depth, alpha, hit = ops.CompositeFn.apply(shaded, depths, deltas, offsets, self.bg_color)
        extra_outputs = {}
        for channel in extra_channels:
            feats = nef(coords=samples, ray_d=hit_ray_d, lod_idx=lod_idx, channels=channel)
            nc = feats.shape[-1]
            outs = []
            for c0 in range(0, nc, 3):                      # integrate 3 channels at a time through the same kernel
                chunk = feats[:, c0:c0 + 3].float()
                pad = torch.zeros(num_samples, 3 - chunk.shape[1], device=dev)
                f3, _, _, _ = ops.CompositeFn.apply(torch.cat([chunk, pad, density.float()], -1), depths, deltas, offsets, (0.0, 0.0, 0.0))
                outs.append(f3[:, :chunk.shape[1]])
            extra_outputs[channel] = alpha * torch.cat(outs, -1)   # packed_rf_tracer.py:176
        return RenderBuffer(depth=depth if "depth" in channels else None, hit=hit, rgb=rgb, alpha=alpha, **extra_outputs)


class PackedSDFTracer(BaseTracer):
    """wisp.tracers.PackedSDFTracer (packed_sdf_tracer.py:20-174): sphere tracing over the nugget list of OctreeAS.raytrace with
    find_depth_bound jumping between occupied cells; normals by central differences.  The reference's Python loop of masked
    torch ops is one persistent cooperative kernel here (csrc/wb_sdf.cu)."""

    def __init__(self, num_steps=64, step_size=1.0, min_dis=1e-4):
        super().__init__()
        self.num_steps, self.step_size, self.min_dis = num_steps, step_size, min_dis

    def get_supported_channels(self):
        return {"depth", "normal", "xyz", "hit", "rgb", "alpha"}

    def get_required_nef_channels(self):
        return {"sdf"}

    def trace(self, nef, rays, channels, extra_channels, lod_idx=None, num_steps=64, step_size=1.0, min_dis=1e-4):
        """packed_sdf_tracer.py:57-174.  The nuggets come from the native raytrace; the sphere-tracing loop, the nugget cursor
        and the finite-difference normals are ONE persistent kernel (ops.sdf_trace -> wb_sdf_trace) for NeuralSDF(OctreeGrid);
        for other fields the per-pack state machine still runs natively and only the field is evaluated through its forward().
        install() runs this body on the reference's PackedSDFTracer too."""
        assert nef.grid is not None and "this tracer requires a grid"
        if lod_idx is None:
            lod_idx = nef.grid.num_lods - 1
        want_normals = "rgb" in channels or "normal" in channels
        out, st = ops.sdf_trace(nef, ops.octree_tensors(nef.grid.blas), rays.origins, rays.dirs, rays.dist_max, ops.raytrace_level(nef.grid, lod_idx), lod_idx,
                                num_steps, step_size, min_dis, want_normals)
        hit = out["hit"]
        self.prev_num_evals = out.get("_evals")                          # device int32 [1] (fused kernel only): field evaluations of the trace
        if st is not None and want_normals and bool(hit.any()):          # generic field: central differences through its forward()
            grad = ops.finitediff_gradient(out["xyz"][hit], nef.get_forward_function("sdf"))
            out["normal"][hit] = torch.nn.functional.normalize(grad, p=2, dim=-1, eps=1e-5)
            out["rgb"] = (out["normal"] + 1.0) / 2.0
        extra_outputs = {}
        for channel in extra_channels:                                    # queried at the surface points (:153-156)
            feats = nef(coords=out["xyz"][hit], lod_idx=lod_idx, channels=channel)
            buf = torch.zeros(*rays.origins.shape[:-1], feats.shape[-1], device=feats.device)
            buf[hit] = feats.to(buf.dtype)
            extra_outputs[channel] = buf
        return RenderBuffer(xyz=out["xyz"], depth=out["depth"], hit=hit, normal=out["normal"], rgb=out["rgb"], alpha=out["alpha"], **extra_outputs)
