"""Tensor-level operators over the C ABI: the functions the wisp-facing classes (and wisp itself, once patched by
wisp_b200.install()) call.  Each one names the reference operator it stands in for.
"""
from __future__ import annotations

import ctypes as C
import os
from dataclasses import dataclass
from typing import List, Optional, Sequence

import torch

from . import _cabi as A
from . import spc
from .core import RenderBuffer

# Optional per-stage device timing (bench.py): when PROFILE is a list, every native stage appends
# (name, start_event, end_event) recorded on the launching (current torch) stream.
PROFILE: Optional[list] = None


class _stage:
    def __init__(self, name: str):
        self.name = name

    def __enter__(self):
        if PROFILE is not None:
            self.e0 = torch.cuda.Event(enable_timing=True); self.e1 = torch.cuda.Event(enable_timing=True)
            self.e0.record()
        return self

    def __exit__(self, *exc):
        if PROFILE is not None:
            self.e1.record()
            PROFILE.append((self.name, self.e0, self.e1))
        return False


# --------------------------------------------------------------------------------------------------------------
# octree handle: the SPC tensors the reference's OctreeAS keeps (octree_as.py:58-62) + the optional dense bitmask
# --------------------------------------------------------------------------------------------------------------
COARSE_LEVEL = int(os.environ.get("WB_COARSE_LEVEL", "6"))      # level of the dilated mask the marcher uses to skip empty 32-candidate words (0 disables it)


@dataclass
class OctreeTensors:
    octree: torch.Tensor          # uint8 [nbytes]
    prefix: torch.Tensor          # int32 [nbytes+1]
    points: torch.Tensor          # int16 [total,3]
    pyramid: torch.Tensor         # int32 [2, max_level+2] (CPU)
    max_level: int
    bits: Optional[torch.Tensor] = None
    bits_level: int = -1
    bbox: Optional[tuple] = None          # (lo[3], hi[3]) of the occupied cells of `bits_level`, normalised coords
    coarse: Optional[torch.Tensor] = None # dilated occupancy of `coarse_level` (word-skipping in the marcher), or None
    coarse_level: int = 0

    def desc(self) -> A.OctreeDesc:
        d = A.OctreeDesc()
        d.octree, d.prefix, d.nbytes, d.max_level = self.octree.data_ptr(), self.prefix.data_ptr(), self.octree.shape[0], self.max_level
        d.bits = self.bits.data_ptr() if self.bits is not None else None
        d.bits_level = self.bits_level
        d.has_bbox = 0
        if self.bbox is not None:
            d.has_bbox = 1
            for a in range(3):
                d.bbox_lo[a], d.bbox_hi[a] = self.bbox[0][a], self.bbox[1][a]
        d.coarse_bits = self.coarse.data_ptr() if self.coarse is not None else None
        d.coarse_level = self.coarse_level if self.coarse is not None else 0
        return d

    def ensure_bits(self, level: int) -> None:
        """Dense occupancy bitmask of `level` (<= 10): 8^level bits, built once per octree by wb_octree_build_bits."""
        if level > 10 or (self.bits is not None and self.bits_level == level):
            return
        A.require_device(self.octree)
        words = (8 ** level + 31) // 32
        bits = torch.zeros(words, dtype=torch.int32, device=self.octree.device)
        start, cnt = int(self.pyramid[1, level]), int(self.pyramid[0, level])
        lvl = self.points[start:start + cnt].contiguous()
        A.lib().wb_octree_build_bits(A.ptr(lvl), cnt, level, A.ptr(bits), A.stream())
        self.bits, self.bits_level = bits, level
        self.coarse, self.coarse_level = None, 0
        cl = min(level - 1, COARSE_LEVEL)
        if cl >= 2 and cnt > 0:
            coarse = torch.zeros((8 ** cl + 31) // 32, dtype=torch.int32, device=self.octree.device)
            A.lib().wb_octree_build_coarse(A.ptr(lvl), cnt, level, cl, A.ptr(coarse), A.stream())
            self.coarse, self.coarse_level = coarse, cl
        if cnt > 0:     # one-off (per octree) host read of the occupied extent; exact dyadic cell faces
            mn, mx = lvl.min(0).values.cpu().tolist(), lvl.max(0).values.cpu().tolist()
            res = float(2 ** level)
            self.bbox = ([2.0 * m / res - 1.0 for m in mn], [2.0 * (m + 1) / res - 1.0 for m in mx])


def octree_tensors(blas) -> OctreeTensors:
    """The OctreeTensors of an OctreeAS (this package's or the reference's), cached on the BLAS and rebuilt when its octree tensor
    is replaced.  prefix and pyramid are cast to int32 (the C ABI's type; already so for spc.scan_octree's)."""
    t = getattr(blas, "_wb_tensors", None)
    if t is None or t.octree.data_ptr() != blas.octree.data_ptr():
        t = OctreeTensors(blas.octree.contiguous(), blas.prefix.contiguous().int(), blas.points.contiguous(), blas.pyramid.cpu().int(), blas.max_level)
        blas._wb_tensors = t
    return t


def query(oct: OctreeTensors, coords: torch.Tensor, level: int, with_parents: bool = False) -> torch.Tensor:
    """spc_ops.unbatched_query(octree, prefix, coords, level, with_parents)  (octree_as.py:162)."""
    A.require_device(coords)
    c = A.f32c(coords)
    N = c.shape[0]
    out = torch.empty((N, level + 1) if with_parents else (N,), dtype=torch.int32, device=c.device)
    d = oct.desc()
    A.lib().wb_query(d, A.ptr(c), N, level, int(with_parents), A.ptr(out), A.stream())
    return out


# --------------------------------------------------------------------------------------------------------------
# raymarch 'ray'
# --------------------------------------------------------------------------------------------------------------
@dataclass
class MarchState:
    """Intermediate state of one raymarch: per-ray hit bitmask, counts and offsets (device), total (host)."""
    rays: A.RaysDesc
    keep: list
    n: int
    jitter: Optional[torch.Tensor]
    seed: int
    hitmask: Optional[torch.Tensor]
    counts: Optional[torch.Tensor]
    offsets: torch.Tensor            # int64 [R+1]: sample range of every ray
    total: int
    records: Optional[tuple] = None  # (t, delta, ray) already produced by the 'voxel' / 'uniform' samplers


def march_count(oct: OctreeTensors, origins, dirs, dist_min, dist_max, num_samples: int, level: int,
                jitter: Optional[torch.Tensor] = None, seed: int = 0, defer_total: bool = False):
    """Sample culling of OctreeAS._raymarch_ray (octree_as.py:272-288) without materialising candidates."""
    A.require_device(origins)
    oct.ensure_bits(level)
    rays, keep = A.make_rays(origins, dirs, dist_min, dist_max)
    R = rays.num_rays
    dev = origins.device
    nw = (num_samples + 31) // 32
    hitmask = torch.empty((R, nw), dtype=torch.int32, device=dev)
    counts = torch.empty(R, dtype=torch.int32, device=dev)
    offsets = torch.empty(R + 1, dtype=torch.int64, device=dev)
    jit = None if jitter is None else A.f32c(jitter)
    if jit is not None and tuple(jit.shape) != (R, num_samples):
        raise A.WispB200Error(f"jitter must be [{R}, {num_samples}]")
    od = oct.desc()
    L = A.lib()
    with _stage("march_count"):
        L.wb_raymarch_ray_count(od, level, rays, num_samples, A.ptr(jit),
                                seed & 0xFFFFFFFF, A.ptr(hitmask), A.ptr(counts), A.stream())
    wsb = int(L.wb_scan_workspace_bytes(R))
    ws = torch.empty(wsb, dtype=torch.uint8, device=dev)
    with _stage("scan"):
        L.wb_scan_counts(A.ptr(counts), R, A.ptr(offsets), A.ptr(ws), wsb, A.stream())
    ms = MarchState(rays, keep + [jit], num_samples, jit, seed & 0xFFFFFFFF, hitmask, counts, offsets, -1)
    if defer_total:                        # pre-march on a side stream: the total travels to pinned memory, no host sync here
        host = _pinned_slot()
        host.copy_(offsets[-1:], non_blocking=True)
        ev = torch.cuda.Event(); ev.record(torch.cuda.current_stream(dev))
        return PendingMarch(ms, host, ev, torch.cuda.current_stream(dev))
    ms.total = int(offsets[-1].item())     # the one host sync of the path (the reference syncs in torch.nonzero, octree_as.py:288)
    return ms


_PINNED_RING: list = []
_PINNED_NEXT = 0


def _pinned_slot() -> torch.Tensor:
    """One of 8 page-locked int64 slots allocated once per process (cudaHostAlloc in the training loop costs milliseconds and
    synchronises); a slot is reused only 8 pre-marches later, long after its copy has been consumed."""
    global _PINNED_NEXT
    if not _PINNED_RING:
        buf = torch.empty(8, dtype=torch.int64, pin_memory=True)
        _PINNED_RING.extend(buf[i:i + 1] for i in range(8))
    _PINNED_NEXT = (_PINNED_NEXT + 1) % 8
    return _PINNED_RING[_PINNED_NEXT]


@dataclass
class PendingMarch:
    """A raymarch whose kernels were enqueued on a side stream (PackedRFTracer.premarch): finalize() makes the consumer stream
    wait for them and reads the sample total (normally long since on the host by the time the batch is rendered)."""
    ms: MarchState
    host_total: torch.Tensor
    event: "torch.cuda.Event"
    stream: "torch.cuda.Stream"

    def finalize(self) -> MarchState:
        cur = torch.cuda.current_stream(self.ms.offsets.device)
        cur.wait_event(self.event)
        for t in (self.ms.hitmask, self.ms.counts, self.ms.offsets):
            t.record_stream(cur)
        self.event.synchronize()
        self.ms.total = int(self.host_total[0])
        return self.ms


def march_fill_reference_layout(ms: MarchState, device):
    """ASRaymarchResults tensors (base_as.py:57-84)."""
    S = ms.total
    ridx = torch.empty(S, dtype=torch.int64, device=device)
    samples = torch.empty((S, 3), dtype=torch.float32, device=device)
    depth = torch.empty((S, 1), dtype=torch.float32, device=device)
    deltas = torch.empty((S, 1), dtype=torch.float32, device=device)
    boundary = torch.empty(S, dtype=torch.bool, device=device)
    if S > 0:
        A.lib().wb_raymarch_ray_fill(ms.rays, ms.n, A.ptr(ms.jitter), ms.seed, A.ptr(ms.hitmask),
                                     A.ptr(ms.offsets), A.ptr(ridx), A.ptr(samples), A.ptr(depth), A.ptr(deltas), A.ptr(boundary), A.stream())
    return ridx, samples, depth, deltas, boundary


_CAP_FLOOR = 0      # high-water capacity of the per-sample buffers (samples); only grows


def reserve_samples(S: int) -> int:
    """Pre-size the per-sample buffers for batches of up to S hit samples (trainer warm-up: the reference sizes its ray batch
    from prev_num_samples the same way, multiview_trainer.py:95-109).  Returns the capacity now in force."""
    global _CAP_FLOOR
    _CAP_FLOOR = max(_CAP_FLOOR, _bucket_raw(int(S)))
    return _CAP_FLOOR


def _bucket_raw(S: int) -> int:
    if S <= 0:
        return 0
    gran = max(1 << 16, 1 << max(0, S.bit_length() - 4))
    return (S + gran - 1) // gran * gran


def _bucket(S: int) -> int:
    """Capacity for a per-sample buffer: S rounded up to 1/8 of its power of two (<= 12.5 % slack, >= 64 Ki samples), and never
    below the largest capacity handed out so far.  The sample count changes with every batch of rays; one stable size lets
    the caching allocator hand the same blocks back instead of going to cudaMalloc / cudaFree (a device sync, ~10 ms) whenever
    S crosses a bucket boundary.  A batch that outgrows the high-water mark raises it with 1/16 headroom."""
    global _CAP_FLOOR
    if S <= 0:
        return 0
    b = _bucket_raw(S)
    if b > _CAP_FLOOR:
        _CAP_FLOOR = _bucket_raw(S + S // 16)
    return _CAP_FLOOR


_NUG_FLOOR = 0


def reserve_nuggets(n: int) -> int:
    """Pre-size the per-nugget buffers of raytrace() (render loops over many cameras: the largest nugget count of the orbit)."""
    global _NUG_FLOOR
    _NUG_FLOOR = max(_NUG_FLOOR, _bucket_raw(int(n)))
    return _NUG_FLOOR


def _empty_n(n: int, tail: tuple, dtype, device):
    """Per-nugget buffer (raytrace outputs) with its own high-water capacity: the nugget count changes with every camera, and an
    exact-size torch.empty sent the caching allocator to cudaMalloc inside render loops (2 per frame in bench.py --config 3)."""
    global _NUG_FLOOR
    if n <= 0:
        return torch.empty((0,) + tuple(tail), dtype=dtype, device=device)
    b = _bucket_raw(n)
    if b > _NUG_FLOOR:
        _NUG_FLOOR = _bucket_raw(n + n // 4)
    return torch.empty((_NUG_FLOOR,) + tuple(tail), dtype=dtype, device=device)[:n]


def _empty_s(S: int, tail: tuple, dtype, device):
    """torch.empty((S, *tail)) carved from a bucketed allocation."""
    return torch.empty((_bucket(S),) + tuple(tail), dtype=dtype, device=device)[:S]


def march_fill_records(ms: MarchState, device):
    """Fused-path sample records: depth t, delta, ray index (12 B/sample)."""
    if ms.records is not None:
        return ms.records
    S = ms.total
    rec_t = _empty_s(S, (), torch.float32, device)
    rec_delta = _empty_s(S, (), torch.float32, device)
    rec_ray = _empty_s(S, (), torch.int32, device)
    if S > 0:
        with _stage("march_fill"):
            A.lib().wb_rf_march_fill(ms.rays, ms.n, A.ptr(ms.jitter), ms.seed, A.ptr(ms.hitmask),
                                     A.ptr(ms.offsets), A.ptr(rec_t), A.ptr(rec_delta), A.ptr(rec_ray), A.stream())
    return rec_t, rec_delta, rec_ray


# --------------------------------------------------------------------------------------------------------------
# raytrace + 'voxel' / 'uniform' samplers
# --------------------------------------------------------------------------------------------------------------
def _scan(counts: torch.Tensor) -> torch.Tensor:
    n = counts.shape[0]
    offsets = torch.empty(n + 1, dtype=torch.int64, device=counts.device)
    L = A.lib()
    wsb = int(L.wb_scan_workspace_bytes(n))
    ws = torch.empty(wsb, dtype=torch.uint8, device=counts.device)
    L.wb_scan_counts(A.ptr(counts), n, A.ptr(offsets), A.ptr(ws), wsb, A.stream())
    return offsets


RAYTRACE_CACHE_K = 24      # nuggets per ray kept by the counting traversal (0: two traversals, wb_raytrace_count + wb_raytrace_fill)


_RT_SCRATCH: dict = {}


def _raytrace_scratch(nbytes: int, dev) -> torch.Tensor:
    """The nugget cache of raytrace() (12 B x K per ray, 75 MB for a 512^2 frame) is kept per (device, stream) instead of being
    allocated per call: returned to the caching allocator between frames, the block was carved up for the frame's output buffers
    and the next frame went to cudaMalloc for a new one (1-7 ms inside a 1.5 ms render, seen as outliers of bench.py --config 3)."""
    key = (dev.index if dev.index is not None else torch.cuda.current_device(), int(torch.cuda.current_stream(dev).cuda_stream))
    buf = _RT_SCRATCH.get(key)
    if buf is None or buf.numel() < nbytes:
        buf = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        _RT_SCRATCH[key] = buf
    return buf


def raytrace(oct: OctreeTensors, origins, dirs, level: int):
    """spc_render.unbatched_raytrace(..., return_depth=True, with_exit=True) (octree_as.py:183-185)
    -> ridx int32 [Ng], pidx int32 [Ng], depth f32 [Ng,2], ray_offsets int64 [R+1]."""
    A.require_device(origins)
    rays, keep = A.make_rays(origins, dirs, 0.0, 0.0)
    R, dev, L = rays.num_rays, origins.device, A.lib()
    od = oct.desc()
    counts = torch.empty(R, dtype=torch.int32, device=dev)
    # one traversal: the count pass caches the first RAYTRACE_CACHE_K nuggets of every ray, the fill copies them (rays with more are
    # traversed again); the cache is scratch (12 B x K per ray) and is skipped for ray counts where it would be unreasonably large
    K = RAYTRACE_CACHE_K if (RAYTRACE_CACHE_K > 0 and R * RAYTRACE_CACHE_K * 12 <= (2 << 30)) else 0
    cache = _raytrace_scratch(int(L.wb_raytrace_cache_bytes(R, K)), dev) if K > 0 else None
    with _stage("raytrace_count"):
        if K > 0:
            L.wb_raytrace_count_cached(od, level, rays, A.ptr(counts), A.ptr(cache), K, A.stream())
        else:
            L.wb_raytrace_count(od, level, rays, A.ptr(counts), A.stream())
    offsets = _scan(counts)
    Ng = int(offsets[-1].item())
    ridx = _empty_n(Ng, (), torch.int32, dev); pidx = _empty_n(Ng, (), torch.int32, dev)
    depth = _empty_n(Ng, (2,), torch.float32, dev)
    if Ng > 0:
        with _stage("raytrace_fill"):
            if K > 0:
                L.wb_raytrace_fill_cached(od, level, rays, A.ptr(offsets), A.ptr(cache), K,
                                          A.ptr(ridx), A.ptr(pidx), A.ptr(depth), A.stream())
            else:
                L.wb_raytrace_fill(od, level, rays, A.ptr(offsets), A.ptr(ridx), A.ptr(pidx), A.ptr(depth), A.stream())
    return ridx, pidx, depth, offsets


def spc_trace(oct: OctreeTensors, origins, dirs, level: int, colors: torch.Tensor, point_offset: int):
    """PackedSPCTracer.trace (packed_spc_tracer.py:50-90) in one launch (wb_spc_trace): the first nugget of every ray at `level`
    -> RenderBuffer(depth f32 [R, 1], hit bool [R], rgb f32 [R, 3], alpha f32 [R, 1]), rgb = colors[pidx - point_offset, :3].
    colors: f32 [M, >= 3] with unit column stride on the rays' device, holding a row for every point of `level`."""
    A.require_device(origins)
    first, cnt = int(oct.pyramid[1, level]), int(oct.pyramid[0, level])
    if (colors.dtype != torch.float32 or colors.dim() != 2 or colors.shape[1] < 3 or colors.stride(1) != 1 or colors.device != origins.device
            or not 0 <= point_offset <= first or first + cnt - point_offset > colors.shape[0]):
        raise A.WispB200Error(f"spc_trace: colors must be f32 [M >= {first + cnt - point_offset}, >= 3] with unit column stride on "
                              f"{origins.device} and 0 <= point_offset <= {first}; got {tuple(colors.shape)} {colors.dtype} on {colors.device}, "
                              f"point_offset {point_offset}")
    rays, keep = A.make_rays(origins, dirs, 0.0, 0.0)
    R, dev = rays.num_rays, origins.device
    depth = torch.empty((R, 1), dtype=torch.float32, device=dev)
    hit = torch.empty(R, dtype=torch.bool, device=dev)
    rgb = torch.empty((R, 3), dtype=torch.float32, device=dev)
    alpha = torch.empty((R, 1), dtype=torch.float32, device=dev)
    od = oct.desc()
    with _stage("spc_trace"):
        A.lib().wb_spc_trace(od, level, rays, A.ptr(colors), colors.stride(0), point_offset,
                             A.ptr(depth), A.ptr(hit), A.ptr(rgb), A.ptr(alpha), A.stream())
    return RenderBuffer(depth=depth, hit=hit, rgb=rgb, alpha=alpha)


def spc_colors(nef) -> Optional[torch.Tensor]:
    """The f32 [M, 3] rows SPCField.rgba gathers (spc_field.py:130-147: colors[:, :3]) as a view of the field's colours, made once per
    colour tensor and kept on the field; None unless the colours are an f32 [M, >= 3] CUDA tensor (the reference's tracer writes
    them into an f32 buffer with an index put, which refuses any other dtype: packed_spc_tracer.py:87)."""
    src = getattr(nef, "colors", None)
    if not torch.is_tensor(src) or not src.is_cuda or src.dtype != torch.float32 or src.dim() != 2 or src.shape[1] < 3:
        return None
    cached = getattr(nef, "_wb_spc_colors", None)
    if cached is None or cached[0] is not src or cached[1] != src._version:
        view = src.detach()[:, :3]
        cached = (src, src._version, view if view.stride(1) == 1 else view.contiguous())
        nef._wb_spc_colors = cached
    return cached[2]


def uniform_scale(num_samples: int) -> int:
    """octree_as.py:336-338."""
    import math
    return int(math.ceil(1.0 / (2.0 * math.sqrt(3.0) / num_samples)))


def march_nuggets(oct: OctreeTensors, origins, dirs, level: int, num_samples: int, kind: str, reference_layout: bool,
                  jitter: Optional[torch.Tensor] = None, seed: int = 0):
    """'voxel' / 'uniform' sampling on top of raytrace.  Returns (MarchState with records, reference-layout dict or None)."""
    ridx_n, pidx_n, depth_n, ray_off = raytrace(oct, origins, dirs, level)
    rays, keep = A.make_rays(origins, dirs, 0.0, 0.0)
    R, dev, L = rays.num_rays, origins.device, A.lib()
    Ng = ridx_n.shape[0]
    if kind == 'voxel':
        S = Ng * num_samples
        sample_off = None
    else:
        scale = uniform_scale(num_samples)
        cnt = torch.empty(Ng, dtype=torch.int32, device=dev)
        L.wb_raymarch_uniform_count(A.ptr(depth_n), Ng, scale, A.ptr(cnt), A.stream())
        sample_off = _scan(cnt)
        S = int(sample_off[-1].item())
    t = torch.empty(S, dtype=torch.float32, device=dev); dl = torch.empty(S, dtype=torch.float32, device=dev)
    rr = torch.empty(S, dtype=torch.int32, device=dev)
    ref = None
    ridx = samples = boundary = None
    if reference_layout:
        ridx = torch.empty(S, dtype=torch.int64, device=dev); samples = torch.empty((S, 3), dtype=torch.float32, device=dev)
        boundary = torch.empty(S, dtype=torch.bool, device=dev)
    jit = None if jitter is None else A.f32c(jitter)
    with _stage("march_" + kind):
        if kind == 'voxel':
            L.wb_raymarch_voxel_fill(rays, A.ptr(ridx_n), A.ptr(depth_n), Ng, num_samples, A.ptr(jit),
                                     seed & 0xFFFFFFFF, A.ptr(ridx), A.ptr(samples), A.ptr(t), A.ptr(dl), A.ptr(boundary), A.ptr(rr), A.stream())
            offsets = ray_off * num_samples
        else:
            L.wb_raymarch_uniform_fill(rays, A.ptr(ridx_n), A.ptr(depth_n), Ng, scale, A.ptr(sample_off), A.ptr(ray_off),
                                       A.ptr(ridx), A.ptr(samples), A.ptr(t), A.ptr(dl), A.ptr(boundary), A.ptr(rr), A.stream())
            offsets = sample_off[ray_off]
    ms = MarchState(rays, keep, num_samples, None, seed & 0xFFFFFFFF, None, None, offsets.contiguous(), S, records=(t, dl, rr))
    if reference_layout:
        ref = dict(ridx=ridx, samples=samples, depth_samples=t[:, None], deltas=dl[:, None], boundary=boundary)
    return ms, ref


def march(grid, lod_idx: int, rays, raymarch_type: str, num_steps: int, jitter: Optional[torch.Tensor] = None, seed: int = 0) -> MarchState:
    """The march of a fused trace at `lod_idx` over the grid's BLAS: 'ray' -> march_count, 'voxel' / 'uniform' -> march_nuggets."""
    oct, level = octree_tensors(grid.blas), raymarch_level(grid, lod_idx)
    if raymarch_type == 'ray':
        return march_count(oct, rays.origins, rays.dirs, rays.dist_min, rays.dist_max, num_steps, level, jitter=jitter, seed=seed)
    return march_nuggets(oct, rays.origins, rays.dirs, level, num_steps, raymarch_type, reference_layout=False, jitter=jitter, seed=seed)[0]


# --------------------------------------------------------------------------------------------------------------
# hash grid interpolate (unfused drop-in for wisp.ops.grid.hashgrid)
# --------------------------------------------------------------------------------------------------------------
def _no_coords_grad(ctx, i: int) -> None:
    """The native grid kernels return no gradient with respect to the sample coordinates (Kaolin's trilinear interpolation does not
    either; the reference's hash-grid grad_coords branch, hashgrid_interpolate_cuda.cu:163-210, is not replicated): refuse loudly instead of
    silently cutting the graph (eikonal losses, autodiff normals must stay on the reference path, INTEGRATION.md section 3)."""
    if ctx.needs_input_grad[i]:
        raise A.WispB200Error("wisp_b200 grid kernels do not provide gradients with respect to coords (coords.requires_grad is set)")


class HashGridInterpolate(torch.autograd.Function):
    """wisp.ops.grid.HashGridInterpolate (ops/grid.py:77-126) over wb_hashgrid_fwd / wb_hashgrid_bwd ([N, 3] coordinates) or
    wb_hashgrid2d_fwd / wb_hashgrid2d_bwd ([N, 2], app/image), chosen from the coordinate width as the reference's kernel does.
    Differences by design: all LODs in one launch; the table is read as fp32 master (no per-call .half() copy,
    ops/grid.py:88-89) and gradients accumulate in fp32."""

    @staticmethod
    def forward(ctx, coords, resolutions, codebook_bitwidth, lod_idx, codebook, codebook_first_idx):
        if codebook.shape[-1] % 2 == 1:
            raise Exception("The codebook feature dimension needs to be a multiple of 2.")   # ops/grid.py:83-84
        _no_coords_grad(ctx, 0)
        dim = coords.shape[-1]
        if dim not in (2, 3):
            raise ValueError(f"HashGrid.interpolate: coordinates must be 2-D or 3-D (the reference's coord_dim), got width {dim}")
        A.require_device(codebook)
        c = A.f32c(coords)
        res = [int(r) for r in torch.as_tensor(resolutions).reshape(-1).tolist()]
        begin = [int(b) for b in codebook_first_idx.tolist()] if torch.is_tensor(codebook_first_idx) else list(codebook_first_idx)
        table = A.f32c(codebook.detach())
        desc = A.make_grid_desc(table, res, begin, 2 ** codebook_bitwidth)
        feats = torch.empty((c.shape[0], len(res) * table.shape[1]), dtype=torch.float32, device=c.device)
        fwd = A.lib().wb_hashgrid_fwd if dim == 3 else A.lib().wb_hashgrid2d_fwd
        fwd(A.ptr(c), c.shape[0], desc, A.ptr(feats), A.stream())
        ctx.save_for_backward(c, table)
        ctx.meta = (res, begin, codebook_bitwidth)
        return feats

    @staticmethod
    def backward(ctx, grad_output):
        c, table = ctx.saved_tensors
        res, begin, bw = ctx.meta
        desc = A.make_grid_desc(table, res, begin, 2 ** bw)
        g = A.f32c(grad_output)
        gt = torch.zeros_like(table)                      # hashgrid_interpolate.cpp:85
        bwd = A.lib().wb_hashgrid_bwd if c.shape[-1] == 3 else A.lib().wb_hashgrid2d_bwd
        bwd(A.ptr(c), c.shape[0], desc, A.ptr(g), A.ptr(gt), A.stream())
        return None, None, None, None, gt, None


def hashgrid(coords, codebook_bitwidth, lod_idx, codebook):
    """wisp.ops.grid.hashgrid (ops/grid.py:128-144); `codebook` is a MultiTable."""
    batch, dim = coords.shape
    feats = HashGridInterpolate.apply(coords.contiguous(), codebook.resolutions, codebook_bitwidth, lod_idx,
                                      codebook.feats, codebook.begin_idxes)
    feature_dim = codebook.feats.shape[1] * len(codebook.resolutions)
    return feats.reshape(batch, feature_dim)


# --------------------------------------------------------------------------------------------------------------
# ImageNeuralField (app/image): wb_image_eval / wb_image_train
# --------------------------------------------------------------------------------------------------------------
IMAGE_BANDS = (1.0, 2.0, 4.0)          # get_positional_embedder(frequencies=3): 2^linspace(0, 2, 3)


def image_field(nef):
    """(grid desc, hidden_dim, decoder pointers, keepalive) of an ImageNeuralField for wb_image_eval / wb_image_train, or None when the
    kernels do not take the field: a grid other than a hash grid of 2, 4 or 8 features per LOD, a decoder other than one relu hidden
    layer (a multiple of 4 up to 128 wide) with biases and 3 outputs, an embedder other than the reference's 3-band one with input, a
    decoder input wider than the kernels' shared-memory image allows, or parameters that are not contiguous fp32 on the device.
    The decoder pointers are a host array [W0, b0, Wout, bout] aimed at the parameters themselves: no copy, no launch."""
    grid, dec, emb = getattr(nef, "grid", None), getattr(nef, "decoder", None), getattr(nef, "embedder", None)
    cb = getattr(grid, "codebook", None)
    if grid is None or dec is None or emb is None or not hasattr(cb, "feats") or not hasattr(cb, "begin_idxes"):
        return None
    if getattr(grid, "multiscale_type", None) not in ("cat", "sum") or getattr(dec, "activation", None) is not torch.relu:
        return None
    layers = list(getattr(dec, "layers", []))
    if len(layers) != 1 or getattr(dec, "skip", []) or any(type(l) is not torch.nn.Linear or l.bias is None for l in layers + [dec.lout]):
        return None
    bands = getattr(emb, "bands", None)
    if (not getattr(emb, "include_input", False) or not torch.is_tensor(bands) or bands.numel() != 3
            or [float(b) for b in bands.detach().reshape(-1).tolist()] != list(IMAGE_BANDS)):
        return None
    F, L = int(cb.feats.shape[1]), len(grid.resolutions)
    fw = F * L if grid.multiscale_type == "cat" else F
    H = int(layers[0].out_features)
    if layers[0].in_features != fw + 14 or dec.lout.out_features != 3:
        return None
    params = decoder_params(dec)
    table = cb.feats
    if any(not p.is_cuda or p.dtype != torch.float32 or not p.is_contiguous() for p in params + [table]):
        return None
    res = [int(r) for r in torch.as_tensor(grid.resolutions).reshape(-1).tolist()]
    desc = A.make_grid_desc(table.data, res, [int(b) for b in cb.begin_idxes.tolist()], 2 ** int(grid.codebook_bitwidth), grid.multiscale_type)
    if A.lib().wb_image_smem_bytes(desc, H, 1) < 0:
        return None
    ptrs = (C.c_void_p * 4)(*[p.data_ptr() for p in params])
    return desc, H, ptrs, [table] + params


def image_eval(nef, coords: torch.Tensor, lod_idx: int) -> Optional[torch.Tensor]:
    """ImageNeuralField.rgb in one launch (wb_image_eval): rgb [N, 3], or None when image_field declines the field."""
    fd = image_field(nef)
    if fd is None:
        return None
    desc, H, params, _ = fd
    A.require_device(coords)
    c = A.f32c(coords)
    rgb = torch.empty((c.shape[0], 3), dtype=torch.float32, device=c.device)
    A.lib().wb_image_eval(desc, H, params, lod_idx, A.ptr(c), c.shape[0], A.ptr(rgb), A.stream())
    return rgb


def image_rgb(nef, coords: torch.Tensor, lod=None) -> Optional[torch.Tensor]:
    """ImageNeuralField.rgb's native route: rgb [N, 3] from image_eval for a non-empty [N, 2] CUDA batch outside autograd and
    autocast (the trainer's validate() over 1 M-pixel chunks, render_final_view); None otherwise or when the kernel declines the field."""
    if (coords.dim() != 2 or coords.shape[-1] != 2 or coords.shape[0] == 0 or not coords.is_cuda or torch.is_grad_enabled()
            or torch.is_autocast_enabled()):
        return None
    return image_eval(nef, coords, len(nef.grid.resolutions) - 1 if lod is None else int(lod))


def image_train(fd, coords: torch.Tensor, rgb_gt: torch.Tensor, lod_idx: int, grad_table: torch.Tensor, grad_params: torch.Tensor,
                loss_out: torch.Tensor) -> None:
    """Forward, F.mse_loss and backward of ImageTrainer.step in one launch (wb_image_train) for fd = image_field(nef); coords f32 [N, 2],
    rgb_gt f32 [N, 3] on the device.  Accumulates loss_out[0] += mean (y - gt)^2, grad_table (codebook.feats) and grad_params
    (packed [W0, b0, Wout, bout])."""
    desc, H, params, _ = fd
    A.require_device(coords)
    N = int(coords.shape[0])
    if N == 0:
        raise A.WispB200Error("image_train: empty batch (the reference's mse_loss averages over it)")
    c, g = A.f32c(coords), A.f32c(rgb_gt)
    A.lib().wb_image_train(desc, H, params, lod_idx, A.ptr(c), A.ptr(g), N,
                           1.0 / (3.0 * N), A.ptr(grad_table), A.ptr(grad_params), A.ptr(loss_out), A.stream())


# --------------------------------------------------------------------------------------------------------------
# triplanar grid interpolate
# --------------------------------------------------------------------------------------------------------------
class TriplaneInterpolate(torch.autograd.Function):
    """All LODs x 3 planes of TriplanarGrid.interpolate in one launch (triplanar_grid.py:98-143, 205-223).
    planes: fmx, fmy, fmz of LOD 0, then LOD 1, ... each [1, fdim, res+1, res+1].  Returns [N, num_lods*3*fdim]."""

    @staticmethod
    def forward(ctx, coords, num_lods, *planes):
        A.require_device(planes[0])
        _no_coords_grad(ctx, 0)
        c = A.f32c(coords)
        N, fdim = c.shape[0], planes[0].shape[1]
        pl = [A.f32c(p.detach()) for p in planes[:3 * num_lods]]
        res = (C.c_int32 * num_lods)(*[pl[3 * l].shape[-1] - 1 for l in range(num_lods)])
        ptrs = (C.c_void_p * (3 * num_lods))(*[p.data_ptr() for p in pl])
        feats = torch.empty((N, num_lods * 3 * fdim), dtype=torch.float32, device=c.device)
        A.lib().wb_triplane_fwd(A.ptr(c), N, num_lods, fdim, res, ptrs, A.ptr(feats), A.stream())
        ctx.save_for_backward(c, *pl)
        ctx.num_lods, ctx.nplanes = num_lods, len(planes)
        return feats

    @staticmethod
    def backward(ctx, grad_output):
        c, *pl = ctx.saved_tensors
        num_lods, fdim = ctx.num_lods, pl[0].shape[1]
        g = A.f32c(grad_output)
        gp = [torch.zeros_like(p) for p in pl]
        res = (C.c_int32 * num_lods)(*[pl[3 * l].shape[-1] - 1 for l in range(num_lods)])
        ptrs = (C.c_void_p * (3 * num_lods))(*[p.data_ptr() for p in pl])
        gptrs = (C.c_void_p * (3 * num_lods))(*[p.data_ptr() for p in gp])
        A.lib().wb_triplane_bwd(A.ptr(c), c.shape[0], num_lods, fdim, res, ptrs, A.ptr(g), gptrs, A.stream())
        return (None, None, *gp, *([None] * (ctx.nplanes - len(gp))))


# --------------------------------------------------------------------------------------------------------------
# octree grid interpolate + SDF-tracer helpers
# --------------------------------------------------------------------------------------------------------------
class OctreeInterpolate(torch.autograd.Function):
    """OctreeGrid.interpolate for LODs 0..lod_idx in one launch (octree_grid.py:165-219)."""

    @staticmethod
    def forward(ctx, coords, oct, trinkets, base_lod, multiscale, half_round, *feats):
        A.require_device(feats[0])
        _no_coords_grad(ctx, 0)
        c = A.f32c(coords)
        N, F, nl = c.shape[0], feats[0].shape[1], len(feats)
        fl = [A.f32c(f.detach()) for f in feats]
        ptrs = (C.c_void_p * nl)(*[f.data_ptr() for f in fl])
        out = torch.empty((N, F if multiscale == 'sum' else nl * F), dtype=torch.float32, device=c.device)
        od = oct.desc()
        A.lib().wb_octree_interp_fwd(od, A.ptr(oct.points), A.ptr(trinkets), A.ptr(c), N, F, base_lod,
                                     nl, 1 if multiscale == 'sum' else 0, int(half_round), ptrs, A.ptr(out), A.stream())
        ctx.save_for_backward(c, trinkets, *fl)
        ctx.meta = (oct, base_lod, multiscale)
        return out

    @staticmethod
    def backward(ctx, g):
        c, trinkets, *fl = ctx.saved_tensors
        oct, base_lod, multiscale = ctx.meta
        nl, F = len(fl), fl[0].shape[1]
        gf = [torch.zeros_like(f) for f in fl]
        ptrs = (C.c_void_p * nl)(*[f.data_ptr() for f in fl]); gptrs = (C.c_void_p * nl)(*[f.data_ptr() for f in gf])
        od = oct.desc()
        A.lib().wb_octree_interp_bwd(od, A.ptr(oct.points), A.ptr(trinkets), A.ptr(c), c.shape[0], F, base_lod,
                                     nl, 1 if multiscale == 'sum' else 0, ptrs, A.ptr(A.f32c(g)), gptrs, A.stream())
        return (None, None, None, None, None, None, *gf)


class CodebookRows(torch.autograd.Function):
    """CodebookOctreeGrid._index_features (codebook_grid.py:103-131) evaluated once per corner ROW: logits [rows, 2^bw], dictionary
    [2^bw, F] -> E [rows, F] (straight-through softmax selection when `training`, argmax selection otherwise)."""

    @staticmethod
    def forward(ctx, logits, dictionary, training):
        A.require_device(logits)
        lg, dc = A.f32c(logits.detach()), A.f32c(dictionary.detach())
        rows, K, F = lg.shape[0], lg.shape[1], dc.shape[1]
        E = torch.empty((rows, F), dtype=torch.float32, device=lg.device)
        A.lib().wb_codebook_rows_fwd(A.ptr(lg), A.ptr(dc), rows, K, F, int(training), A.ptr(E), None, A.stream())
        ctx.save_for_backward(lg, dc)
        ctx.training = bool(training)
        return E

    @staticmethod
    def backward(ctx, dE):
        lg, dc = ctx.saved_tensors
        if not ctx.training:            # eval: dictionary[argmax] -- the reference's indexing gives the dictionary a gradient, the logits none
            am = lg.argmax(-1)
            gd = torch.zeros_like(dc).index_add_(0, am, A.f32c(dE))
            return None, gd, None
        g_lg, g_dc = torch.zeros_like(lg), torch.zeros_like(dc)
        de = A.f32c(dE)
        A.lib().wb_codebook_rows_bwd(A.ptr(lg), A.ptr(dc), A.ptr(de), lg.shape[0], lg.shape[1], dc.shape[1],
                                     A.ptr(g_lg), A.ptr(g_dc), A.stream())
        return g_lg, g_dc, None


def find_depth_bound(query: torch.Tensor, nug_depth: torch.Tensor, info=None, curr_idxes: Optional[torch.Tensor] = None) -> torch.Tensor:
    """wisp.ops.geometric.find_depth_bound (geometric.py:15-22)."""
    if curr_idxes is None:
        curr_idxes = torch.nonzero(info)[..., 0].int()
    A.require_device(query)
    q, ci, dp = A.f32c(query).reshape(-1), curr_idxes.int().contiguous(), A.f32c(nug_depth)
    out = torch.empty(q.shape[0], dtype=torch.int32, device=q.device)
    A.lib().wb_find_depth_bound(A.ptr(q), A.ptr(ci), A.ptr(dp), q.shape[0], dp.shape[0], A.ptr(out), A.stream())
    return out


def finitediff_gradient(x: torch.Tensor, f, eps: float = 0.005) -> torch.Tensor:
    """wisp.ops.differential.finitediff_gradient (gradients.py:29-45)."""
    ex = torch.tensor([eps, 0.0, 0.0], device=x.device); ey = torch.tensor([0.0, eps, 0.0], device=x.device); ez = torch.tensor([0.0, 0.0, eps], device=x.device)
    grad = torch.cat([f(x + ex) - f(x - ex), f(x + ey) - f(x - ey), f(x + ez) - f(x - ez)], dim=-1)
    return grad / (eps * 2.0)


# --------------------------------------------------------------------------------------------------------------
# NeuralSDF(OctreeGrid) + sphere tracing (app/nglod)
# --------------------------------------------------------------------------------------------------------------
def sdf_field(nef):
    """-> (SdfDesc, OctreeTensors, keepalive) for a NeuralSDF over an OctreeGrid ('linear'), or (SdfDesc, None, keepalive) for a
    NeuralSDF over a 3D HashGrid of 4 or 8 features per LOD; None when the field is outside what wb_sdf_eval / wb_sdf_train
    evaluate natively (other grids, activations, skip connections, > 128 wide).  Only octree fields go to wb_sdf_trace."""
    g, dec = getattr(nef, "grid", None), getattr(nef, "decoder", None)
    if g is None or dec is None:
        return None
    octree = all(hasattr(g, a) for a in ("trinkets", "features", "base_lod", "num_lods", "multiscale_type", "blas"))
    if not octree:
        # HashGrid (hash_grid.py:27-89): F = 4 or 8 rows are one or two float4; narrower tables (F = 2) keep the autograd route
        if not all(hasattr(g, a) for a in ("codebook", "codebook_bitwidth", "resolutions", "multiscale_type", "feature_dim")):
            return None
        if int(getattr(g, "coord_dim", 3)) != 3 or int(g.feature_dim) not in (4, 8) or g.multiscale_type not in ('cat', 'sum'):
            return None
    if getattr(g, "interpolation_type", "linear") != "linear" or getattr(nef, "activation_type", "relu") != "relu":
        return None
    layers = _decoder_layers(dec)
    if layers is None or any(l.bias is None for l in layers):       # the SDF decoder: bias on every layer, equal widths, one output
        return None
    H, nh = layers[0].out_features, len(layers) - 1
    if not (1 <= nh <= 4 and H <= 128 and layers[-1].out_features == 1 and all(l.out_features == H for l in layers[:-1])):
        return None
    if nh > 1 and H % 4:
        return None
    em = _embedder_mode(getattr(nef, "pos_embedder", None))
    if em is None or em[1] > 10 or g.feature_dim > 64:          # wb_make_sdf: pos_freq <= 10, feature_dim <= 64
        return None
    num_lods = int(g.num_lods) if octree else len(g.resolutions)
    in_dim = layers[0].in_features
    if in_dim != _embed_width(*em) + (g.feature_dim if g.multiscale_type == 'sum' else g.feature_dim * num_lods):
        return None
    # the decoder input must be at most 132 wide and its shared-memory image must fit in 200 KB: the same limits and formula as
    # wb_make_sdf (csrc/wb_sdf.cuh)
    smem_floats = H * ((in_dim + 3) & ~3) + H + (nh - 1) * (H * H + H) + H + 4
    if in_dim > 132 or smem_floats * 4 > 200 * 1024:
        return None
    params = torch.cat([t.detach().reshape(-1).float() for l in layers for t in (l.weight, l.bias)]).contiguous()
    d = A.SdfDesc()
    d.feature_dim, d.num_lods = int(g.feature_dim), num_lods
    d.multiscale = 1 if g.multiscale_type == 'sum' else 0
    d.pos_mode, d.pos_freq = em
    d.num_layers, d.hidden_dim, d.params = nh, H, params.data_ptr()
    if not octree:
        # the whole codebook.feats [rows, F] as one table; LOD l at rows begin_idxes[l] .. (utils.py:13-71)
        table = A.f32c(g.codebook.feats.detach())
        res = [int(r) for r in torch.as_tensor(g.resolutions).reshape(-1).tolist()]
        hd = A.make_grid_desc(table, res, _hash_begin(g), 2 ** int(g.codebook_bitwidth), g.multiscale_type)
        d.hash = C.pointer(hd)
        return d, None, [hd, table, params]
    dev = g.features[0].device
    oct = octree_tensors(g.blas)
    if g.trinkets.device != dev:
        g.trinkets = g.trinkets.to(dev)
    feats = [A.f32c(f.detach()) for f in g.features]
    trinkets = g.trinkets.int().contiguous()
    ptrs = (C.c_void_p * len(feats))(*[f.data_ptr() for f in feats])
    d.points, d.trinkets, d.feats = oct.points.data_ptr(), trinkets.data_ptr(), ptrs
    d.base_lod = int(g.base_lod)
    d.half_round = int(getattr(g, "half_features", True))
    return d, oct, [ptrs, feats, params, trinkets]


def sdf_eval(nef, coords: torch.Tensor, lod_idx: Optional[int] = None) -> Optional[torch.Tensor]:
    """NeuralSDF.sdf (neural_sdf.py:120-155) in one launch -> [N, 1]; None when the field is not natively supported."""
    fd = sdf_field(nef)
    if fd is None:
        return None
    d, oct, keep = fd
    if lod_idx is None:
        lod_idx = d.num_lods - 1
    if d.multiscale == 0 and lod_idx != d.num_lods - 1 and not d.hash:    # an octree 'cat' grid below its finest LOD: nn.Linear raises
        return None
    A.require_device(coords)
    c = A.f32c(coords).reshape(-1, 3)
    out = torch.empty((c.shape[0], 1), dtype=torch.float32, device=c.device)
    od = _sdf_octree(oct)
    with _stage("sdf_eval"):
        A.lib().wb_sdf_eval(od, d, lod_idx, A.ptr(c), c.shape[0], A.ptr(out), A.stream())
    return out


def sdf_channel(nef, coords: torch.Tensor, lod_idx: Optional[int] = None) -> Optional[dict]:
    """NeuralSDF.sdf's native route: {"sdf": [..., 1]} from sdf_eval for a non-empty CUDA batch outside autograd and autocast (the
    sphere tracer, the trainer's validation slices); None otherwise or when sdf_eval declines the field (the caller's own body runs)."""
    if coords.shape[0] == 0 or not coords.is_cuda or torch.is_grad_enabled() or torch.is_autocast_enabled():
        return None
    fused = sdf_eval(nef, coords, lod_idx)
    return None if fused is None else dict(sdf=fused.reshape(*coords.shape[:-1], 1))


def _sdf_octree(oct):
    """The wb_octree argument of wb_sdf_eval / wb_sdf_train: the octree grid's occupancy, NULL for a hash field."""
    return None if oct is None else oct.desc()


def sdf_train_smem_bytes(fd) -> int:
    """Shared memory of a wb_sdf_train launch for the field fd = sdf_field(nef), or < 0 when the fused step cannot train it
    (its weights, weight-gradient accumulators and smallest sample tile exceed an SM's shared memory)."""
    return int(A.lib().wb_sdf_train_smem_bytes(fd[0]))


def sdf_train_tc_smem_bytes(fd) -> int:
    """Shared memory of a wb_sdf_train_tc launch (precision 1: fp16 weight packs, fp32 weight-gradient accumulators and one
    64-sample tile) for the field fd = sdf_field(nef), or < 0 when the tensor-core step cannot train it."""
    return int(A.lib().wb_sdf_train_tc_smem_bytes(fd[0]))


def sdf_train(fd, coords: torch.Tensor, sdf_gt: torch.Tensor, lod_idx: int, inv_count: float, grad_feats: Sequence[torch.Tensor],
              grad_params: torch.Tensor, loss_out: torch.Tensor, precision: int = 0) -> None:
    """Forward, L2 loss and backward of SDFTrainer.step (sdf_trainer.py:65-124) for one loss LOD in one launch (wb_sdf_train), for
    decoders of 1 to 4 hidden layers whose sdf_train_smem_bytes(fd) >= 0.  fd: sdf_field(nef) (its params pointer may be re-aimed
    at a flat decoder buffer); coords f32 [N,3], sdf_gt f32 [N] on the device.  Accumulates: loss_out[0] += sum (y - gt)^2 *
    inv_count, grad_params (packed like the decoder: [W0, b0, W1, b1, ..., Wout, bout]) and grad_feats[k], k <= lod_idx (octree
    grid); for a hash field grad_feats[0] is dL/d codebook.feats [rows, F].  precision 1: the reference's enable_amp arithmetic on
    the tensor cores (wb_sdf_train_tc: fp16 decoder operands and outputs, fp32 gradients), for fields whose
    sdf_train_tc_smem_bytes(fd) >= 0."""
    if precision not in (0, 1):
        raise A.WispB200Error(f"sdf_train: precision must be 0 (fp32) or 1 (fp16 tensor cores), got {precision!r}")
    d, oct, _ = fd
    A.require_device(coords)
    if not (coords.dtype == sdf_gt.dtype == grad_params.dtype == loss_out.dtype == torch.float32 and coords.is_contiguous() and sdf_gt.is_contiguous()):
        raise A.WispB200Error("sdf_train wants contiguous float32 coords / sdf_gt and float32 gradient and loss buffers")
    if sdf_gt.numel() != coords.shape[0]:
        raise A.WispB200Error(f"sdf_gt has {sdf_gt.numel()} values for {coords.shape[0]} points")
    gptrs = (C.c_void_p * len(grad_feats))(*[g.data_ptr() for g in grad_feats])
    od = _sdf_octree(oct)
    fn = A.lib().wb_sdf_train_tc if precision == 1 else A.lib().wb_sdf_train
    with _stage("sdf_train"):
        fn(od, d, lod_idx, A.ptr(coords), A.ptr(sdf_gt), coords.shape[0], inv_count, gptrs, A.ptr(grad_params), A.ptr(loss_out), A.stream())


class _SdfState:
    """Per-pack state tensors of the sphere tracer (struct wb_sdf_state), owned by PyTorch."""

    def __init__(self, R: int, num_steps: int, dev):
        L = A.lib()
        i32 = lambda n: torch.empty(max(n, 1), dtype=torch.int32, device=dev)
        f32 = lambda n: torch.empty(max(n, 1), dtype=torch.float32, device=dev)
        self.flags, self.pack_ray, self.cursor0, self.cursor1 = i32(R), i32(R), i32(R), i32(R)
        self.pack_off = torch.empty(R + 1, dtype=torch.int64, device=dev)
        self.scan_ws = torch.empty(max(int(L.wb_scan_workspace_bytes(R)), 1), dtype=torch.uint8, device=dev)
        self.t, self.dist, self.dist_prev, self.x = f32(R), f32(R), f32(R), f32(3 * R)
        self.state = torch.empty(max(R, 1), dtype=torch.uint8, device=dev)
        self.iterflags = i32(2 * num_steps + 4)
        s = A.SdfState()
        s.flags, s.pack_off, s.scan_ws, s.scan_ws_bytes, s.pack_ray = self.flags.data_ptr(), self.pack_off.data_ptr(), self.scan_ws.data_ptr(), self.scan_ws.numel(), self.pack_ray.data_ptr()
        s.t, s.dist, s.dist_prev, s.x = self.t.data_ptr(), self.dist.data_ptr(), self.dist_prev.data_ptr(), self.x.data_ptr()
        s.cursor0, s.cursor1, s.state, s.iterflags = self.cursor0.data_ptr(), self.cursor1.data_ptr(), self.state.data_ptr(), self.iterflags.data_ptr()
        self.c = s


def _sdf_buffers(R: int, dev, want_normals: bool):
    """Output buffers as the reference initialises them (packed_sdf_tracer.py:149-168)."""
    z = lambda *shape: torch.zeros(*shape, dtype=torch.float32, device=dev)
    out = dict(xyz=z(R, 3), depth=z(R, 1), hit=torch.zeros(R, dtype=torch.bool, device=dev), normal=z(R, 3), alpha=z(R, 1))
    out["rgb"] = torch.full((R, 3), 0.5, dtype=torch.float32, device=dev) if want_normals else z(R, 3)    # rgb = (normal + 1) / 2 for every ray
    return out


def sdf_trace(nef, oct: OctreeTensors, origins, dirs, dist_max, level: int, lod_idx: int, num_steps: int, step_size: float, min_dis: float,
              want_normals: bool):
    """PackedSDFTracer.trace (packed_sdf_tracer.py:78-174): raytrace + ONE persistent sphere-tracing kernel (wb_sdf_trace) when the
    field is a NeuralSDF(OctreeGrid); otherwise the same state machine phase by phase (wb_sdf_phase) with the field evaluated through
    its own forward() (a NeuralSDF(HashGrid) in sdf_field's range: one wb_sdf_eval per evaluation).  -> dict(xyz, depth, hit,
    normal, rgb, alpha) per ray."""
    A.require_device(origins)
    R, dev, L = origins.shape[0], origins.device, A.lib()
    _, _, nug_depth, ray_off = raytrace(oct, origins, dirs, level)
    Ng = nug_depth.shape[0]
    out = _sdf_buffers(R, dev, want_normals)
    if Ng == 0 or R == 0:
        return out, None
    if torch.is_tensor(dist_max):
        if dist_max.numel() != 1:
            raise A.WispB200Error("PackedSDFTracer compares t with a scalar dist_max (packed_sdf_tracer.py:127)")
        dist_max = float(dist_max)
    rays, keep = A.make_rays(origins, dirs, 0.0, float(dist_max))
    st = _SdfState(R, num_steps, dev)
    od = oct.desc()
    fd = sdf_field(nef)
    if fd is not None and not fd[0].hash and not (fd[0].multiscale == 0 and lod_idx != fd[0].num_lods - 1):
        d, _, keep2 = fd
        with _stage("sdf_trace"):
            L.wb_sdf_trace(od, d, lod_idx, rays, A.ptr(nug_depth), Ng, A.ptr(ray_off),
                           num_steps, step_size, min_dis, int(want_normals), st.c,
                           A.ptr(out["xyz"]), A.ptr(out["depth"]), A.ptr(out["hit"]), A.ptr(out["normal"]), A.ptr(out["rgb"]), A.ptr(out["alpha"]), A.stream())
        out["_evals"] = st.iterflags[2 * num_steps + 2: 2 * num_steps + 3]      # device counter: field evaluations of this launch
        return out, None

    # ---- generic field: the state machine runs natively, the field through its own forward() between the phases ----
    def phase(ph, it=0):
        L.wb_sdf_phase(ph, rays, A.ptr(nug_depth), Ng, A.ptr(ray_off), num_steps, it,
                       min_dis, st.c, A.ptr(out["xyz"]), A.ptr(out["depth"]), A.ptr(out["hit"]), A.ptr(out["alpha"]), A.stream())

    def field(x):
        return nef(coords=x, lod_idx=lod_idx, channels="sdf").reshape(-1).float() * 1.0 * step_size

    with torch.no_grad():
        phase(0)
        P = int(st.pack_off[-1].item())
        phase(1)
        x = st.x[:3 * P].view(P, 3)
        st.dist[:P] = field(x)
        st.dist_prev[:P] = st.dist[:P]
        for it in range(num_steps):
            phase(2, it)
            if int(st.iterflags[2 * it].item()) == 0:
                break
            phase(3, it)
            if int(st.iterflags[2 * it + 1].item()) == 0:
                break
            alive = torch.nonzero(st.state[:P] & 1)[:, 0]
            st.dist[alive] = field(x[alive])
        phase(4)
    return out, st


# --------------------------------------------------------------------------------------------------------------
# packed compositing
# --------------------------------------------------------------------------------------------------------------
def _bg3(bg) -> "C.Array":
    v = [float(x) for x in (bg.detach().cpu().reshape(-1).tolist() if torch.is_tensor(bg) else bg)]
    return (C.c_float * 3)(*v[:3])


class CompositeFn(torch.autograd.Function):
    """exponential_integration + sum_reduce + per-ray scatter of PackedRFTracer.trace (packed_rf_tracer.py:136-165).
    shaded [S,4] = (r,g,b,sigma); returns rgb [R,3], depth [R,1], alpha [R,1], hit [R] (bool)."""

    @staticmethod
    def forward(ctx, shaded, depth, deltas, offsets, bg):
        A.require_device(shaded)
        R = offsets.shape[0] - 1
        dev = shaded.device
        sh, dp, dl = A.f32c(shaded), A.f32c(depth).reshape(-1), A.f32c(deltas).reshape(-1)
        rgb = torch.empty((R, 3), dtype=torch.float32, device=dev)
        dout = torch.empty((R, 1), dtype=torch.float32, device=dev)
        alpha = torch.empty((R, 1), dtype=torch.float32, device=dev)
        hit = torch.empty(R, dtype=torch.bool, device=dev)
        bgv = _bg3(bg)
        A.lib().wb_composite_fwd(A.ptr(sh), A.ptr(dp), A.ptr(dl), A.ptr(offsets), R, bgv,
                                 A.ptr(rgb), A.ptr(dout), A.ptr(alpha), A.ptr(hit), A.stream())
        ctx.save_for_backward(sh, dp, dl, offsets)
        ctx.bg = bgv
        ctx.mark_non_differentiable(hit)
        return rgb, dout, alpha, hit

    @staticmethod
    def backward(ctx, g_rgb, g_depth, g_alpha, _g_hit):
        sh, dp, dl, offsets = ctx.saved_tensors
        R = offsets.shape[0] - 1
        g_sh = torch.zeros_like(sh)
        A.lib().wb_composite_bwd(A.ptr(sh), A.ptr(dp), A.ptr(dl), A.ptr(offsets), R, ctx.bg,
                                 A.ptr(A.f32c(g_rgb)), A.ptr(A.f32c(g_depth).reshape(-1)) if g_depth is not None else None,
                                 A.ptr(A.f32c(g_alpha).reshape(-1)) if g_alpha is not None else None, A.ptr(g_sh), None, A.stream())
        return g_sh, None, None, None, None


# --------------------------------------------------------------------------------------------------------------
# fused render path
# --------------------------------------------------------------------------------------------------------------
GRID_KINDS = {"hash": 0, "triplanar": 1, "octree": 2}
SPLIT_BWD = __import__("os").environ.get("WB_SPLIT_BWD", "0") == "1"


@dataclass
class NefSpec:
    """Static description of a NeuralRadianceField that the fused path supports.  kind 'hash': HashGrid (resolutions, begin_idxes,
    codebook_size); 'triplanar': TriplanarGrid (resolutions = plane side - 1 of the LODs used, feature_dim = 3 * fdim);
    'octree': OctreeGrid (feature_dim = F, base_lod).  For the last two num_lods counts the LODs 0..lod_idx actually used."""
    resolutions: List[int]
    begin_idxes: List[int]
    codebook_size: int
    feature_dim: int
    multiscale: str
    lod_idx: int
    pos_mode: int
    pos_freq: int
    view_mode: int
    view_freq: int
    has_bias: bool
    dens_dims: List[int]
    col_dims: List[int]
    kind: str = "hash"
    num_lods: int = 0
    base_lod: int = 0
    half_round: bool = True

    def desc(self, grid: Sequence[torch.Tensor], dens_flat: torch.Tensor, col_flat: torch.Tensor, oct: Optional[OctreeTensors] = None,
             trinkets: Optional[torch.Tensor] = None, grads: Optional[Sequence[torch.Tensor]] = None, layout: int = 0):
        """-> (NefDesc, keepalive).  grid: [table] | planes (fmx, fmy, fmz per LOD) | feature levels.  layout 1 (triplanar): `grid`
        and `grads` are channel-last copies (triplane_channel_last)."""
        keep = []
        if self.kind == "hash":
            d = A.make_grid_desc(grid[0], self.resolutions, self.begin_idxes, self.codebook_size, self.multiscale, self.lod_idx)
        else:
            d = self.header()
            d.grid_layout = int(layout)
            for i, r in enumerate(self.resolutions):
                d.resolutions[i] = int(r)
            ptrs = (C.c_void_p * len(grid))(*[t.data_ptr() for t in grid])
            d.grid_ptrs = ptrs; keep.append(ptrs)
            if grads is not None:
                gptrs = (C.c_void_p * len(grads))(*[t.data_ptr() for t in grads])
                d.grid_grads = gptrs; keep.append(gptrs)
            if self.kind == "octree":
                od = oct.desc()
                keep.append(od)
                d.oct, d.points, d.trinkets = C.addressof(od), oct.points.data_ptr(), trinkets.data_ptr()
                d.base_lod, d.half_round = self.base_lod, int(self.half_round)
        if not self.fill_decoders(d, dens_flat.data_ptr(), col_flat.data_ptr()):
            raise A.WispB200Error("decoder too deep for the fused path")
        return d, keep

    def header(self):
        """NefDesc holding the grid fields the decoder checks read: grid kind, LOD count, feature width, multiscale and lod_idx
        (a triplanar or octree spec's LODs are all in use).  A hash spec's desc() gets the same fields from make_grid_desc."""
        d = A.NefDesc()
        d.grid_kind = GRID_KINDS[self.kind]
        d.num_lods = len(self.resolutions) if self.kind == "hash" else self.num_lods
        d.feature_dim, d.multiscale = self.feature_dim, (0 if self.multiscale == "cat" else 1)
        d.lod_idx = self.lod_idx if self.kind == "hash" else self.num_lods
        return d

    def fill_decoders(self, d, dens_params: int, col_params: int) -> bool:
        """The embedding and decoder fields of NefDesc `d`; False (nothing written) when a decoder is deeper than WB_MAX_LAYERS."""
        if len(self.dens_dims) - 1 > A.WB_MAX_LAYERS or len(self.col_dims) - 1 > A.WB_MAX_LAYERS:
            return False
        d.pos_mode, d.pos_freq, d.view_mode, d.view_freq = self.pos_mode, self.pos_freq, self.view_mode, self.view_freq
        d.has_bias = int(self.has_bias)
        d.dens_layers, d.col_layers = len(self.dens_dims) - 1, len(self.col_dims) - 1
        for i, v in enumerate(self.dens_dims):
            d.dens_dims[i] = v
        for i, v in enumerate(self.col_dims):
            d.col_dims[i] = v
        d.dens_params, d.col_params = dens_params, col_params
        return True


def triplane_wants_channel_last(spec: "NefSpec") -> bool:
    """The fused kernels read a 4-channel texel as one 16-byte load (and reduce its gradient with one 16-byte red) when the planes
    are channel-last; the reference's nn.Parameter layout [1, fdim, H, W] (triplanar_grid.py:178-180) costs four 4-byte accesses."""
    return spec.kind == "triplanar" and spec.feature_dim == 12


def triplane_relayout(src: Sequence[torch.Tensor], to_channel_last: bool, out: Optional[Sequence[torch.Tensor]] = None) -> List[torch.Tensor]:
    """All planes in one native launch (wb_triplane_relayout): [1, C, H, W] -> [H, W, C] fp32 copies, or back (into `out` if given)."""
    src = [A.f32c(t) for t in src]
    A.require_device(src[0])
    if to_channel_last:
        Cc = int(src[0].shape[1]); sizes = [int(t.shape[2]) for t in src]
        dst = [torch.empty((n, n, Cc), dtype=torch.float32, device=t.device) for n, t in zip(sizes, src)] if out is None else list(out)
    else:
        Cc = int(src[0].shape[2]); sizes = [int(t.shape[0]) for t in src]
        dst = [torch.empty((1, Cc, n, n), dtype=torch.float32, device=t.device) for n, t in zip(sizes, src)] if out is None else list(out)
    n = len(src)
    sp = (C.c_void_p * n)(*[t.data_ptr() for t in src]); dp = (C.c_void_p * n)(*[t.data_ptr() for t in dst])
    sz = (C.c_int32 * n)(*sizes)
    A.lib().wb_triplane_relayout(sp, dp, sz, n, Cc, 1 if to_channel_last else 0, A.stream())
    return dst


def _flatten(params: Sequence[torch.Tensor]) -> torch.Tensor:
    return torch.cat([p.detach().reshape(-1).float() for p in params]) if params else torch.zeros(0)


def _embedder_mode(emb):
    """(mode, freq) of an embedder object (nerf.py:110-141): None -> (0, 0); nn.Identity -> (1, 0); PositionalEmbedder with the
    get_positional_embedder bands 2^0..2^(f-1) -> (3 | 2, f); anything else (e.g. the tcnn spherical harmonics) -> None."""
    if emb is None:
        return 0, 0
    if isinstance(emb, torch.nn.Identity):
        return 1, 0
    nf = getattr(emb, "num_freq", None)
    if nf is None or not getattr(emb, "log_sampling", True):
        return None
    nf = int(nf)
    if nf < 1 or int(round(float(getattr(emb, "max_freq_log2", nf - 1)))) != nf - 1 or int(getattr(emb, "out_dim", 0)) not in (6 * nf, 3 + 6 * nf):
        return None
    return (3 if getattr(emb, "include_input", True) else 2), nf


def _embed_width(mode: int, freq: int) -> int:
    """Width of an embedding of _embedder_mode (mode, freq)."""
    return 0 if mode == 0 else 3 if mode == 1 else 6 * freq + (3 if mode == 3 else 0)


def _decoder_layers(dec):
    """Linear layers of a BasicDecoder(relu, no skip) (basic_decoders.py:59-101), or None."""
    if getattr(dec, "skip", None) or getattr(dec, "activation", torch.relu) not in (torch.relu, torch.nn.functional.relu):
        return None
    layers = list(dec.layers) + [dec.lout]
    if not all(isinstance(l, torch.nn.Linear) for l in layers):
        return None
    return layers


def decoder_params(dec) -> List[torch.Tensor]:
    """[W0, b0?, W1, b1?, ...] -- the order the C ABI expects (include/wispb200.h)."""
    out = []
    for l in list(dec.layers) + [dec.lout]:
        out.append(l.weight)
        if l.bias is not None:
            out.append(l.bias)
    return out


def raymarch_level(grid, lod_idx: int) -> int:
    """Octree level the tracer marches (BLASGrid.raymarch overrides: hash_grid.py:235-240 max_level, octree_grid.py:221-226 base_lod,
    triplanar_grid.py:145-150 level 0)."""
    if hasattr(grid, "codebook"):
        return grid.blas.max_level
    if hasattr(grid, "trinkets"):
        return grid.base_lod
    return 0


def raytrace_level(grid, lod_idx: int) -> int:
    """Octree level PackedSDFTracer raytraces (packed_sdf_tracer.py:86 asks for active_lods[lod_idx]; BLASGrid.raytrace passes it
    through, blas_grid.py:42-45, and TriplanarGrid.raytrace traces level 0 of its AABB blas instead, triplanar_grid.py:152-157)."""
    if hasattr(grid, "codebook") or hasattr(grid, "trinkets"):
        return grid.active_lods[lod_idx]
    return 0


def _hash_begin(g) -> List[int]:
    """MultiTable.begin_idxes of a hash grid as host ints: one device read, cached on the grid (the table layout never changes)."""
    begin = getattr(g, "_wb_begin", None)
    if begin is None or len(begin) != len(g.resolutions) + 1:
        begin = [int(b) for b in g.codebook.begin_idxes.tolist()]
        try:
            g._wb_begin = begin
        except Exception:
            pass
    return begin


def nef_spec(nef, lod_idx: Optional[int] = None) -> Optional[NefSpec]:
    """Describe a NeuralRadianceField -- this package's mirror or the reference's own class (install()) -- for the fused path, or
    None when something is outside it (embedders other than none/identity/positional, activations other than relu, skip
    connections, grids other than Hash/Triplanar/Octree 'linear')."""
    g = getattr(nef, "grid", None)
    if g is None or getattr(nef, "activation_type", "relu") != "relu" or getattr(nef, "layer_type", "linear") not in ("linear", "none"):
        return None
    ld, lc = _decoder_layers(nef.decoder_density), _decoder_layers(nef.decoder_color)
    pe, ve = _embedder_mode(getattr(nef, "pos_embedder", None)), _embedder_mode(getattr(nef, "view_embedder", None))
    if ld is None or lc is None or pe is None or ve is None:
        return None
    if lod_idx is None:
        lod_idx = len(g.active_lods) - 1
    lod_idx = int(lod_idx)
    has_bias = ld[0].bias is not None
    if any((l.bias is not None) != has_bias for l in ld + lc):
        return None
    dims = lambda ls: [ls[0].in_features] + [l.out_features for l in ls]
    common = dict(multiscale=g.multiscale_type, pos_mode=pe[0], pos_freq=pe[1], view_mode=ve[0], view_freq=ve[1], has_bias=has_bias,
                  dens_dims=dims(ld), col_dims=dims(lc))
    if g.multiscale_type not in ("cat", "sum"):
        return None
    if hasattr(g, "codebook"):                                   # HashGrid
        if g.feature_dim > 8 or getattr(g, "coord_dim", 3) != 3:
            return None
        begin = _hash_begin(g)
        return NefSpec(resolutions=[int(r) for r in g.resolutions], begin_idxes=begin, codebook_size=int(g.codebook_size),
                       feature_dim=int(g.feature_dim), lod_idx=lod_idx, kind="hash", num_lods=len(g.resolutions), **common)
    nl = lod_idx + 1
    if nl > 12 or getattr(g, "interpolation_type", "linear") != "linear":
        return None
    if hasattr(g, "trinkets"):                                    # OctreeGrid (the VQAD CodebookOctreeGrid keeps indices, not features)
        if g.feature_dim > 32 or hasattr(g, "dictionary"):
            return None
        spec = NefSpec(resolutions=[], begin_idxes=[], codebook_size=0, feature_dim=int(g.feature_dim), lod_idx=lod_idx, kind="octree",
                       num_lods=nl, base_lod=int(g.base_lod), half_round=bool(getattr(g, "half_features", True)), **common)
    elif all(hasattr(f, "fmx") for f in getattr(g, "features", [])) and len(getattr(g, "features", [])) > 0:      # TriplanarGrid
        fdim = g.features[0].fmx.shape[1]
        if fdim > 8 or any(getattr(f, "padding_mode", "reflection") != "reflection" for f in g.features):
            return None
        spec = NefSpec(resolutions=[int(g.features[i].fmx.shape[-1]) - 1 for i in range(nl)], begin_idxes=[], codebook_size=0,
                       feature_dim=3 * int(fdim), lod_idx=lod_idx, kind="triplanar", num_lods=nl, **common)
    else:
        return None
    feat = spec.feature_dim if (g.multiscale_type == "sum" or (spec.kind == "octree" and nl == 1)) else nl * spec.feature_dim
    if spec.dens_dims[0] != feat + _embed_width(*pe):                    # e.g. 'cat' evaluated below its finest LOD: the reference fails in nn.Linear
        return None
    return spec


def grid_tensors(nef, spec: NefSpec) -> List[torch.Tensor]:
    """The grid's trainable tensors in the order NefSpec.desc expects."""
    g = nef.grid
    if spec.kind == "hash":
        return [g.codebook.feats]
    if spec.kind == "triplanar":
        out = []
        for i in range(spec.num_lods):
            f = g.features[i]
            out += [f.fmx, f.fmy, f.fmz]
        return out
    return [g.features[i] for i in range(spec.num_lods)]


def _grid_context(nef, spec: NefSpec):
    """(OctreeTensors, trinkets) of an octree-grid field, else (None, None)."""
    if spec.kind != "octree":
        return None, None
    g = nef.grid
    dev = g.features[0].device
    if g.trinkets.device != dev:
        g.trinkets = g.trinkets.to(dev)
    return octree_tensors(g.blas), g.trinkets.int().contiguous()


class RFTraceFn(torch.autograd.Function):
    """PackedRFTracer.trace + NeuralRadianceField.rgba + grid.interpolate as one native pipeline:
         march(count/scan/fill) -> shade (gather + decoders fused) -> composite        (forward)
         composite_bwd -> shade_bwd (decoder recompute, grid scatter)                   (backward)
    Inputs: the grid tensors (NefSpec order), then the decoder parameters in packing order [W0, b0?, W1, b1?, ...] for density
    then colour.
    """

    @staticmethod
    def forward(ctx, ms: MarchState, spec: NefSpec, n_grid: int, n_dens: int, bg, precision: int, want_grad: bool, octctx, *tensors):
        grid, params = tensors[:n_grid], tensors[n_grid:]
        A.require_device(grid[0])
        L = A.lib()
        dev = grid[0].device
        gt = [A.f32c(t.detach()) for t in grid]
        layout = 1 if triplane_wants_channel_last(spec) else 0
        if layout:                                          # channel-last copies of the planes (one launch, 17 MB at config 4)
            gt = triplane_relayout(gt, True)
        dens_flat, col_flat = _flatten(params[:n_dens]), _flatten(params[n_dens:])
        oct, trinkets = octctx if octctx is not None else (None, None)
        desc, keep = spec.desc(gt, dens_flat, col_flat, oct, trinkets, layout=layout)
        nblob = int(L.wb_rf_param_blob_floats(desc, precision))
        if nblob < 0:
            raise A.WispB200Error(L.wb_last_error().decode())
        blob = torch.empty(nblob, dtype=torch.float32, device=dev)
        L.wb_rf_pack_params(desc, precision, A.ptr(blob), A.stream())
        rec_t, rec_delta, rec_ray = march_fill_records(ms, dev)
        S, R = ms.total, ms.rays.num_rays
        shaded = _empty_s(S, (4,), torch.float32, dev)
        # grad mode is always off inside Function.forward and needs_input_grad ignores torch.no_grad(): the caller (rf_trace_nef)
        # tells us whether a backward pass can follow, so that inference neither saves features nor needs the backward tiles
        need_grad = bool(want_grad) and any(ctx.needs_input_grad[8:])
        Scap = _bucket(S)                                  # byte sizes for the bucketed capacity (layouts still use S)
        wsb = int(L.wb_rf_workspace_bytes(desc, precision, R, Scap, 0))
        ws = torch.empty(wsb, dtype=torch.uint8, device=dev) if wsb > 0 else None
        fb = int(L.wb_rf_feat_bytes(desc, precision, Scap)) if need_grad else 0
        if fb < 0 or wsb < 0:        # e.g. the tensor-core backward of this decoder does not fit: fail at the forward, not mid-backward
            raise A.WispB200Error(L.wb_last_error().decode())
        feat = torch.empty(fb, dtype=torch.uint8, device=dev) if fb > 0 else None
        with _stage("shade_fwd"):
            L.wb_rf_shade_fwd(desc, A.ptr(blob), precision, ms.rays, A.ptr(rec_t), A.ptr(rec_ray),
                              S, A.ptr(shaded), A.ptr(feat), A.ptr(ws), A.stream())
        rgb = torch.empty((R, 3), dtype=torch.float32, device=dev)
        depth = torch.empty((R, 1), dtype=torch.float32, device=dev)
        alpha = torch.empty((R, 1), dtype=torch.float32, device=dev)
        hit = torch.empty(R, dtype=torch.bool, device=dev)
        bgv = _bg3(bg)
        with _stage("composite_fwd"):
            L.wb_composite_fwd(A.ptr(shaded), A.ptr(rec_t), A.ptr(rec_delta), A.ptr(ms.offsets), R, bgv,
                               A.ptr(rgb), A.ptr(depth), A.ptr(alpha), A.ptr(hit), A.stream())
        ctx.ms, ctx.spec, ctx.n_grid, ctx.n_dens, ctx.bg, ctx.precision, ctx.octctx = ms, spec, n_grid, n_dens, bgv, precision, octctx
        ctx.layout = layout
        ctx.param_shapes = [p.shape for p in params]
        ctx.feat = feat
        ctx.save_for_backward(dens_flat, col_flat, blob, rec_t, rec_delta, rec_ray, shaded, *gt)
        ctx.mark_non_differentiable(hit)
        return rgb, depth, alpha, hit

    @staticmethod
    def backward(ctx, g_rgb, g_depth, g_alpha, _g_hit):
        dens_flat, col_flat, blob, rec_t, rec_delta, rec_ray, shaded, *gt = ctx.saved_tensors
        ms, spec = ctx.ms, ctx.spec
        L = A.lib()
        S, R = ms.total, ms.rays.num_rays
        oct, trinkets = ctx.octctx if ctx.octctx is not None else (None, None)
        g_grid = [torch.zeros_like(t) for t in gt]
        desc, keep = spec.desc(gt, dens_flat, col_flat, oct, trinkets, grads=g_grid, layout=ctx.layout)
        g_table = g_grid[0] if spec.kind == "hash" else None
        g_sh = _empty_s(S, (4,), torch.float32, shaded.device)
        gd = A.f32c(g_depth).reshape(-1) if g_depth is not None else None
        ga = A.f32c(g_alpha).reshape(-1) if g_alpha is not None else None
        grgb = A.f32c(g_rgb)
        absmax = torch.zeros(1, dtype=torch.float32, device=shaded.device) if ctx.precision == 1 else None
        with _stage("composite_bwd"):
            L.wb_composite_bwd(A.ptr(shaded), A.ptr(rec_t), A.ptr(rec_delta), A.ptr(ms.offsets), R, ctx.bg,
                               A.ptr(grgb), A.ptr(gd), A.ptr(ga), A.ptr(g_sh), A.ptr(absmax), A.stream())
        g_dens = torch.zeros_like(dens_flat)
        g_col = torch.zeros_like(col_flat)
        scale = None
        if ctx.precision == 1 and S > 0:
            # power-of-two loss scale computed on the device (no host sync): largest |gradient| -> ~64 in fp16
            scale = torch.empty(1, dtype=torch.float32, device=shaded.device)
            L.wb_rf_loss_scale(A.ptr(absmax), A.ptr(scale), A.stream())
        wsb = int(L.wb_rf_workspace_bytes(desc, ctx.precision, R, _bucket(S), 1))
        ws = torch.empty(wsb, dtype=torch.uint8, device=shaded.device) if wsb > 0 else None
        if ctx.precision == 1 and S > 0 and SPLIT_BWD:        # the two stages as separate launches (profiling; WB_SPLIT_BWD=1)
            with _stage("decoder_bwd"):
                L.wb_rf_decoder_bwd(desc, A.ptr(blob), ms.rays, A.ptr(rec_t), A.ptr(rec_ray), S, A.ptr(g_sh),
                                    A.ptr(scale), A.ptr(ctx.feat), A.ptr(ws), A.ptr(g_dens), A.ptr(g_col), A.stream())
            with _stage("table_scatter"):
                L.wb_rf_table_scatter(desc, ms.rays, A.ptr(rec_t), A.ptr(rec_ray), S, A.ptr(scale), A.ptr(ws),
                                      A.ptr(g_table), A.stream())
        else:   # precision 1: decoder backward with the hash-table scatter fused into its last epilogue (one kernel) where the shape allows
            with _stage("shade_bwd"):
                L.wb_rf_shade_bwd(desc, A.ptr(blob), ctx.precision, ms.rays, A.ptr(rec_t), A.ptr(rec_ray),
                                  S, A.ptr(g_sh), A.ptr(scale), A.ptr(ctx.feat), A.ptr(ws), A.ptr(g_table), A.ptr(g_dens), A.ptr(g_col), A.stream())
        grads = []
        for flat, shapes in ((g_dens, ctx.param_shapes[:ctx.n_dens]), (g_col, ctx.param_shapes[ctx.n_dens:])):
            o = 0
            for shp in shapes:
                n = int(torch.Size(shp).numel())
                grads.append(flat[o:o + n].reshape(shp)); o += n
        if ctx.layout:                                      # gradients back into the layout of the plane parameters
            g_grid = triplane_relayout(g_grid, False)
        return (None, None, None, None, None, None, None, None, *g_grid, *grads)


_SUPPORT_CACHE: dict = {}


def precision_supported(spec: NefSpec, nef, precision: int, backward: bool) -> bool:
    """Host-side query (wb_rf_precision_supported): can this decoder configuration run at `precision`?  Depends only on the
    static description, so the answer is memoised (the tracer asks once per trace() call)."""
    if precision == 0:
        return True
    key = (spec.kind, spec.feature_dim, spec.num_lods, spec.multiscale, spec.lod_idx, spec.pos_mode, spec.pos_freq, spec.view_mode, spec.view_freq,
           spec.has_bias, tuple(spec.dens_dims), tuple(spec.col_dims), int(precision), bool(backward))
    ans = _SUPPORT_CACHE.get(key)
    if ans is None:
        # the query looks at widths only: stand-in one-element tensors, no parameter flattening
        dummy = torch.zeros(1)
        d = spec.header()
        ans = spec.fill_decoders(d, dummy.data_ptr(), dummy.data_ptr()) and bool(A.lib().wb_rf_precision_supported(d, precision, 1 if backward else 0))
        _SUPPORT_CACHE[key] = ans
    return ans


def resolve_precision(precision: Optional[int], spec: NefSpec, nef, backward: bool) -> int:
    """Decoder arithmetic of a fused trace: 0 = fp32, 1 = fp16 tensor cores with fp32 accumulation.  An explicit precision is taken
    literally (an unsupported configuration raises); None follows autocast and quietly stays on the fp32 kernels when the decoders
    do not fit the tensor-core path (both are native CUDA)."""
    if precision is not None:
        return int(precision)
    return 1 if (torch.is_autocast_enabled() and precision_supported(spec, nef, 1, backward)) else 0


def rf_trace_nef(ms: MarchState, spec: NefSpec, nef, bg, precision: int = 0):
    """Fused trace of `nef` (mirror or reference class) over the marched samples -> rgb [R,3], depth [R,1], alpha [R,1], hit [R]."""
    grid = grid_tensors(nef, spec)
    dens, col = decoder_params(nef.decoder_density), decoder_params(nef.decoder_color)
    octctx = _grid_context(nef, spec) if spec.kind == "octree" else None
    return RFTraceFn.apply(ms, spec, len(grid), len(dens), bg, precision, torch.is_grad_enabled(), octctx, *grid, *dens, *col)


# --------------------------------------------------------------------------------------------------------------
# NeuralRadianceField.prune
# --------------------------------------------------------------------------------------------------------------
_PRUNE_CALLS = 0


def prune_field(nef, jitter: Optional[torch.Tensor] = None, seed: Optional[int] = None, group=None) -> bool:
    """NeuralRadianceField.prune (nerf.py:175-212) on the native path: probe points (wb_prune_samples) -> density through the fused
    shade kernel (grid gather + decoders, no torch nn.Linear) -> occupancy decay / max / threshold (wb_prune_update) -> octree
    rebuilt from the surviving cells.  Returns False (nothing touched) when the field is outside the fused path, so that callers
    can fall back to the reference body; True otherwise (including the reference's early returns).

    Rank consistency (SURVEY 8(e)): the probe points come from a counter-based stream keyed by `seed` (default: the number of
    prune calls so far, identical on every rank), and with torch.distributed initialised the updated occupancy is broadcast from
    rank 0 before thresholding, so every rank rebuilds the same octree even if the parameters have drifted by a rounding."""
    global _PRUNE_CALLS
    if getattr(nef, "prune_density_decay", None) is None or getattr(nef, "prune_min_density", None) is None:
        return True
    g = getattr(nef, "grid", None)
    if g is None:
        return True
    if not hasattr(g, "occupancy") or not hasattr(g, "dense_points"):
        return False
    spec = nef_spec(nef, None)
    if spec is None:
        return False
    grid = grid_tensors(nef, spec)
    dev = grid[0].device
    if dev.type != "cuda":
        return False
    A.require_device(grid[0])
    L = A.lib()
    points = g.dense_points.to(dev).contiguous()
    if points.dtype != torch.int16:
        points = points.to(torch.int16)
    N = points.shape[0]
    level = g.blas.max_level
    occ = A.f32c(g.occupancy.to(dev)).clone()
    if seed is None:
        seed = 0x5EED0000 + _PRUNE_CALLS
    _PRUNE_CALLS += 1
    u = None if jitter is None else A.f32c(jitter.to(dev))
    if u is not None and tuple(u.shape) != (N, 3):
        raise A.WispB200Error(f"prune jitter must be [{N}, 3]")
    samples = torch.empty((N, 3), dtype=torch.float32, device=dev); dirs = torch.empty_like(samples)
    rec_t = torch.empty(N, dtype=torch.float32, device=dev); rec_ray = torch.empty(N, dtype=torch.int32, device=dev)
    with _stage("prune_samples"):
        L.wb_prune_samples(A.ptr(points), N, level, A.ptr(u), seed & 0xFFFFFFFF, A.ptr(samples), A.ptr(dirs),
                           A.ptr(rec_t), A.ptr(rec_ray), A.stream())
    gt = [A.f32c(t.detach()) for t in grid]
    dens_flat, col_flat = _flatten(decoder_params(nef.decoder_density)), _flatten(decoder_params(nef.decoder_color))
    oct, trinkets = _grid_context(nef, spec)
    desc, keep_alive = spec.desc(gt, dens_flat, col_flat, oct, trinkets)
    blob = torch.empty(int(L.wb_rf_param_blob_floats(desc, 0)), dtype=torch.float32, device=dev)
    L.wb_rf_pack_params(desc, 0, A.ptr(blob), A.stream())
    rays, keep_rays = A.make_rays(samples, dirs, 0.0, 0.0)
    shaded = torch.empty((N, 4), dtype=torch.float32, device=dev)
    with _stage("prune_density"):             # fp32 decoders: the reference probes under torch.no_grad() outside autocast
        L.wb_rf_shade_fwd(desc, A.ptr(blob), 0, rays, A.ptr(rec_t), A.ptr(rec_ray), N, A.ptr(shaded),
                          None, None, A.stream())
    keep = torch.empty(N, dtype=torch.bool, device=dev)
    with _stage("prune_update"):
        L.wb_prune_update(A.ptr(shaded), N, float(nef.prune_density_decay), float(nef.prune_min_density),
                          A.ptr(occ), A.ptr(keep), A.stream())
    import torch.distributed as dist
    if dist.is_available() and dist.is_initialized() and dist.get_world_size(group) > 1:
        dist.broadcast(occ, src=dist.get_global_rank(group, 0) if group is not None else 0, group=group)
        keep = occ > float(nef.prune_min_density)
    g.occupancy = occ
    kept = points[keep]
    if kept.shape[0] == 0:
        return True
    cls = g.blas.__class__
    if not hasattr(cls, "from_quantized_points"):
        raise Exception(f"The BLAS {cls.__name__} does not support initialization from_quantized_points, which is required for pruning.")
    g.blas = cls.from_quantized_points(kept, level)
    return True


# --------------------------------------------------------------------------------------------------------------
# mesh SDF labels (wisp/ops/mesh/compute_sdf.py): the dataset side of app/nglod
# --------------------------------------------------------------------------------------------------------------
def compute_sdf(V: torch.Tensor, F: torch.Tensor, points: torch.Tensor, split_size: int = 10 ** 6) -> torch.Tensor:
    """wisp.ops.mesh.compute_sdf (compute_sdf.py:18-45): the signed distance from each point to the mesh (V, F) -> f64 [N, 1] on the
    current CUDA device, the value the reference's kernel (mesh2sdf_gpu_fast_nopre) returns for the same inputs in float64, in one
    wb_mesh_sdf call that culls pairs through a bounding-volume hierarchy built per call.
    V: [#V, 3] and points: [N, 3], float32 or float64 on any device (float32 widens to float64 exactly, so a float32 call returns the
    reference's answer for the .double() inputs; the reference itself refuses float32).  F: [#F, 3] integer indices into V.
    split_size: accepted for the reference's signature; the result does not depend on it (the reference splits the points only to
    bound its per-point scratch, which this route does not have).  Without a CUDA device it raises WispB200Error."""
    if not torch.cuda.is_available():
        raise A.WispB200Error("compute_sdf needs a CUDA device (H100, sm_90a); there is no CPU fallback")
    for name, t in (("V", V), ("points", points)):
        if t.dtype not in (torch.float32, torch.float64) or t.dim() != 2 or t.shape[1] != 3:
            raise A.WispB200Error(f"compute_sdf: {name} must be float32 or float64 [n, 3], got {t.dtype} {tuple(t.shape)}")
    if F.dtype.is_floating_point or F.dtype == torch.bool or F.dim() != 2 or F.shape[1] != 3:
        raise A.WispB200Error(f"compute_sdf: F must be integer [#F, 3], got {F.dtype} {tuple(F.shape)}")
    dev = torch.device("cuda", torch.cuda.current_device())
    pts = points.to(dev, torch.float64).contiguous()
    A.require_device(pts)
    out = torch.empty((pts.shape[0], 1), dtype=torch.float64, device=dev)
    if pts.shape[0] == 0:
        return out
    tris = V.to(dev, torch.float64)[F.to(dev, torch.int64)].reshape(-1, 9).contiguous()
    L = A.lib()
    nbytes = int(L.wb_mesh_sdf_workspace_bytes(tris.shape[0]))
    if nbytes < 0:
        raise A.WispB200Error(f"compute_sdf: {L.wb_last_error().decode()}")
    ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    with _stage("mesh_sdf"):
        L.wb_mesh_sdf(A.ptr(tris), tris.shape[0], A.ptr(pts), pts.shape[0], A.ptr(ws), nbytes, A.ptr(out), A.stream())
    return out


# --------------------------------------------------------------------------------------------------------------
# mesh octree (wisp/ops/spc/conversions.py:91-109): the octree OctreeAS.from_mesh builds, app/nglod's first step
# --------------------------------------------------------------------------------------------------------------
def mesh_to_octree(vertices: torch.Tensor, faces: torch.Tensor, level: int, num_samples: int = 10 ** 8,
                   seed: Optional[int] = None) -> torch.Tensor:
    """wisp.ops.spc.mesh_to_octree (conversions.py:91-109) -> the uint8 octree of `level` on the current CUDA device: the cells of
    num_samples area-weighted surface samples and of their jittered copies, drawn from the reference's distribution in one
    wb_mesh_octree_bits launch over a dense bitmask (no sample is materialised), then spc.points_to_octree of the set cells.
    vertices: float32 [#V, 3] (what OctreeAS.from_mesh passes), faces: integer [#F, 3], on any device.  The face areas are the
    reference's fp32 ones (0.5 |cross(v0 - v1, v1 - v2)|); their float64 prefix sum is the CDF the kernel inverts.
    seed: of the counter-based stream (DESIGN.md "Sampling contract"); None takes one from torch's default generator, so
    torch.manual_seed reproduces the octree.  Raises WispB200Error without a CUDA device, for a level outside 1..10, non-float32
    vertices, no faces, num_samples < 1, or a total area that is zero or not finite (the reference's Categorical refuses it)."""
    if not torch.cuda.is_available():
        raise A.WispB200Error("mesh_to_octree needs a CUDA device (H100, sm_90a); there is no CPU fallback")
    if isinstance(level, bool) or int(level) != level or not 1 <= int(level) <= 10:
        raise A.WispB200Error(f"mesh_to_octree: level must be 1..10 (the dense bitmask's limit), got {level!r}")
    level = int(level)
    if vertices.dtype != torch.float32 or vertices.dim() != 2 or vertices.shape[1] != 3:
        raise A.WispB200Error(f"mesh_to_octree: vertices must be float32 [#V, 3], got {vertices.dtype} {tuple(vertices.shape)}")
    if faces.dtype.is_floating_point or faces.dtype == torch.bool or faces.dim() != 2 or faces.shape[1] != 3 or faces.shape[0] == 0:
        raise A.WispB200Error(f"mesh_to_octree: faces must be integer [#F >= 1, 3], got {faces.dtype} {tuple(faces.shape)}")
    if int(num_samples) < 1:
        raise A.WispB200Error(f"mesh_to_octree: num_samples must be >= 1, got {num_samples}")
    if seed is None:
        seed = int(torch.randint(0, 2 ** 31 - 1, (1,)))
    dev = torch.device("cuda", torch.cuda.current_device())
    tris = vertices.to(dev)[faces.to(dev, torch.int64)]                                  # [T, 3, 3]
    A.require_device(tris)
    area = torch.norm(torch.cross(tris[:, 0] - tris[:, 1], tris[:, 1] - tris[:, 2], dim=1), p=2, dim=1) * 0.5
    cdf = torch.zeros(tris.shape[0] + 1, dtype=torch.float64, device=dev)
    torch.cumsum(area.double(), 0, out=cdf[1:])
    total = float(cdf[-1])
    if not (total > 0.0 and total != float("inf")):
        raise A.WispB200Error(f"mesh_to_octree: the total face area is {total} (it must be positive and finite)")
    tris = tris.reshape(-1, 9)
    bits = torch.zeros((8 ** level + 31) // 32, dtype=torch.int32, device=dev)
    with _stage("mesh_octree"):
        A.lib().wb_mesh_octree_bits(A.ptr(tris), A.ptr(cdf), tris.shape[0], int(num_samples), level,
                                    int(seed) & 0xFFFFFFFF, A.ptr(bits), A.stream())
    words = torch.nonzero(bits).reshape(-1)
    set_bits = (bits[words, None] >> torch.arange(32, dtype=torch.int32, device=dev)) & 1
    w, b = torch.nonzero(set_bits, as_tuple=True)
    idx = words[w] * 32 + b
    mask = (1 << level) - 1
    points = torch.stack([idx >> (2 * level), (idx >> level) & mask, idx & mask], 1).to(torch.int16)
    return spc.points_to_octree(points, level)
