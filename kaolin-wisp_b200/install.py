"""install(): route an importable kaolin-wisp through this path by overriding methods on wisp's own classes
(INTEGRATION.md section 3).  Nothing is patched unless `wisp` imports; WISP_B200=0 disables the hook.

What is patched (reference file:line -> native replacement):
  wisp.ops.grid.hashgrid                        (ops/grid.py:128-144)              ops.hashgrid ([N, 3] and, for app/image, [N, 2])
  OctreeAS.query / raytrace                     (octree_as.py:146-186)             wb_query / wb_raytrace_*
  OctreeAS._raymarch_ray / _voxel / _uniform    (octree_as.py:188-374)             wb_raymarch_*
  TriplanarGrid.interpolate                     (triplanar_grid.py:98-121)         wb_triplane_*
  OctreeGrid.interpolate                        (octree_grid.py:165-219)           wb_octree_interp_*
  PackedRFTracer.trace                          (packed_rf_tracer.py:84-181)       fused render path (ops.rf_trace_nef)
  PackedSDFTracer.trace                         (packed_sdf_tracer.py:57-174)      wb_sdf_trace
  PackedSPCTracer.trace                         (packed_spc_tracer.py:37-90)       wb_spc_trace (torch + OctreeAS.raytrace below max_level)
  NeuralSDF.sdf (no-grad)                       (neural_sdf.py:120-155)            wb_sdf_eval
  ImageNeuralField.rgb (no-grad)                (image_nef.py:77-97)               wb_image_eval
  NeuralRadianceField.prune                     (nerf.py:175-212)                  ops.prune_field
  wisp.ops.mesh.compute_sdf                     (ops/mesh/compute_sdf.py:18-45)    wb_mesh_sdf (ops.compute_sdf)
  wisp.ops.spc(.conversions).mesh_to_octree     (ops/spc/conversions.py:91-109)    wb_mesh_octree_bits (ops.mesh_to_octree)
Every replacement keeps the reference signature, falls back to the original method for configurations outside the native
path (unknown embedders, activations, grids), and keeps the attributes other wisp code reads (`prev_num_samples`, `bg_color`).
SPCField itself is not patched: its Kaolin calls build the octree (like OctreeAS's constructor) and its rgba() is plain torch.
The grid, SDF- and SPC-tracer replacements run the methods of this package's mirror classes (grids.py, tracers.py); the rest share
their host logic with the mirrors through ops (octree_tensors, march, resolve_precision, sdf_channel, image_rgb).
ImageTrainer.step itself is not patched: wisp_b200.ImageStep is its native counterpart (INTEGRATION.md).
"""
from __future__ import annotations

import os

import torch

from . import grids, ops, tracers

_ORIG = {}          # (class name, method) -> original function, for uninstall() and the fall-backs


def _seed() -> int:
    """The reference draws torch.rand per call (octree_as.py:273): a fresh seed of the counter-based stream per call."""
    return int(torch.randint(0, 2 ** 31 - 1, (1,)))


def _patch(cls, name, fn):
    key = (cls.__name__ if isinstance(cls, type) else cls.__name__, name)
    if key not in _ORIG:
        _ORIG[key] = (cls, getattr(cls, name))
    fn.__name__ = name
    fn.__wrapped__ = _ORIG[key][1]
    setattr(cls, name, fn)


def _mesh_to_octree(mod):
    """The replacement of `mod`.mesh_to_octree: levels 1..10 of float32 vertices go to ops.mesh_to_octree, the rest to the original."""
    key = (mod.__name__, "mesh_to_octree")

    def mesh_to_octree(vertices, faces, level, num_samples=100000000):
        if not (isinstance(level, int) and 1 <= level <= 10) or vertices.dtype != torch.float32:
            return _ORIG[key][1](vertices, faces, level, num_samples)
        return ops.mesh_to_octree(vertices, faces, level, num_samples)
    return mesh_to_octree


def uninstall() -> None:
    for (_, name), (cls, fn) in list(_ORIG.items()):
        setattr(cls, name, fn)
    _ORIG.clear()


def install() -> bool:
    if os.environ.get("WISP_B200", "1") == "0":
        return False
    try:
        import wisp.ops.grid as grid_ops
        from wisp.accelstructs import OctreeAS
        from wisp.accelstructs.base_as import ASQueryResults, ASRaymarchResults, ASRaytraceResults
        from wisp.core import RenderBuffer
        from wisp.models.grids import HashGrid, OctreeGrid, TriplanarGrid
        from wisp.models.nefs import NeuralRadianceField, NeuralSDF
        from wisp.tracers import PackedRFTracer, PackedSDFTracer, PackedSPCTracer
    except Exception:          # wisp (or one of its dependencies) is not importable here
        return False

    _patch(grid_ops, "hashgrid", lambda coords, codebook_bitwidth, lod_idx, codebook: ops.hashgrid(coords, codebook_bitwidth, lod_idx, codebook))

    # ---- OctreeAS ------------------------------------------------------------------------------------------------
    def query(self, coords, level=None, with_parents=False):
        return ASQueryResults(pidx=ops.query(ops.octree_tensors(self), coords, self.max_level if level is None else level, with_parents))

    def raytrace(self, rays, level=None, with_exit=False):
        ridx, pidx, depth, _ = ops.raytrace(ops.octree_tensors(self), rays.origins, rays.dirs, self.max_level if level is None else level)
        return ASRaytraceResults(ridx=ridx, pidx=pidx, depth=depth if with_exit else depth[:, 0:1].contiguous())

    def _raymarch_ray(self, rays, num_samples, level=None):
        ms = ops.march_count(ops.octree_tensors(self), rays.origins, rays.dirs, rays.dist_min, rays.dist_max, num_samples,
                             self.max_level if level is None else level, seed=_seed())
        ridx, samples, depth, deltas, boundary = ops.march_fill_reference_layout(ms, rays.origins.device)
        return ASRaymarchResults(ridx=ridx, samples=samples, depth_samples=depth, deltas=deltas, boundary=boundary, pack_info=None)

    def _nuggets(self, rays, num_samples, level, kind):
        _, ref = ops.march_nuggets(ops.octree_tensors(self), rays.origins, rays.dirs, self.max_level if level is None else level, num_samples, kind,
                                   reference_layout=True, seed=_seed())
        return ASRaymarchResults(pack_info=None, **ref)

    def _raymarch_voxel(self, rays, num_samples, level=None):
        return _nuggets(self, rays, num_samples, level, 'voxel')

    def _raymarch_uniform(self, rays, num_samples, level=None):
        return _nuggets(self, rays, num_samples, level, 'uniform')

    for name, fn in (("query", query), ("raytrace", raytrace), ("_raymarch_ray", _raymarch_ray), ("_raymarch_voxel", _raymarch_voxel),
                     ("_raymarch_uniform", _raymarch_uniform)):
        _patch(OctreeAS, name, fn)

    # ---- grids ---------------------------------------------------------------------------------------------------
    def triplanar_interpolate(self, coords, lod_idx):
        if self.interpolation_type != 'linear' or any(getattr(self.features[i], "padding_mode", "reflection") != "reflection" for i in range(lod_idx + 1)):
            return _ORIG[("TriplanarGrid", "interpolate")][1](self, coords, lod_idx)
        return grids.TriplanarGrid.interpolate(self, coords, lod_idx)

    def octree_interpolate(self, coords, lod_idx):
        if self.interpolation_type != 'linear':
            return _ORIG[("OctreeGrid", "interpolate")][1](self, coords, lod_idx)
        return grids.OctreeGrid.interpolate(self, coords, lod_idx)

    _patch(TriplanarGrid, "interpolate", triplanar_interpolate)
    _patch(OctreeGrid, "interpolate", octree_interpolate)

    # ---- radiance field tracer -----------------------------------------------------------------------------------
    orig_trace = PackedRFTracer.trace

    def rf_trace(self, nef, rays, channels, extra_channels, lod_idx=None, raymarch_type='voxel', num_steps=64, step_size=1.0, bg_color='white'):
        if lod_idx is None:
            lod_idx = nef.grid.num_lods - 1
        spec = None
        if isinstance(nef, NeuralRadianceField) and raymarch_type in ('ray', 'voxel', 'uniform') and not extra_channels:
            spec = ops.nef_spec(nef, lod_idx)
        if spec is None:
            return orig_trace(self, nef, rays, channels, extra_channels, lod_idx=lod_idx, raymarch_type=raymarch_type,
                              num_steps=num_steps, step_size=step_size, bg_color=bg_color)
        self.bg_color = self.bg_color.to(rays.origins.device)
        ms = ops.march(nef.grid, lod_idx, rays, raymarch_type, num_steps, seed=_seed())
        self.prev_num_samples = ms.total
        need_bwd = torch.is_grad_enabled() and any(p.requires_grad for p in nef.parameters())
        rgb, depth, alpha, hit = ops.rf_trace_nef(ms, spec, nef, self.bg_color, precision=ops.resolve_precision(None, spec, nef, need_bwd))
        return RenderBuffer(depth=depth if "depth" in channels else None, hit=hit, rgb=rgb, alpha=alpha)

    _patch(PackedRFTracer, "trace", rf_trace)

    # ---- SDF tracer ----------------------------------------------------------------------------------------------
    def sdf_trace(self, nef, rays, channels, extra_channels, lod_idx=None, num_steps=64, step_size=1.0, min_dis=1e-4):
        rb = tracers.PackedSDFTracer.trace(self, nef, rays, channels, extra_channels, lod_idx, num_steps, step_size, min_dis)
        # wisp code calls wisp's RenderBuffer methods (blend, image, exr_dict ...); the keyword order sets its fields' order
        return RenderBuffer(**{c: getattr(rb, c) for c in ("xyz", "depth", "hit", "normal", "rgb", "alpha", *extra_channels)})

    _patch(PackedSDFTracer, "trace", sdf_trace)

    orig_sdf = NeuralSDF.sdf

    def sdf(self, coords, lod_idx=None):
        return ops.sdf_channel(self, coords, lod_idx) or orig_sdf(self, coords, lod_idx)

    _patch(NeuralSDF, "sdf", sdf)

    # ---- SPC tracer (no Kaolin: mark_pack_boundaries is torch in the mirror's body) ------------------------------------------
    def spc_trace(self, nef, rays, channels, extra_channels, lod_idx=None):
        rb = tracers.PackedSPCTracer.trace(self, nef, rays, channels, extra_channels, lod_idx)
        return RenderBuffer(depth=rb.depth, hit=rb.hit, rgb=rb.rgb, alpha=rb.alpha)

    _patch(PackedSPCTracer, "trace", spc_trace)

    # ---- image field (app/image; a wisp without it keeps every other patch) ---------------------------------------
    try:
        from wisp.models.nefs.image_nef import ImageNeuralField
    except Exception:
        ImageNeuralField = None
    if ImageNeuralField is not None:
        orig_rgb = ImageNeuralField.rgb

        def image_rgb(self, coords, lod=None):
            fused = ops.image_rgb(self, coords, lod)
            return fused if fused is not None else orig_rgb(self, coords, lod)

        _patch(ImageNeuralField, "rgb", image_rgb)

    # ---- mesh SDF labels of the SDF datasets (a wisp whose wisp.ops.mesh does not import keeps every other patch) -----
    try:
        import wisp.ops.mesh as mesh_ops
    except Exception:
        mesh_ops = None
    if mesh_ops is not None:
        _patch(mesh_ops, "compute_sdf", lambda V, F, points, split_size=10 ** 6: ops.compute_sdf(V, F, points, split_size))

    # ---- mesh octree of OctreeAS.from_mesh (wisp.ops.spc) and of mesh_to_spc (its own module's global) --------------------
    try:
        import wisp.ops.spc as spc_ops
        import wisp.ops.spc.conversions as spc_conversions
    except Exception:
        spc_ops = None
    if spc_ops is not None:
        for mod in (spc_ops, spc_conversions):
            _patch(mod, "mesh_to_octree", _mesh_to_octree(mod))

    # ---- pruning -------------------------------------------------------------------------------------------------
    orig_prune = NeuralRadianceField.prune

    def prune(self):
        if not ops.prune_field(self):
            orig_prune(self)

    _patch(NeuralRadianceField, "prune", prune)
    return True
