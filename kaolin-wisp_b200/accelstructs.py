"""OctreeAS: host-side mirror of wisp.accelstructs.OctreeAS (wisp/accelstructs/octree_as.py:37-440) whose
query / raymarch run on the sm_90a kernels behind the C ABI.  Result holders mirror base_as.py:18-84."""
from __future__ import annotations

from dataclasses import dataclass
from typing import List, Optional

import torch

from . import ops, spc


@dataclass
class ASQueryResults:
    pidx: torch.Tensor


@dataclass
class ASRaytraceResults:
    ridx: torch.Tensor
    pidx: torch.Tensor
    depth: torch.Tensor


@dataclass
class ASRaymarchResults:
    ridx: torch.Tensor
    samples: torch.Tensor
    depth_samples: torch.Tensor
    deltas: torch.Tensor
    boundary: torch.Tensor
    pack_info: Optional[torch.Tensor] = None


class OctreeAS:
    """Octree bottom-level acceleration structure over the SPC byte format (octree_as.py:43-62)."""

    def __init__(self, octree: torch.Tensor):
        self.octree = octree
        self.points, self.pyramid, self.prefix = spc.octree_to_spc(octree)
        self.max_level = self.pyramid.shape[-1] - 2
        self.extent = dict()
        self._tensors: Optional[ops.OctreeTensors] = None

    # --- constructors (octree_as.py:122-144) ---------------------------------------------------------------
    @classmethod
    def from_quantized_points(cls, quantized_points: torch.Tensor, level: int) -> "OctreeAS":
        return cls(spc.points_to_octree(quantized_points, level))

    @classmethod
    def from_pointcloud(cls, pointcloud: torch.Tensor, level: int) -> "OctreeAS":
        return cls(spc.points_to_octree(spc.quantize_points(pointcloud, level), level))

    @classmethod
    def make_dense(cls, level: int, device="cuda") -> "OctreeAS":
        return cls(spc.create_dense_octree(level, device=device))

    # --- native handle ---------------------------------------------------------------------------------------
    def tensors(self) -> ops.OctreeTensors:
        t = self._tensors
        if t is None or t.octree.data_ptr() != self.octree.data_ptr():
            t = ops.OctreeTensors(self.octree.contiguous(), self.prefix.contiguous(), self.points.contiguous(), self.pyramid.cpu(), self.max_level)
            self._tensors = t
        return t

    def to(self, device) -> "OctreeAS":
        self.octree, self.points, self.prefix = self.octree.to(device), self.points.to(device), self.prefix.to(device)
        self._tensors = None
        return self

    # --- queries (octree_as.py:146-163) ----------------------------------------------------------------------
    def query(self, coords, level=None, with_parents=False) -> ASQueryResults:
        if level is None:
            level = self.max_level
        return ASQueryResults(pidx=ops.query(self.tensors(), coords, level, with_parents))

    def raytrace(self, rays, level=None, with_exit=False) -> ASRaytraceResults:
        """octree_as.py:165-186: all ray / cell intersections ("nuggets") of `level`, by ray then front to back."""
        if level is None:
            level = self.max_level
        ridx, pidx, depth, _ = ops.raytrace(self.tensors(), rays.origins, rays.dirs, level)
        return ASRaytraceResults(ridx=ridx, pidx=pidx, depth=depth if with_exit else depth[:, 0:1].contiguous())

    def _raymarch_nuggets(self, rays, num_samples, level, kind, jitter=None, seed=0) -> ASRaymarchResults:
        _, ref = ops.march_nuggets(self.tensors(), rays.origins, rays.dirs, self.max_level if level is None else level, num_samples, kind,
                                   reference_layout=True, jitter=jitter, seed=seed)
        return ASRaymarchResults(pack_info=None, **ref)

    def _raymarch_voxel(self, rays, num_samples, level=None, jitter=None, seed=0) -> ASRaymarchResults:
        """octree_as.py:188-245."""
        return self._raymarch_nuggets(rays, num_samples, level, 'voxel', jitter, seed)

    def _raymarch_uniform(self, rays, num_samples, level=None) -> ASRaymarchResults:
        """octree_as.py:311-374."""
        return self._raymarch_nuggets(rays, num_samples, level, 'uniform')

    # --- raymarch (octree_as.py:380-429) ------------------------------------------------------------------------
    def _raymarch_ray(self, rays, num_samples, level=None, jitter=None, seed=0) -> ASRaymarchResults:
        ms = ops.march_count(self.tensors(), rays.origins, rays.dirs, rays.dist_min, rays.dist_max, num_samples,
                             self.max_level if level is None else level, jitter=jitter, seed=seed)
        ridx, samples, depth, deltas, boundary = ops.march_fill_reference_layout(ms, rays.origins.device)
        return ASRaymarchResults(ridx=ridx, samples=samples, depth_samples=depth, deltas=deltas, boundary=boundary, pack_info=None)

    def raymarch(self, rays, raymarch_type, num_samples, level=None, jitter=None, seed=0) -> ASRaymarchResults:
        if level is None:
            level = self.max_level
        if raymarch_type == 'voxel':
            return self._raymarch_voxel(rays=rays, num_samples=num_samples, level=level, jitter=jitter, seed=seed)
        elif raymarch_type == 'ray':
            return self._raymarch_ray(rays=rays, num_samples=num_samples, level=level, jitter=jitter, seed=seed)
        elif raymarch_type == 'uniform':
            return self._raymarch_uniform(rays=rays, num_samples=num_samples, level=level)
        else:
            raise TypeError(f"Raymarch sampler type: {raymarch_type} is not supported by OctreeAS.")

    def occupancy(self) -> List[int]:
        return self.pyramid[0, :-2].cpu().numpy().tolist()

    def capacity(self) -> List[int]:
        return [8 ** lod for lod in range(self.max_level)]

    def name(self) -> str:
        return "Octree"


class AxisAlignedBBoxAS(OctreeAS):
    """wisp.accelstructs.AxisAlignedBBoxAS (aabb_as.py:13-27): a one-level dense octree used as a bounding box."""

    def __init__(self, device="cuda"):
        super().__init__(spc.create_dense_octree(1, device=device))

    def name(self) -> str:
        return "AABB"
