"""HashGrid / MultiTable: host-side mirrors of wisp.models.grids.HashGrid (wisp/models/grids/hash_grid.py:20-265)
and wisp.models.grids.utils.MultiTable (wisp/models/grids/utils.py:13-71).  Parameter names are the reference's
(`codebook.feats`, `codebook.begin_idxes`) so state_dicts and the trainer's name-based optimiser groups
(base_trainer.py:216-235) carry over."""
from __future__ import annotations

from typing import List, Optional, Tuple

import numpy as np
import torch
import torch.nn as nn

from . import ops, spc
from .accelstructs import ASRaymarchResults, OctreeAS


class MultiTable(nn.Module):
    def __init__(self, resolutions: Tuple[int, ...], coord_dim: int, feature_dim: int, std: float = 0.01, max_feats: Optional[int] = None):
        super().__init__()
        self.num_lods = len(resolutions)
        self.max_feats = max_feats
        self.register_buffer("begin_idxes", torch.zeros(self.num_lods + 1, dtype=torch.int64))
        self.register_buffer("num_feats", torch.zeros(self.num_lods, dtype=torch.int64))
        self.coord_dim = coord_dim
        self.feature_dim = feature_dim
        self.resolutions = torch.zeros([self.num_lods, 1], dtype=torch.int64)
        num_so_far = 0
        for i in range(self.num_lods):
            self.resolutions[i] = resolutions[i]
            n = int(resolutions[i]) ** coord_dim
            if max_feats:
                n = min(max_feats, n)
            self.begin_idxes[i] = num_so_far
            self.num_feats[i] = n
            num_so_far += n
        self.begin_idxes[self.num_lods] = num_so_far
        self.total_feats = num_so_far
        self.feats = nn.Parameter(torch.randn(self.total_feats, feature_dim) * std)

    def get_level(self, idx):
        return self.feats[self.begin_idxes[idx]:self.begin_idxes[idx + 1]]


class HashGrid(nn.Module):
    """Multi-resolution hash grid (hash_grid.py:27-89)."""

    def __init__(self, blas: OctreeAS, feature_dim: int, resolutions: List[int], multiscale_type: str = 'sum',
                 feature_std: float = 0.0, feature_bias: float = 0.0, codebook_bitwidth: int = 8, coord_dim: int = 3):
        super().__init__()
        assert coord_dim in (2, 3)                         # hash_grid.py:62
        self.blas = blas
        if blas is not None:
            lvl = blas.max_level
            s, c = int(blas.pyramid[1, lvl]), int(blas.pyramid[0, lvl])
            self.dense_points = blas.points[s:s + c].clone()
            self.num_cells = self.dense_points.shape[0]
            self.occupancy = torch.zeros(self.num_cells)
        self.feature_dim = feature_dim
        self.multiscale_type = multiscale_type
        self.feature_std = feature_std
        self.feature_bias = feature_bias
        self.codebook_bitwidth = codebook_bitwidth
        self.resolutions = [int(r) for r in resolutions]
        self.num_lods = len(resolutions)
        self.active_lods = [x for x in range(self.num_lods)]
        self.max_lod = self.num_lods - 1
        self.codebook_size = 2 ** codebook_bitwidth
        self.coord_dim = coord_dim
        self.codebook = MultiTable(self.resolutions, coord_dim, feature_dim, feature_std, self.codebook_size)

    @classmethod
    def from_octree(cls, blas, feature_dim, base_lod=2, num_lods=1, multiscale_type='sum', feature_std=0.0, feature_bias=0.0,
                    codebook_bitwidth=8, coord_dim=3):
        resolutions = [2 ** (base_lod + x) for x in range(num_lods)]
        return cls(blas, feature_dim, resolutions, multiscale_type, feature_std, feature_bias, codebook_bitwidth, coord_dim)

    @classmethod
    def from_geometric(cls, blas, feature_dim, num_lods, multiscale_type='sum', feature_std=0.0, feature_bias=0.0,
                       codebook_bitwidth=8, min_grid_res=16, max_grid_res=None, coord_dim=3):
        b = np.exp((np.log(max_grid_res) - np.log(min_grid_res)) / (num_lods - 1))          # hash_grid.py:160-161
        resolutions = [int(np.floor(min_grid_res * (b ** l))) for l in range(num_lods)]
        return cls(blas, feature_dim, resolutions, multiscale_type, feature_std, feature_bias, codebook_bitwidth, coord_dim)

    @classmethod
    def from_resolutions(cls, blas, feature_dim, resolutions=None, multiscale_type='sum', feature_std=0.0, feature_bias=0.0,
                         codebook_bitwidth=8, coord_dim=3):
        assert resolutions is not None, 'HashGrid.from_resolutions() constructor cannot accept a None resolutions arg.'
        return cls(blas, feature_dim, resolutions, multiscale_type, feature_std, feature_bias, codebook_bitwidth, coord_dim)

    def freeze(self):
        self.codebook.requires_grad_(False)

    def interpolate(self, coords, lod_idx):
        """hash_grid.py:205-233 (including the 'cat' zeroing of LODs >= lod_idx)."""
        output_shape = coords.shape[:-1]
        if coords.ndim == 3:
            batch, num_samples, coords_dim = coords.shape
            coords = coords.reshape(batch * num_samples, coords_dim)
        feats = ops.hashgrid(coords, self.codebook_bitwidth, lod_idx, self.codebook)
        if self.multiscale_type == 'cat':
            feats = feats.reshape(*output_shape, feats.shape[-1])
            mask = torch.ones(feats.shape[-1], device=feats.device, dtype=feats.dtype)
            mask[lod_idx * self.feature_dim:] = 0       # reference writes zeros in place (hash_grid.py:228)
            return feats * mask
        elif self.multiscale_type == 'sum':
            return feats.reshape(*output_shape, len(self.resolutions), feats.shape[-1] // len(self.resolutions)).sum(-2)
        else:
            raise NotImplementedError

    def raymarch(self, rays, raymarch_type, num_samples, level=None, **kw) -> ASRaymarchResults:
        return self.blas.raymarch(rays, raymarch_type=raymarch_type, num_samples=num_samples, level=self.blas.max_level, **kw)

    def raytrace(self, rays, level=None, with_exit=False):
        return self.blas.raytrace(rays, level=level, with_exit=with_exit)

    def query(self, coords, level=None, with_parents=False):
        return self.blas.query(coords, level=level, with_parents=with_parents)

    def name(self) -> str:
        return "Hash Grid"


class TriplanarFeatureVolume(nn.Module):
    """One LOD of a TriplanarGrid: three [1, fdim, fsize+1, fsize+1] feature planes (triplanar_grid.py:184-203)."""

    def __init__(self, fdim, fsize, std, bias):
        super().__init__()
        self.fsize, self.fdim = fsize, fdim
        self.fmx = nn.Parameter(torch.randn(1, fdim, fsize + 1, fsize + 1) * std + bias)
        self.fmy = nn.Parameter(torch.randn(1, fdim, fsize + 1, fsize + 1) * std + bias)
        self.fmz = nn.Parameter(torch.randn(1, fdim, fsize + 1, fsize + 1) * std + bias)
        self.padding_mode = 'reflection'


class TriplanarGrid(nn.Module):
    """wisp.models.grids.TriplanarGrid (triplanar_grid.py:24-150): parameter names features.N.fmx/fmy/fmz as in the reference."""

    def __init__(self, blas, feature_dim: int, log_base_resolution: int = 4, num_lods: int = 1, interpolation_type: str = 'linear',
                 multiscale_type: str = 'sum', feature_std: float = 0.0, feature_bias: float = 0.0):
        super().__init__()
        if interpolation_type != 'linear':
            raise ValueError(f"Interpolation mode '{interpolation_type}' is not supported")       # triplanar_grid.py:141
        self.blas = blas
        self.feature_dim = feature_dim * 3          # the reference multiplies by 3 planes (:74)
        self.num_lods, self.log_base_resolution = num_lods, log_base_resolution
        self.interpolation_type, self.multiscale_type = interpolation_type, multiscale_type
        self.feature_std, self.feature_bias = feature_std, feature_bias
        self.active_lods = [log_base_resolution + x for x in range(num_lods)]
        self.features = nn.ModuleList([TriplanarFeatureVolume(feature_dim, 2 ** i, feature_std, feature_bias) for i in self.active_lods])
        self.num_feat = sum(((2 ** i + 1) ** 2) * self.feature_dim * 3 for i in self.active_lods)

    def freeze(self):
        self.features.requires_grad_(False)

    def interpolate(self, coords, lod_idx):
        """triplanar_grid.py:98-121."""
        output_shape = coords.shape[:-1]
        if coords.ndim < 3:
            coords = coords[:, None]                 # (batch, 3) -> (batch, num_samples, 3), as the reference (:110-111)
        planes = []
        for i in range(lod_idx + 1):
            f = self.features[i]
            planes += [f.fmx, f.fmy, f.fmz]
        feats = ops.TriplaneInterpolate.apply(coords.reshape(-1, 3), lod_idx + 1, *planes)
        feats = feats.reshape(*coords.shape[:-1], feats.shape[-1])      # 'cat' keeps the inflated shape in the reference
        if self.multiscale_type == 'sum':
            feats = feats.reshape(*output_shape, lod_idx + 1, feats.shape[-1] // (lod_idx + 1)).sum(-2)
        return feats

    def raymarch(self, rays, raymarch_type, num_samples, level=None, **kw) -> ASRaymarchResults:
        """triplanar_grid.py:145-150: the blas is only used as an AABB tracer (level 0)."""
        return self.blas.raymarch(rays, raymarch_type=raymarch_type, num_samples=num_samples, level=0, **kw)

    def raytrace(self, rays, level=None, with_exit=False):
        """triplanar_grid.py:152-157: the blas is only used as an AABB tracer (level 0)."""
        return self.blas.raytrace(rays, level=0, with_exit=with_exit)

    def query(self, coords, level=None, with_parents=False):
        return self.blas.query(coords, level=level, with_parents=with_parents)

    def name(self) -> str:
        return "Triplanar Grid"


class OctreeGrid(nn.Module):
    """wisp.models.grids.OctreeGrid (octree_grid.py:24-226), 'linear' interpolation.  Parameters: features.0 ... features.N-1."""

    def __init__(self, blas, feature_dim: int, num_lods: int = 1, interpolation_type: str = 'linear', multiscale_type: str = 'cat',
                 feature_std: float = 0.0, feature_bias: float = 0.0):
        super().__init__()
        if interpolation_type != 'linear':
            raise Exception(f"Interpolation mode {interpolation_type} is not supported.")          # octree_grid.py:103,161
        self.blas = blas
        self.feature_dim, self.max_lod, self.num_lods = feature_dim, blas.max_level, num_lods
        self.base_lod = self.max_lod - self.num_lods + 1
        self.interpolation_type, self.multiscale_type = interpolation_type, multiscale_type
        self.feature_std, self.feature_bias = feature_std, feature_bias
        self.active_lods = [self.base_lod + x for x in range(self.num_lods)]
        self.points_dual, self.pyramid_dual, self.trinkets, self.parents = spc.make_trilinear_spc(blas.points, blas.pyramid)
        self.features = nn.ParameterList([])
        for al in self.active_lods:                                                                 # octree_grid.py:88-104
            fts = torch.zeros(int(self.pyramid_dual[0, al]) + 1, feature_dim) + feature_bias
            fts = fts + torch.randn_like(fts) * feature_std
            self.features.append(nn.Parameter(fts))
        self.num_feat = sum(int(self.pyramid_dual[0, al]) + 1 for al in self.active_lods)
        self.half_features = True        # the reference interpolates `feats.half()` and returns `.float()` (octree_grid.py:147-149)

    def freeze(self):
        for f in self.features:
            f.requires_grad_(False)

    def interpolate(self, coords, lod_idx):
        """octree_grid.py:165-219.  install() runs this body on the reference's OctreeGrid too, which has no `half_features` and
        always rounds the features to half (octree_grid.py:149)."""
        output_shape = coords.shape[:-1]
        dev = self.features[0].device
        if self.trinkets.device != dev:
            self.trinkets = self.trinkets.to(dev)
        feats = ops.OctreeInterpolate.apply(coords.reshape(-1, 3), ops.octree_tensors(self.blas), self.trinkets.int(), self.base_lod,
                                            self.multiscale_type if lod_idx > 0 else 'cat', getattr(self, "half_features", True),
                                            *[self.features[i] for i in range(lod_idx + 1)])
        return feats.reshape(*output_shape, feats.shape[-1])

    def raymarch(self, rays, raymarch_type, num_samples, level=None, **kw) -> ASRaymarchResults:
        """octree_grid.py:221-226: samples over the coarsest LOD that has features."""
        return self.blas.raymarch(rays, raymarch_type=raymarch_type, num_samples=num_samples, level=self.base_lod, **kw)

    def raytrace(self, rays, level=None, with_exit=False):
        return self.blas.raytrace(rays, level=level, with_exit=with_exit)

    def query(self, coords, level=None, with_parents=False):
        return self.blas.query(coords, level=level, with_parents=with_parents)

    def name(self) -> str:
        return "Octree Grid"


class CodebookOctreeGrid(OctreeGrid):
    """wisp.models.grids.CodebookOctreeGrid (codebook_grid.py:20-172): an OctreeGrid whose corner rows hold logits over a per-LOD
    dictionary of 2^codebook_bitwidth feature vectors (VQAD).  Parameters as in the reference: `dictionary.N` [2^bw, feature_dim],
    `features.N` [rows_N, 2^bw].  Evaluation is row-wise (csrc/wb_codebook.cu): selection once per row and LOD, then the ordinary
    native trilinear blend through the trinkets, in fp32 (the codebook grid does not cast to half, :164-165)."""

    def __init__(self, blas, feature_dim: int, num_lods: int = 1, interpolation_type: str = 'linear', multiscale_type: str = 'cat',
                 feature_std: float = 0.0, feature_bias: float = 0.0, codebook_bitwidth: int = 8):
        self.bitwidth = codebook_bitwidth
        super().__init__(blas, feature_dim, num_lods, interpolation_type, multiscale_type, feature_std, feature_bias)
        self.dictionary_size = 2 ** self.bitwidth
        rows = [int(f.shape[0]) for f in self.features]
        self.dictionary = nn.ParameterList([nn.Parameter(torch.randn(self.dictionary_size, feature_dim) * feature_std) for _ in self.active_lods])
        self.features = nn.ParameterList([nn.Parameter(torch.randn(r, self.dictionary_size) * feature_std) for r in rows])     # codebook_grid.py:92-96
        self.half_features = False

    def interpolate(self, coords, lod_idx):
        """octree_grid.py:165-219 with _index_features replaced by the row-wise selection."""
        output_shape = coords.shape[:-1]
        dev = self.features[0].device
        if self.trinkets.device != dev:
            self.trinkets = self.trinkets.to(dev)
        rows = [ops.CodebookRows.apply(self.features[i], self.dictionary[i], self.training) for i in range(lod_idx + 1)]
        feats = ops.OctreeInterpolate.apply(coords.reshape(-1, 3), ops.octree_tensors(self.blas), self.trinkets, self.base_lod,
                                            self.multiscale_type if lod_idx > 0 else 'cat', False, *rows)
        return feats.reshape(*output_shape, feats.shape[-1])

    def name(self) -> str:
        return "Codebook Grid"
