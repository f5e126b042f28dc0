"""The hash grid in the float64 interval reference of NeuralSDF (TEST INFRASTRUCTURE, NOT PRODUCT CODE).

oracle/sdf_reference.py models NeuralSDF(OctreeGrid): its forward and train (and tests/sdf_deep_reference.py's train, which builds
on them) reach the grid only through three module functions -- cells (corner rows and coefficients), features (the blend) and
_scatter (the atomics of dL/dfeat).  This module adds a HashField and hooks those three functions for it; every other field takes
the unchanged octree functions, so octree results stay bit-identical.  Importing the module installs the hook.

Rounding points of a hash field (wb_sdf.cuh: sdf_hash_features, wb_sdf_train.cu: sdf_hash_scatter)
  cells      tests/grid_index_reference.py: corners (wb_cell, wb_corner_setup, wb_corner_indices).  Bit-exact.
  features   per LOD fl(v_0 c_0), then fmaf over corners 1..7 (wb_hashgrid_fwd's order); 'sum' adds all LODs in LOD order whatever
             lod_idx, 'cat' is L * F wide with the LODs >= lod_idx zero.  Bit-exact, radius 0.
  scatter    fl(g c_j) per sample, LOD and corner, one atomic each (colliding corners of one sample count separately); the zeroed 'cat'
             LODs get nothing."""
from __future__ import annotations

from dataclasses import dataclass
from typing import Sequence

import numpy as np

from oracle import sdf_reference as S

import grid_index_reference as GR

P1, P2 = GR.P1, GR.P2


@dataclass
class HashField(S.Field):
    """NeuralSDF(HashGrid): feats[l] = rows begin_idxes[l] .. begin_idxes[l+1] of codebook.feats; spc / trinkets unused."""
    resolutions: Sequence[int] = ()
    bitwidth: int = 19

    def table(self) -> np.ndarray:
        return np.concatenate(self.feats)


def hash_field(table, begin, resolutions, bitwidth, multiscale, Ws, bs, pos_mode=1, pos_freq=0) -> HashField:
    feats = [np.asarray(table[begin[l]:begin[l + 1]], np.float32) for l in range(len(resolutions))]
    return HashField(None, None, feats, 0, multiscale, [np.asarray(W, np.float32) for W in Ws], [np.asarray(b, np.float32) for b in bs],
                     pos_mode, pos_freq, False, [int(r) for r in resolutions], int(bitwidth))


def _hash_cells(field: HashField, coords: np.ndarray) -> S.Cells:
    c = np.asarray(coords, np.float32)
    oks, tks, cfs = [], [], []
    for res in field.resolutions:
        tk, cf = GR.corners(c, res, field.bitwidth)
        oks.append(np.ones(c.shape[0], bool)); tks.append(tk); cfs.append(cf.astype(np.float64))
    return S.Cells(oks, tks, cfs)


def _active(field: HashField, nl: int) -> int:
    """LODs the kernels evaluate: all of them for 'sum', those below lod_idx = nl - 1 for 'cat'."""
    return field.num_lods if field.multiscale == "sum" else nl - 1


def _hash_features(field: HashField, coords: np.ndarray, nl: int, exact: bool = False, cl=None):
    N, F, L = coords.shape[0], field.F, field.num_lods
    cl = cl or _hash_cells(field, coords)
    blends = []
    for l in range(_active(field, nl)):
        v = field.feats[l].astype(np.float64)[cl.tk[l]]                      # [N, 8, F]
        cf = cl.cf[l]
        if exact:
            a = (v * cf[:, :, None]).sum(1)
        else:
            a = S.r32(v[:, 0] * cf[:, :1])
            for j in range(1, 8):
                a = S.fma32(v[:, j], cf[:, j:j + 1], a)
        blends.append(a)
    if field.multiscale == "sum":
        c = np.zeros((N, F))
        for a in blends:
            c = c + a if exact else S.r32(c + a)
    else:
        c = np.concatenate(blends + [np.zeros((N, F))] * (L - len(blends)), -1)
    return c, np.zeros_like(c), np.zeros(N, bool), cl


def _hash_scatter(field: HashField, gx_c, gx_r, cl, nl, sum_, rnd):
    act = _active(field, nl)
    out = _octree_scatter(field, gx_c, gx_r, cl, act, field.multiscale == "sum", rnd) if act > 0 else []
    for l in range(act, field.num_lods):
        rows = field.feats[l].shape[0]
        out.append((np.zeros((rows, field.F)), np.zeros((rows, field.F)), np.zeros((rows, field.F)), np.zeros(rows)))
    return out


_octree_cells, _octree_features, _octree_scatter = S.cells, S.features, S._scatter


def cells(field, coords, nl):
    return _hash_cells(field, coords) if isinstance(field, HashField) else _octree_cells(field, coords, nl)


def features(field, coords, nl, exact=False, cl=None):
    return _hash_features(field, coords, nl, exact, cl) if isinstance(field, HashField) else _octree_features(field, coords, nl, exact, cl)


def _scatter(field, gx_c, gx_r, cl, nl, sum_, rnd):
    return _hash_scatter(field, gx_c, gx_r, cl, nl, sum_, rnd) if isinstance(field, HashField) else _octree_scatter(field, gx_c, gx_r, cl, nl, sum_, rnd)


if getattr(S, "_hash_hook", None) is None:
    S.cells, S.features, S._scatter = cells, features, _scatter
    S._hash_hook = True


def table_grad(tr: S.Train):
    """The per-LOD grid gradients of a Train as one codebook.feats gradient (centre, radius)."""
    return np.concatenate([c for c, _ in tr.grid]), np.concatenate([r for _, r in tr.grid])
