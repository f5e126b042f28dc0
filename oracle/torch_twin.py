"""PyTorch-CPU twin of the reference hot path (TEST INFRASTRUCTURE, NOT PRODUCT CODE).

An op-for-op restatement, in plain differentiable torch ops, of what the reference executes per
tracer call (SURVEY.md 3.1).  Its two jobs:
  * cross-check the C oracle (oracle/wisp_oracle.c) forward values, and
  * provide ground-truth gradients (torch autograd) for the hand-written backward passes.
Kaolin externals are replaced by their SURVEY Appendix-A definitions; octree queries go through the
C oracle (integer work, no gradient).
"""
from __future__ import annotations

import numpy as np
import torch
import torch.nn.functional as F

from . import oracle as O

PRIMES = (1, 2654435761, 805459861)


def hash_corner_index(pos: torch.Tensor, res: int, T: int) -> torch.Tensor:
    """hash_utils.cuh:18-40 on int64 tensors [...,3] -> [...]."""
    if res < T and res * res < T and res * res * res < T:
        return pos[..., 0] + pos[..., 1] * res + pos[..., 2] * res * res
    m = 0xFFFFFFFF
    h = ((pos[..., 0] * PRIMES[0]) & m) ^ ((pos[..., 1] * PRIMES[1]) & m) ^ ((pos[..., 2] * PRIMES[2]) & m)
    return h % T


def hashgrid(coords: torch.Tensor, table: torch.Tensor, resolutions, codebook_bitwidth: int) -> torch.Tensor:
    """hashgrid_interpolate_3d_cuda_kernel (hashgrid_interpolate_cuda.cu:19-81), all levels -> [N, L*F]."""
    T = 2 ** codebook_bitwidth
    begin = O.table_layout(resolutions, codebook_bitwidth)
    outs = []
    cd = coords.detach().double()
    for l, res in enumerate(resolutions):
        hi = np.float32(np.float64(res - 1) - 1e-5)
        x = (res * (cd * 0.5 + 0.5)).float()
        x = torch.clamp(x, 0.0, float(hi))
        pos = torch.floor(x)
        w = x - pos
        iw = (1.0 - w.double()).float()
        pos = pos.long()
        tb = table[int(begin[l]): int(begin[l + 1])]
        acc = 0
        for j in range(8):
            off = torch.tensor([(j & 4) >> 2, (j & 2) >> 1, j & 1])
            idx = hash_corner_index(pos + off, res, T)
            cx = w[:, 0] if (j & 4) else iw[:, 0]
            cy = w[:, 1] if (j & 2) else iw[:, 1]
            cz = w[:, 2] if (j & 1) else iw[:, 2]
            coef = (cx * cy * cz)[:, None]
            acc = acc + tb[idx] * coef
        outs.append(acc)
    return torch.cat(outs, -1)


def grid_interpolate(coords, table, resolutions, bw, multiscale: str, lod_idx: int, F_: int) -> torch.Tensor:
    """HashGrid.interpolate post-ops (hash_grid.py:224-233)."""
    feats = hashgrid(coords, table, resolutions, bw)
    if multiscale == "cat":
        mask = torch.ones(feats.shape[-1])
        mask[lod_idx * F_:] = 0
        return feats * mask
    return feats.reshape(feats.shape[0], len(resolutions), F_).sum(-2)


def embed(mode: int, freq: int, x: torch.Tensor):
    """PositionalEmbedder.forward (positional_embedder.py:51-66)."""
    if mode == 0:
        return None
    if mode == 1:
        return x
    bands = 2.0 ** torch.linspace(0.0, freq - 1, freq)
    winded = (x[:, None] * bands[None, :, None]).reshape(x.shape[0], 3 * freq)
    enc = torch.cat([torch.sin(winded), torch.cos(winded)], -1)
    return torch.cat([x, enc], -1) if mode == 3 else enc


def mlp(x, Ws, bs):
    """BasicDecoder.forward (basic_decoders.py:73-101), relu, no skip."""
    h = x
    for i, W in enumerate(Ws[:-1]):
        h = torch.relu(F.linear(h, W, None if bs is None else bs[i]))
    return F.linear(h, Ws[-1], None if bs is None else bs[-1])


class TwinParams:
    """Differentiable copies of an oracle.Nef."""

    def __init__(self, nef: O.Nef):
        self.nef = nef
        t = lambda a: torch.tensor(np.asarray(a), dtype=torch.float32, requires_grad=True)
        self.table = t(nef.table)
        self.dW = [t(w) for w in nef.dens_W]; self.cW = [t(w) for w in nef.col_W]
        self.db = None if nef.dens_b is None else [t(b) for b in nef.dens_b]
        self.cb = None if nef.col_b is None else [t(b) for b in nef.col_b]

    def leaves(self):
        out = [self.table] + self.dW + self.cW
        if self.db is not None:
            out += self.db + self.cb
        return out

    def packed_grads(self):
        def flat(Ws, bs):
            parts = []
            for i, w in enumerate(Ws):
                parts.append((w.grad if w.grad is not None else torch.zeros_like(w)).reshape(-1))
                if bs is not None:
                    parts.append((bs[i].grad if bs[i].grad is not None else torch.zeros_like(bs[i])).reshape(-1))
            return torch.cat(parts).numpy()
        tg = self.table.grad if self.table.grad is not None else torch.zeros_like(self.table)
        return tg.numpy(), flat(self.dW, self.db), flat(self.cW, self.cb)


def rgba(p: TwinParams, coords: torch.Tensor, ray_d: torch.Tensor):
    """NeuralRadianceField.rgba (nerf.py:219-264)."""
    nef = p.nef
    lod = nef.L - 1 if nef.lod_idx is None else nef.lod_idx
    feats = grid_interpolate(coords, p.table, nef.resolutions, nef.codebook_bitwidth, nef.multiscale, lod, nef.feature_dim)
    pe = embed(nef.pos_mode, nef.pos_freq, coords)
    if pe is not None:
        feats = torch.cat([feats, pe], -1)
    df = mlp(feats, p.dW, p.db)
    ve = embed(nef.view_mode, nef.view_freq, ray_d)
    fdir = torch.cat([df, ve], -1) if ve is not None else df
    colors = torch.sigmoid(mlp(fdir[..., 1:], p.cW, p.cb))
    density = torch.relu(df[..., 0:1])
    return colors, density


def pack_index(boundary: torch.Tensor) -> torch.Tensor:
    return torch.cumsum(boundary.long(), 0) - 1


def cumsum_pack(x: torch.Tensor, boundary: torch.Tensor, exclusive: bool) -> torch.Tensor:
    """[KAOLIN-EXT] spc_render.cumsum: segmented prefix sum, restarted at every pack.  Formed as a running sum over all packs minus
    the sum before the pack, in float64 and rounded once: in float32 every pack would inherit the rounding error of the running
    sum of all the packs before it (the reference sums each pack on its own), and that error would depend on how the CPU's
    torch.cumsum orders its additions."""
    pid = pack_index(boundary)
    xd = x.double()
    cs = torch.cumsum(xd, 0)
    starts = torch.nonzero(boundary)[:, 0]
    base = torch.cat([torch.zeros(1, x.shape[1], dtype=torch.float64), cs])[starts]     # cumsum before each pack
    out = cs - base[pid]
    return (out - xd if exclusive else out).to(x.dtype)


def sum_reduce(x: torch.Tensor, boundary: torch.Tensor) -> torch.Tensor:
    pid = pack_index(boundary)
    P = int(boundary.sum())
    return torch.zeros(P, x.shape[1]).index_add(0, pid, x)


def exponential_integration(feats, tau, boundary, exclusive=True):
    """[KAOLIN-EXT] spc_render.exponential_integration (SURVEY K2)."""
    alpha = 1.0 - torch.exp(-tau)
    T = torch.exp(-1.0 * cumsum_pack(tau, boundary, exclusive))
    w = T * alpha
    return sum_reduce(w * feats, boundary), w


def raymarch_ray(spc: O.SPC, origins: torch.Tensor, dirs: torch.Tensor, near: float, far: float, n: int, jitter: torch.Tensor, level=None):
    """OctreeAS._raymarch_ray (octree_as.py:247-309) with torch.rand replaced by `jitter` [R,n]."""
    R = origins.shape[0]
    depth = torch.linspace(0, 1.0, n)[None] + (jitter / n)
    depth = depth * (far - near)
    depth = depth + near
    samples = torch.addcmul(origins[:, None], dirs[:, None], depth[..., None])
    pidx = torch.from_numpy(O.query(spc, samples.reshape(-1, 3).numpy(), level)).reshape(R, n)
    mask = pidx > -1
    idx = torch.nonzero(mask)
    deltas = depth.diff(dim=-1, prepend=(torch.zeros(R, 1) + near))
    d_s = depth[idx[:, 0], idx[:, 1]][:, None]
    dl = deltas[idx[:, 0], idx[:, 1]].reshape(-1, 1)
    smp = samples[idx[:, 0], idx[:, 1], :]
    ridx = idx[:, 0]
    boundary = torch.ones_like(ridx, dtype=torch.bool)
    boundary[1:] = ridx[1:] != ridx[:-1]
    return dict(ridx=ridx, samples=smp, depth_samples=d_s, deltas=dl, boundary=boundary, step_idx=idx[:, 1])


def trace(p: TwinParams, spc: O.SPC, origins, dirs, near, far, n, jitter, bg, level=None):
    """PackedRFTracer.trace (packed_rf_tracer.py:84-181) -> rgb[R,3], depth[R,1], alpha[R,1], hit[R]."""
    origins = torch.as_tensor(origins); dirs = torch.as_tensor(dirs)
    mr = raymarch_ray(spc, origins, dirs, near, far, n, torch.as_tensor(jitter), level)
    R = origins.shape[0]
    bg = torch.as_tensor(bg, dtype=torch.float32)
    ridx, boundary = mr["ridx"], mr["boundary"]
    hit_ray_d = dirs.index_select(0, ridx)
    color, density = rgba(p, mr["samples"], hit_ray_d)
    rgb = torch.zeros(R, 3) + bg
    depth = torch.zeros(R, 1); out_alpha = torch.zeros(R, 1)
    hit = torch.zeros(R, dtype=torch.bool)
    if ridx.shape[0] == 0:
        return rgb, depth, out_alpha, hit, mr
    ridx_hit = ridx[boundary]
    tau = density * mr["deltas"]
    ray_colors, w = exponential_integration(color, tau, boundary)
    ray_depth = sum_reduce(mr["depth_samples"] * w, boundary)
    alpha = sum_reduce(w, boundary)
    depth = depth.index_put((ridx_hit,), ray_depth)
    out_alpha = out_alpha.index_put((ridx_hit,), alpha)
    hit[ridx_hit] = alpha[..., 0] > 0.0
    rgb = rgb.index_put((ridx_hit,), bg * (1.0 - alpha) + ray_colors)
    return rgb, depth, out_alpha, hit, mr
