"""NeuralRadianceField and its parts: host-side mirrors of
  wisp.models.nefs.NeuralRadianceField   (wisp/models/nefs/nerf.py:25-295)
  wisp.models.nefs.BaseNeuralField       (wisp/models/nefs/base_nef.py:120-202, channel dispatch)
  wisp.models.decoders.BasicDecoder      (wisp/models/decoders/basic_decoders.py:16-101)
  wisp.models.embedders.PositionalEmbedder / get_positional_embedder (positional_embedder.py:15-100)
  wisp.models.nefs.ImageNeuralField      (wisp/models/nefs/image_nef.py:37-97)
  wisp.models.nefs.SPCField              (wisp/models/nefs/spc_field.py:19-157)
Module / parameter names are the reference's (decoder_density.layers.N.weight, decoder_color.lout.bias,
grid.codebook.feats ...).  `rgba()` is the unfused route (our hash-grid kernel + torch Linear); the tracer uses
`fused_spec()` to hand the whole field to the fused native pipeline instead.
"""
from __future__ import annotations

import inspect
from typing import Optional

import numpy as np
import torch
import torch.nn as nn

from . import ops, spc
from .accelstructs import OctreeAS
from .grids import OctreeGrid


class PositionalEmbedder(nn.Module):
    def __init__(self, num_freq, max_freq_log2, log_sampling=True, include_input=True, input_dim=3):
        super().__init__()
        self.num_freq, self.max_freq_log2, self.log_sampling, self.include_input = num_freq, max_freq_log2, log_sampling, include_input
        self.out_dim = input_dim if include_input else 0
        if log_sampling:
            bands = 2.0 ** torch.linspace(0.0, max_freq_log2, steps=num_freq)
        else:
            bands = torch.linspace(1, 2.0 ** max_freq_log2, steps=num_freq)
        self.out_dim += bands.shape[0] * input_dim * 2
        self.bands = nn.Parameter(bands).requires_grad_(False)

    def forward(self, coords):
        N = coords.shape[0]
        winded = (coords[:, None] * self.bands[None, :, None]).reshape(N, coords.shape[1] * self.num_freq)
        encoded = torch.cat([torch.sin(winded), torch.cos(winded)], dim=-1)
        if self.include_input:
            encoded = torch.cat([coords, encoded], dim=-1)
        return encoded


def get_positional_embedder(frequencies, input_dim=3, include_input=True):
    enc = PositionalEmbedder(frequencies, frequencies - 1, input_dim=input_dim, include_input=include_input)
    return enc, enc.out_dim


class BasicDecoder(nn.Module):
    """Linear/activation stack (basic_decoders.py:59-101); only layer=nn.Linear, activation=relu, no skips."""

    def __init__(self, input_dim, output_dim, activation=torch.relu, bias=True, layer=nn.Linear, num_layers=1, hidden_dim=128, skip=None):
        super().__init__()
        self.input_dim, self.output_dim, self.activation, self.bias = input_dim, output_dim, activation, bias
        self.layer, self.num_layers, self.hidden_dim, self.skip = layer, num_layers, hidden_dim, skip or []
        layers = []
        for i in range(num_layers):
            layers.append(layer(input_dim if i == 0 else hidden_dim, hidden_dim, bias=bias))
        self.layers = nn.ModuleList(layers)
        self.lout = layer(hidden_dim, output_dim, bias=bias)

    def forward(self, x, return_h=False):
        h = x
        for l in self.layers:
            h = self.activation(l(h))
        out = self.lout(h)
        return (out, h) if return_h else out

    def packed_params(self):
        """[W0, b0?, W1, b1?, ...] -- the order the C ABI expects (include/wispb200.h)."""
        return ops.decoder_params(self)

    def dims(self):
        return [self.input_dim] + [self.hidden_dim] * self.num_layers + [self.output_dim]


class BaseNeuralField(nn.Module):
    """Channel dispatch of base_nef.py:120-202."""

    def __init__(self):
        super().__init__()
        self._forward_functions = {}
        self.register_forward_functions()

    def _register_forward_function(self, fn, channels):
        if isinstance(channels, str):
            channels = [channels]
        self._forward_functions[fn] = set(channels)

    def get_supported_channels(self):
        out = set()
        for v in self._forward_functions.values():
            out |= v
        return out

    def forward(self, channels=None, **kwargs):
        if not (isinstance(channels, (str, list, set)) or channels is None):
            raise Exception(f"Channels type invalid, got {type(channels)}."
                            "Make sure your arguments for the nef are provided as keyword arguments.")
        requested = self.get_supported_channels() if channels is None else {channels} if isinstance(channels, str) else set(channels)
        unsupported = requested - self.get_supported_channels()
        if unsupported:
            raise Exception(f"Channels {unsupported} are not supported in {self.__class__.__name__}")
        fns = sorted(((len(ch & requested), fn) for fn, ch in self._forward_functions.items() if ch & requested), key=lambda x: x[0], reverse=True)
        ret = {}
        for _, fn in fns:
            supported = self._forward_functions[fn] & requested
            requested = requested - supported
            if supported:
                spec = inspect.getfullargspec(fn)
                nreq = len(spec.args) - (len(spec.defaults) if spec.defaults else 0)
                args = {}
                for a in spec.args[1:nreq]:
                    if a not in kwargs:
                        raise Exception(f"Argument {a} not found as input to in {self.__class__.__name__}.{fn.__name__}()")
                    args[a] = kwargs[a]
                for a in spec.args[nreq:]:
                    if a in kwargs:
                        args[a] = kwargs[a]
                out = fn(**args)
                for c in supported:
                    ret[c] = out[c]
        if isinstance(channels, str):
            return ret.get(channels)
        if isinstance(channels, list):
            return [ret[c] for c in channels]
        return ret


def sample_unif_sphere(n):
    """Uniformly random points on the unit sphere, np.array [n, 3] (wisp/ops/geometric.py:25-39)."""
    u = np.random.rand(2, n)
    z = 1 - 2 * u[0, :]
    r = np.sqrt(1. - z * z)
    phi = 2 * np.pi * u[1, :]
    return np.array([r * np.cos(phi), r * np.sin(phi), z]).transpose()


class NeuralRadianceField(BaseNeuralField):
    def __init__(self, grid, pos_embedder='none', view_embedder='none', pos_multires=10, view_multires=4, position_input=False,
                 activation_type='relu', layer_type='linear', hidden_dim=128, num_layers=1, bias=False,
                 prune_density_decay: Optional[float] = (0.01 * 512) / np.sqrt(3), prune_min_density: Optional[float] = 0.6):
        super().__init__()
        self.grid = grid
        if activation_type != 'relu' or layer_type not in ('linear', 'none'):
            raise NotImplementedError("wisp_b200 covers activation_type='relu', layer_type='linear' (the shipped NeRF configs)")
        self.pos_embedder_type, self.view_embedder_type = pos_embedder, view_embedder
        self.pos_multires, self.view_multires, self.position_input = pos_multires, view_multires, position_input
        self.pos_embedder, self.pos_embed_dim = self.init_embedder(pos_embedder, pos_multires, include_input=position_input)
        self.view_embedder, self.view_embed_dim = self.init_embedder(view_embedder, view_multires, include_input=True)
        self.activation_type, self.layer_type, self.hidden_dim, self.num_layers, self.bias = activation_type, layer_type, hidden_dim, num_layers, bias
        self.decoder_density = BasicDecoder(self.density_net_input_dim(), 16, torch.relu, bias, nn.Linear, num_layers, hidden_dim)
        if self.decoder_density.lout.bias is not None:
            self.decoder_density.lout.bias.data[0] = 1.0                        # nerf.py:162-163
        self.decoder_color = BasicDecoder(self.color_net_input_dim(), 3, torch.relu, bias, nn.Linear, num_layers + 1, hidden_dim)
        self.prune_density_decay, self.prune_min_density = prune_density_decay, prune_min_density

    def init_embedder(self, embedder_type, frequencies=None, include_input=False):
        """nerf.py:110-141."""
        if embedder_type == 'none' and not include_input:
            return None, 0
        if embedder_type == 'identity' or (embedder_type == 'none' and include_input):
            return nn.Identity(), 3
        if embedder_type == 'positional':
            return get_positional_embedder(frequencies=frequencies, include_input=include_input)
        raise NotImplementedError(f'Unsupported embedder type for NeuralRadianceField: {embedder_type}')

    def prune(self, jitter=None, seed=None):
        """Prunes the blas based on the current state (nerf.py:175-212): decay the running occupancy, probe the density at one
        jittered point per finest-level cell, keep the cells above `prune_min_density`, rebuild the occupancy structure from them.
        All of it runs on the native path (ops.prune_field: probe points, fused gather + decoders, occupancy update); the next
        raymarch rebuilds the native bit masks (ops.octree_tensors).  `jitter` ([cells, 3] in [0,1)) replays a given draw; `seed`
        selects the counter-based stream (default: the prune-call count, identical on all ranks)."""
        if self.prune_density_decay is None or self.prune_min_density is None or self.grid is None:
            return
        if not hasattr(self.grid, "occupancy") or not hasattr(self.grid, "dense_points"):
            raise NotImplementedError(f'Pruning not implemented for grid type {self.grid.__class__.__name__}')
        if not ops.prune_field(self, jitter=jitter, seed=seed):
            raise NotImplementedError("prune(): this field configuration is outside the native path (ops.nef_spec)")

    def register_forward_functions(self):
        self._register_forward_function(self.rgba, ["density", "rgb"])

    def rgba(self, coords, ray_d, lod_idx=None):
        """nerf.py:219-264, unfused: hash-grid kernel + torch decoders."""
        if lod_idx is None:
            lod_idx = len(self.grid.active_lods) - 1
        batch, _ = coords.shape
        feats = self.grid.interpolate(coords, lod_idx).reshape(batch, self.effective_feature_dim())
        if self.pos_embedder is not None:
            feats = torch.cat([feats, self.pos_embedder(coords).view(batch, self.pos_embed_dim)], dim=-1)
        density_feats = self.decoder_density(feats)
        if self.view_embedder is not None:
            fdir = torch.cat([density_feats, self.view_embedder(ray_d).view(batch, self.view_embed_dim)], dim=-1)
        else:
            fdir = density_feats
        colors = torch.sigmoid(self.decoder_color(fdir[..., 1:]))
        density = torch.relu(density_feats[..., 0:1])
        return dict(rgb=colors, density=density)

    def effective_feature_dim(self):
        return self.grid.feature_dim * self.grid.num_lods if self.grid.multiscale_type == 'cat' else self.grid.feature_dim

    def density_net_input_dim(self):
        return self.effective_feature_dim() + self.pos_embed_dim

    def color_net_input_dim(self):
        return 15 + self.view_embed_dim

    # ---- fused path ----------------------------------------------------------------------------------------
    def fused_spec(self, lod_idx: Optional[int] = None) -> Optional[ops.NefSpec]:
        """Description of this field for wb_rf_* (ops.nef_spec); None when the configuration is outside the fused path."""
        return ops.nef_spec(self, lod_idx)


class NeuralSDF(BaseNeuralField):
    """wisp.models.nefs.NeuralSDF (neural_sdf.py:24-180): grid features (+ position) -> BasicDecoder(bias=True, output_dim=1)."""

    def __init__(self, grid, pos_embedder='none', pos_multires=10, position_input=True, activation_type='relu', layer_type='none',
                 hidden_dim=128, num_layers=1):
        super().__init__()
        self.grid = grid
        if activation_type != 'relu' or layer_type not in ('linear', 'none'):
            raise NotImplementedError("wisp_b200 covers activation_type='relu', layer_type='linear'/'none'")
        self.pos_multires, self.position_input = pos_multires, position_input
        self.pos_embedder, self.pos_embed_dim = self.init_embedder(pos_embedder, pos_multires, position_input)
        self.activation_type, self.layer_type, self.hidden_dim, self.num_layers = activation_type, layer_type, hidden_dim, num_layers
        self.decoder = BasicDecoder(self.decoder_input_dim(), 1, torch.relu, True, nn.Linear, num_layers, hidden_dim)

    def init_embedder(self, embedder_type, frequencies=None, position_input=True):
        """neural_sdf.py:86-99."""
        if embedder_type == 'none' and not position_input:
            return None, 0
        if embedder_type == 'identity' or (embedder_type == 'none' and position_input):
            return nn.Identity(), 3
        if embedder_type == 'positional':
            return get_positional_embedder(frequencies=frequencies, include_input=position_input)
        raise NotImplementedError(f'Unsupported embedder type for NeuralSDF: {embedder_type}')

    def register_forward_functions(self):
        self._register_forward_function(self.sdf, ["sdf"])

    def get_forward_function(self, channel):
        fn = next(f for f, ch in self._forward_functions.items() if channel in ch)
        return lambda coords, lod_idx=None: fn(coords, lod_idx)[channel]

    def sdf(self, coords, lod_idx=None):
        """neural_sdf.py:120-155.  Without autograd (the sphere tracer, the SDF slices of the trainer's validation) the whole
        evaluation -- octree descent, trilinear blend of every LOD, position input, decoder -- is one native launch (wb_sdf_eval);
        with autograd it is the native grid kernel + torch decoder."""
        shape = coords.shape
        if shape[0] == 0:
            return dict(sdf=torch.zeros_like(coords)[..., 0:1])
        if lod_idx is None:
            lod_idx = self.grid.num_lods - 1
        fused = ops.sdf_channel(self, coords, lod_idx)
        if fused is not None:
            return fused
        if len(shape) == 2:
            coords = coords[:, None]
        num_samples = coords.shape[1]
        feats = self.grid.interpolate(coords, lod_idx)
        if self.pos_embedder is not None:
            feats = torch.cat([self.pos_embedder(coords.reshape(-1, 3)).view(-1, num_samples, self.pos_embed_dim), feats], dim=-1)
        sdf = self.decoder(feats)
        if len(shape) == 2:
            sdf = sdf[:, 0]
        return dict(sdf=sdf)

    def effective_feature_dim(self):
        return self.grid.feature_dim * self.grid.num_lods if self.grid.multiscale_type == 'cat' else self.grid.feature_dim

    def decoder_input_dim(self):
        return self.effective_feature_dim() + self.pos_embed_dim


class ImageNeuralField(BaseNeuralField):
    """wisp.models.nefs.ImageNeuralField (image_nef.py:37-97): grid features (FIRST) + a 3-band positional embedding of the [N, 2]
    pixel coordinates -> BasicDecoder(bias=True, 3 outputs) -> sigmoid.  Parameter names are the reference's (grid.codebook.feats,
    decoder.layers.0.weight, decoder.lout.bias, embedder.bands)."""

    def __init__(self, grid, activation_type='relu', layer_type='none', hidden_dim=128, num_layers=1):
        super().__init__()
        self.grid = grid
        if activation_type != 'relu' or layer_type not in ('linear', 'none'):
            raise NotImplementedError("wisp_b200 covers activation_type='relu', layer_type='linear'/'none'")
        self.activation_type, self.layer_type, self.hidden_dim, self.num_layers = activation_type, layer_type, hidden_dim, num_layers
        self.feature_dim = grid.feature_dim * len(grid.resolutions) if grid.multiscale_type == 'cat' else grid.feature_dim
        self.embedder, self.embed_dim = get_positional_embedder(frequencies=3, include_input=True)
        self.embed_dim = 14                       # image_nef.py:63: the embedder's out_dim says 21 (input_dim=3), 2-D input gives 14
        self.input_dim = self.feature_dim + self.embed_dim
        self.decoder = BasicDecoder(self.input_dim, 3, torch.relu, True, nn.Linear, num_layers, hidden_dim)

    def register_forward_functions(self):
        self._register_forward_function(self.rgb, ["rgb"])

    def rgb(self, coords, lod=None):
        """image_nef.py:77-97.  Without autograd or autocast (the trainer's validate() and render_final_view) the whole evaluation --
        2-D hash-grid gather of every LOD, embedding, decoder, sigmoid -- is one native launch (wb_image_eval); otherwise the native
        grid kernel + torch embedding and decoder."""
        fused = ops.image_rgb(self, coords, lod)
        if fused is not None:
            return fused
        if lod is None:
            lod = len(self.grid.resolutions) - 1
        batch, _ = coords.shape
        feats = self.grid.interpolate(coords, lod).reshape(-1, self.feature_dim)
        embedded_pos = self.embedder(coords).view(batch, self.embed_dim)
        fpos = torch.cat([feats, embedded_pos], dim=-1)
        return torch.sigmoid(self.decoder(fpos))


class SPCField(BaseNeuralField):
    """wisp.models.nefs.SPCField (spc_field.py:19-157): an SPC rendered with its own per-point colours, no embedder or decoder.
    PackedSPCTracer renders it in one launch (ops.spc_trace) from the f32 [M, 3] rows of ops.spc_colors."""

    def __init__(self, spc_octree: torch.Tensor, features_dict=None, device='cuda'):
        super().__init__()
        self.spc_octree = spc_octree
        self.features_dict = features_dict if features_dict is not None else dict()
        self.spc_device = device
        self.grid = None
        self.colors = None
        self.normals = None
        self.init_grid(spc_octree)

    def init_grid(self, spc_octree: torch.Tensor):
        """spc_field.py:69-114: RGBA colours / 255, else 0.5 * (normals + 1), else the finest level's point coordinates / 2^level
        (each with the reference's dtype promotion)."""
        if "colors" in self.features_dict:
            self.colors = self.features_dict["colors"].reshape(-1, 4) / 255.0
        if "normals" in self.features_dict:
            self.normals = self.features_dict["normals"].reshape(-1, 3)
        if self.colors is None:
            if self.normals is not None:
                colors = 0.5 * (self.normals + 1.0)
            else:
                level, pyramid, _ = spc.scan_octree(spc_octree)
                colors = spc.generate_points(spc_octree, pyramid)[int(pyramid[1, level]):]
                colors = colors / np.power(2, level)
            self.colors = colors
        self.grid = OctreeGrid(OctreeAS(spc_octree), feature_dim=3, num_lods=0)

    @property
    def device(self):
        return self.spc_device

    def register_forward_functions(self):
        self._register_forward_function(self.rgba, ["rgb"])

    def rgba(self, ridx_hit=None):
        """spc_field.py:130-147: colours of point-hierarchy indices, made relative to the finest level -> rgb [batch, 1, 3]."""
        level = self.grid.blas.max_level
        offset = self.grid.blas.pyramid[1, level]
        return dict(rgb=self.colors[ridx_hit - offset, :3].unsqueeze(1))
