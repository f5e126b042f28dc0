"""ctypes binding of libwispb200.so -- the only place the host shim touches native code.

The C ABI (include/wispb200.h) takes raw device pointers, sizes and a cudaStream_t; PyTorch is used here only
as the owner of device memory and streams.  There is NO CPU or eager fallback: if the library is missing, or
the device is not sm_90, every compute entry point raises.
"""
from __future__ import annotations

import ctypes as C
import os
from typing import Optional, Sequence

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "lib", "libwispb200.so")

WB_MAX_LODS = 32
WB_MAX_LAYERS = 8


class NefDesc(C.Structure):
    """struct wb_nef_desc (include/wispb200.h)."""
    _fields_ = [
        ("num_lods", C.c_int32), ("feature_dim", C.c_int32), ("codebook_size", C.c_int32),
        ("multiscale", C.c_int32), ("lod_idx", C.c_int32),
        ("resolutions", C.c_int32 * WB_MAX_LODS),
        ("begin_idxes", C.c_int64 * (WB_MAX_LODS + 1)),
        ("table", C.c_void_p),
        ("pos_mode", C.c_int32), ("pos_freq", C.c_int32), ("view_mode", C.c_int32), ("view_freq", C.c_int32),
        ("has_bias", C.c_int32),
        ("dens_layers", C.c_int32), ("dens_dims", C.c_int32 * (WB_MAX_LAYERS + 1)),
        ("col_layers", C.c_int32), ("col_dims", C.c_int32 * (WB_MAX_LAYERS + 1)),
        ("dens_params", C.c_void_p), ("col_params", C.c_void_p),
        ("grid_kind", C.c_int32), ("base_lod", C.c_int32), ("half_round", C.c_int32),
        ("grid_ptrs", C.POINTER(C.c_void_p)), ("grid_grads", C.POINTER(C.c_void_p)),
        ("oct", C.c_void_p), ("points", C.c_void_p), ("trinkets", C.c_void_p),
        ("grid_layout", C.c_int32),
    ]


class RaysDesc(C.Structure):
    """struct wb_rays."""
    _fields_ = [("origins", C.c_void_p), ("dirs", C.c_void_p), ("num_rays", C.c_int64),
                ("dist_min", C.c_float), ("dist_max", C.c_float), ("near_v", C.c_void_p), ("far_v", C.c_void_p)]


class OctreeDesc(C.Structure):
    """struct wb_octree."""
    _fields_ = [("octree", C.c_void_p), ("prefix", C.c_void_p), ("nbytes", C.c_int64), ("max_level", C.c_int32),
                ("bits", C.c_void_p), ("bits_level", C.c_int32), ("has_bbox", C.c_int32),
                ("bbox_lo", C.c_float * 3), ("bbox_hi", C.c_float * 3),
                ("coarse_bits", C.c_void_p), ("coarse_level", C.c_int32)]


class SdfDesc(C.Structure):
    """struct wb_sdf_desc."""
    _fields_ = [("points", C.c_void_p), ("trinkets", C.c_void_p), ("feats", C.POINTER(C.c_void_p)),
                ("feature_dim", C.c_int32), ("base_lod", C.c_int32), ("num_lods", C.c_int32), ("multiscale", C.c_int32), ("half_round", C.c_int32),
                ("pos_mode", C.c_int32), ("pos_freq", C.c_int32), ("num_layers", C.c_int32), ("hidden_dim", C.c_int32), ("params", C.c_void_p),
                ("hash", C.POINTER(NefDesc))]


class SdfState(C.Structure):
    """struct wb_sdf_state."""
    _fields_ = [("flags", C.c_void_p), ("pack_off", C.c_void_p), ("scan_ws", C.c_void_p), ("scan_ws_bytes", C.c_int64), ("pack_ray", C.c_void_p),
                ("t", C.c_void_p), ("dist", C.c_void_p), ("dist_prev", C.c_void_p), ("x", C.c_void_p), ("cursor0", C.c_void_p), ("cursor1", C.c_void_p),
                ("state", C.c_void_p), ("iterflags", C.c_void_p)]


class AdamSegment(C.Structure):
    """struct wb_adam_segment."""
    _fields_ = [("param", C.c_void_p), ("grad", C.c_void_p), ("exp_avg", C.c_void_p), ("exp_avg_sq", C.c_void_p), ("numel", C.c_int64),
                ("lr", C.c_float), ("weight_decay", C.c_float)]


class RMSpropSegment(C.Structure):
    """struct wb_rmsprop_segment."""
    _fields_ = [("param", C.c_void_p), ("grad", C.c_void_p), ("square_avg", C.c_void_p), ("momentum_buffer", C.c_void_p), ("numel", C.c_int64),
                ("lr", C.c_float), ("weight_decay", C.c_float)]


# The C ABI's prototypes, in header order: name -> (restype, argtypes).  Data pointers (device or host) are c_void_p, host arrays of
# device pointers POINTER(c_void_p), descriptors a POINTER to their mirror above (ctypes then refuses a descriptor of another kind
# and takes the struct itself by reference).
_i32, _int, _i64, _u32, _f32, _f64 = C.c_int32, C.c_int, C.c_int64, C.c_uint32, C.c_float, C.c_double
_p, _pp = C.c_void_p, C.POINTER(C.c_void_p)
_nef, _rays, _oct, _sdf, _state, _adam, _rms = (C.POINTER(s) for s in (NefDesc, RaysDesc, OctreeDesc, SdfDesc, SdfState, AdamSegment, RMSpropSegment))
PROTOTYPES = {
    "wb_last_error": (C.c_char_p, []),
    "wb_version": (_int, []),
    "wb_device_check": (_int, [_int]),
    "wb_launch_count": (_i64, []),
    "wb_octree_build_bits": (_int, [_p, _i64, _i32, _p, _p]),
    "wb_octree_build_coarse": (_int, [_p, _i64, _i32, _i32, _p, _p]),
    "wb_query": (_int, [_oct, _p, _i64, _i32, _i32, _p, _p]),
    "wb_raymarch_ray_count": (_int, [_oct, _i32, _rays, _i32, _p, _u32, _p, _p, _p]),
    "wb_scan_workspace_bytes": (_i64, [_i64]),
    "wb_scan_counts": (_int, [_p, _i64, _p, _p, _i64, _p]),
    "wb_raymarch_ray_fill": (_int, [_rays, _i32, _p, _u32, _p, _p, _p, _p, _p, _p, _p, _p]),
    "wb_raytrace_count": (_int, [_oct, _i32, _rays, _p, _p]),
    "wb_raytrace_fill": (_int, [_oct, _i32, _rays, _p, _p, _p, _p, _p]),
    "wb_raytrace_cache_bytes": (_i64, [_i64, _i32]),
    "wb_raytrace_count_cached": (_int, [_oct, _i32, _rays, _p, _p, _i32, _p]),
    "wb_raytrace_fill_cached": (_int, [_oct, _i32, _rays, _p, _p, _i32, _p, _p, _p, _p]),
    "wb_raymarch_voxel_fill": (_int, [_rays, _p, _p, _i64, _i32, _p, _u32, _p, _p, _p, _p, _p, _p, _p]),
    "wb_raymarch_uniform_count": (_int, [_p, _i64, _i32, _p, _p]),
    "wb_raymarch_uniform_fill": (_int, [_rays, _p, _p, _i64, _i32, _p, _p, _p, _p, _p, _p, _p, _p, _p]),
    "wb_hashgrid_fwd": (_int, [_p, _i64, _nef, _p, _p]),
    "wb_hashgrid_bwd": (_int, [_p, _i64, _nef, _p, _p, _p]),
    "wb_triplane_fwd": (_int, [_p, _i64, _i32, _i32, _p, _pp, _p, _p]),
    "wb_triplane_bwd": (_int, [_p, _i64, _i32, _i32, _p, _pp, _p, _pp, _p]),
    "wb_triplane_relayout": (_int, [_pp, _pp, _p, _i32, _i32, _i32, _p]),
    "wb_octree_interp_fwd": (_int, [_oct, _p, _p, _p, _i64, _i32, _i32, _i32, _i32, _i32, _pp, _p, _p]),
    "wb_octree_interp_bwd": (_int, [_oct, _p, _p, _p, _i64, _i32, _i32, _i32, _i32, _pp, _p, _pp, _p]),
    "wb_find_depth_bound": (_int, [_p, _p, _p, _i64, _i64, _p, _p]),
    "wb_sdf_eval": (_int, [_oct, _sdf, _i32, _p, _i64, _p, _p]),
    "wb_sdf_train": (_int, [_oct, _sdf, _i32, _p, _p, _i64, _f32, _pp, _p, _p, _p]),
    "wb_sdf_train_smem_bytes": (_i64, [_sdf]),
    "wb_sdf_train_tc": (_int, [_oct, _sdf, _i32, _p, _p, _i64, _f32, _pp, _p, _p, _p]),
    "wb_sdf_train_tc_smem_bytes": (_i64, [_sdf]),
    "wb_sdf_trace": (_int, [_oct, _sdf, _i32, _rays, _p, _i64, _p, _i32, _f32, _f64, _i32, _state, _p, _p, _p, _p, _p, _p, _p]),
    "wb_sdf_phase": (_int, [_i32, _rays, _p, _i64, _p, _i32, _i32, _f64, _state, _p, _p, _p, _p, _p]),
    "wb_composite_fwd": (_int, [_p, _p, _p, _p, _i64, _p, _p, _p, _p, _p, _p]),
    "wb_composite_bwd": (_int, [_p, _p, _p, _p, _i64, _p, _p, _p, _p, _p, _p, _p]),
    "wb_rf_march_fill": (_int, [_rays, _i32, _p, _u32, _p, _p, _p, _p, _p, _p]),
    "wb_rf_param_blob_floats": (_i64, [_nef, _i32]),
    "wb_rf_precision_supported": (_int, [_nef, _i32, _i32]),
    "wb_rf_tc_shaped": (_int, [_nef, _i32, _p]),
    "wb_rf_pack_params": (_int, [_nef, _i32, _p, _p]),
    "wb_rf_workspace_bytes": (_i64, [_nef, _i32, _i64, _i64, _i32]),
    "wb_rf_feat_bytes": (_i64, [_nef, _i32, _i64]),
    "wb_rf_shade_fwd": (_int, [_nef, _p, _i32, _rays, _p, _p, _i64, _p, _p, _p, _p]),
    "wb_rf_shade_bwd": (_int, [_nef, _p, _i32, _rays, _p, _p, _i64, _p, _p, _p, _p, _p, _p, _p, _p]),
    "wb_rf_workspace_holds_ray_rows": (_int, [_i32]),
    "wb_rf_loss_scale": (_int, [_p, _p, _p]),
    "wb_rf_decoder_bwd": (_int, [_nef, _p, _rays, _p, _p, _i64, _p, _p, _p, _p, _p, _p, _p]),
    "wb_rf_table_scatter": (_int, [_nef, _rays, _p, _p, _i64, _p, _p, _p, _p]),
    "wb_codebook_rows_fwd": (_int, [_p, _p, _i64, _i32, _i32, _i32, _p, _p, _p]),
    "wb_codebook_rows_bwd": (_int, [_p, _p, _p, _i64, _i32, _i32, _p, _p, _p]),
    "wb_composite_bwd_loss": (_int, [_p, _p, _p, _p, _i64, _p, _p, _p, _i32, _f32, _p, _p, _p, _p]),
    "wb_adam_step": (_int, [_adam, _i32, _f32, _f32, _f32, _i32, _f32, _i32, _p]),
    "wb_adamw_step": (_int, [_adam, _i32, _f32, _f32, _f32, _i32, _f32, _i32, _p]),
    "wb_rmsprop_step": (_int, [_rms, _i32, _f32, _f32, _f32, _f32, _i32, _p]),
    "wb_raygen_lookat": (_int, [_p, _p, _p, _p, _f32, _i32, _i32, _i32, _p, _p, _p]),
    "wb_raygen_pinhole": (_int, [_p, _p, _f32, _f32, _f32, _f32, _i32, _i32, _i32, _i32, _p, _p, _p]),
    "wb_prune_samples": (_int, [_p, _i64, _i32, _p, _u32, _p, _p, _p, _p, _p]),
    "wb_prune_update": (_int, [_p, _i64, _f32, _f32, _p, _p, _p]),
    "wb_tc_selftest": (_int, [_p, _int, _p, _int, _p, _int, _int, _int, _p]),
    "wb_hashgrid2d_fwd": (_int, [_p, _i64, _nef, _p, _p]),
    "wb_hashgrid2d_bwd": (_int, [_p, _i64, _nef, _p, _p, _p]),
    "wb_image_eval": (_int, [_nef, _i32, _pp, _i32, _p, _i64, _p, _p]),
    "wb_image_train": (_int, [_nef, _i32, _pp, _i32, _p, _p, _i64, _f32, _p, _p, _p, _p]),
    "wb_image_smem_bytes": (_i64, [_nef, _i32, _i32]),
    "wb_spc_trace": (_int, [_oct, _i32, _rays, _p, _i64, _i64, _p, _p, _p, _p, _p]),
    "wb_mesh_sdf_workspace_bytes": (_i64, [_i64]),
    "wb_mesh_sdf": (_int, [_p, _i64, _p, _i64, _p, _i64, _p, _p]),
    "wb_mesh_octree_bits": (_int, [_p, _p, _i64, _i64, _i32, _u32, _p, _p]),
}
EXPORTS = list(PROTOTYPES)
# int results that are answers, not a wb_status; every other int result raises WispB200Error when nonzero
NOT_STATUS = ("wb_version", "wb_rf_precision_supported")

_lib: Optional[C.CDLL] = None
_checked_devices = set()


class WispB200Error(RuntimeError):
    """status: the wb_status a library call returned, or None for an error raised on the host side."""

    def __init__(self, message: str, status: Optional[int] = None):
        super().__init__(message)
        self.status = status


def check(rc: int) -> None:
    """Raise WispB200Error for a nonzero wb_status.  The status entry points already raise through their errcheck, so a successful
    call's result passes through: callers written as check(lib().wb_...(...)) keep working."""
    if rc != 0:
        raise WispB200Error(f"libwispb200 error {rc}: {lib().wb_last_error().decode()}", status=rc)


def _raise_on_status(rc: int, func, args) -> int:
    """errcheck of the wb_status entry points: wb_last_error() is read on the calling thread, right after the failed call."""
    check(rc)
    return rc


def lib() -> C.CDLL:
    """Load libwispb200.so; raise loudly if it was not built (no fallback path exists)."""
    global _lib
    if _lib is None:
        global LIB_PATH
        LIB_PATH = os.environ.get("WISPB200_LIB", LIB_PATH)          # debug builds (build.py with WB_LIB_NAME) live beside the product library
        if not os.path.exists(LIB_PATH):
            raise WispB200Error(
                f"{LIB_PATH} not found: build it with `python kaolin-wisp_b200/build.py` (or __graft_entry__.build()). "
                "wisp_b200 has no CPU/eager fallback.")
        L = C.CDLL(LIB_PATH)
        for name, (restype, argtypes) in PROTOTYPES.items():
            fn = getattr(L, name)
            fn.restype, fn.argtypes = restype, argtypes
            if restype is _int and name not in NOT_STATUS:
                fn.errcheck = _raise_on_status
        _lib = L
    return _lib


def require_device(t: torch.Tensor) -> None:
    """Every compute call requires a CUDA tensor on an sm_90 device."""
    if not t.is_cuda:
        raise WispB200Error("wisp_b200 kernels need CUDA tensors on an H100 (sm_90a); there is no CPU fallback")
    idx = t.device.index if t.device.index is not None else torch.cuda.current_device()
    if idx != torch.cuda.current_device():
        raise WispB200Error(f"tensor on cuda:{idx} but the current device is cuda:{torch.cuda.current_device()}: call under torch.cuda.device({idx}) "
                            "(the library launches on the current device; one process per GPU is the supported layout)")
    if idx not in _checked_devices:
        lib().wb_device_check(idx)
        _checked_devices.add(idx)


def launch_count() -> int:
    return int(lib().wb_launch_count())


def ptr(t: Optional[torch.Tensor]):
    if t is None:
        return None
    return C.c_void_p(t.data_ptr())


def stream(t: Optional[torch.Tensor] = None) -> C.c_void_p:
    """The current torch stream (of `t`'s device when given).  The library launches on the CURRENT CUDA device: one process per GPU
    (torchrun + torch.cuda.set_device) is the supported layout; tensors on another device must be used under torch.cuda.device(...)."""
    return C.c_void_p((torch.cuda.current_stream(t.device) if t is not None else torch.cuda.current_stream()).cuda_stream)


def f32c(t: torch.Tensor) -> torch.Tensor:
    if t.dtype != torch.float32:
        t = t.float()
    return t.contiguous()


def _per_ray(v, R: int, device) -> torch.Tensor:
    t = torch.as_tensor(v, dtype=torch.float32, device=device).reshape(-1)
    if t.numel() == 1:
        t = t.expand(R)
    if t.numel() != R:
        raise WispB200Error(f"per-ray dist_min/dist_max must have {R} entries, got {t.numel()}")
    return t.contiguous()


def make_rays(origins: torch.Tensor, dirs: torch.Tensor, dist_min, dist_max):
    """-> (RaysDesc, keepalive).  dist_min/dist_max: python floats or per-ray tensors (wisp/core/rays.py:31-35)."""
    o, d = f32c(origins), f32c(dirs)
    keep = [o, d]
    r = RaysDesc()
    r.origins, r.dirs, r.num_rays = o.data_ptr(), d.data_ptr(), o.shape[0]
    if torch.is_tensor(dist_min) or torch.is_tensor(dist_max):
        nv, fv = _per_ray(dist_min, o.shape[0], o.device), _per_ray(dist_max, o.shape[0], o.device)
        keep += [nv, fv]
        r.near_v, r.far_v, r.dist_min, r.dist_max = nv.data_ptr(), fv.data_ptr(), 0.0, 0.0
    else:
        r.near_v, r.far_v = None, None
        r.dist_min, r.dist_max = float(dist_min), float(dist_max)
    return r, keep


def make_grid_desc(table: torch.Tensor, resolutions: Sequence[int], begin_idxes: Sequence[int], codebook_size: int,
                   multiscale: str = "cat", lod_idx: Optional[int] = None) -> NefDesc:
    d = NefDesc()
    L = len(resolutions)
    if L > WB_MAX_LODS:
        raise WispB200Error(f"num_lods {L} > {WB_MAX_LODS}")
    d.num_lods, d.feature_dim, d.codebook_size = L, table.shape[1], int(codebook_size)
    d.multiscale = 0 if multiscale == "cat" else 1
    d.lod_idx = L - 1 if lod_idx is None else int(lod_idx)
    for i, r in enumerate(resolutions):
        d.resolutions[i] = int(r)
    for i, b in enumerate(begin_idxes):
        d.begin_idxes[i] = int(b)
    d.table = table.data_ptr()
    return d
