"""Ray generation on the device: wisp.ops.raygen.generate_pinhole_rays (wisp/ops/raygen/raygen.py:40-85) and the offline
renderer's _look_at (wisp/trainers/tracker/offline_renderer.py:23-89) as single kernels (csrc/wb_raygen.cu).  A render call then
ships a camera (64 bytes) instead of 24 bytes per ray."""
from __future__ import annotations

import ctypes as C
import math

import numpy as np
import torch

from . import _cabi as A
from .core import Rays


def _unit(v):
    n = float(np.linalg.norm(v))
    return (v / max(n, 1e-12)).astype(np.float32)


def look_at_rays(f, t, height: int, width: int, mode: str = 'persp', fov: float = 90.0, device="cuda", dist_min: float = 0.0, dist_max: float = 6.0) -> Rays:
    """_look_at(f, t, height, width, mode, fov) -> Rays with origins / dirs [height*width, 3] on `device`.
    The 3-vector camera frame (view, right, up: offline_renderer.py:43-46) is computed on the host in fp32, the per-pixel work natively."""
    if mode not in ('persp', 'ortho'):
        raise ValueError('Invalid camera mode!')                                            # offline_renderer.py:86
    fo, to = np.asarray(f, np.float32), np.asarray(t, np.float32)
    view = _unit(to - fo)
    right = _unit(np.cross(view, np.array([0, 1, 0], np.float32)).astype(np.float32))
    up = _unit(np.cross(right, view).astype(np.float32))
    dev = torch.device(device)
    origins = torch.empty((height * width, 3), dtype=torch.float32, device=dev)
    dirs = torch.empty_like(origins)
    A.require_device(origins)
    v3 = lambda a: (C.c_float * 3)(*[float(x) for x in a])
    with torch.cuda.device(dev):
        A.lib().wb_raygen_lookat(v3(fo), v3(view), v3(right), v3(up), float(np.float32(np.tan(np.radians(fov / 2)))),
                                 height, width, 1 if mode == 'ortho' else 0, A.ptr(origins), A.ptr(dirs), A.stream())
    return Rays(origins, dirs, dist_min=dist_min, dist_max=dist_max)


def pinhole_rays(cam_pos, cam_to_world_rot, fov_h_deg: float, img_height: int, img_width: int, res_y: int = None, res_x: int = None,
                 x0: float = 0.0, y0: float = 0.0, near: float = 0.0, far: float = 6.0, device="cuda") -> Rays:
    """generate_pinhole_rays(camera, generate_centered_pixel_coords(img_width, img_height, res_x, res_y)) for a pinhole camera given by its
    world position, camera-to-world rotation (3x3), horizontal field of view, principal point and clipping planes."""
    res_x, res_y = res_x or img_width, res_y or img_height
    tanh = math.tan(math.radians(fov_h_deg) / 2.0)
    tanv = tanh * img_height / img_width
    dev = torch.device(device)
    origins = torch.empty((res_y * res_x, 3), dtype=torch.float32, device=dev)
    dirs = torch.empty_like(origins)
    A.require_device(origins)
    Rm = np.asarray(cam_to_world_rot, np.float32).reshape(9)
    with torch.cuda.device(dev):
        A.lib().wb_raygen_pinhole((C.c_float * 3)(*[float(x) for x in cam_pos]), (C.c_float * 9)(*[float(x) for x in Rm]), x0, y0,
                                  tanh, tanv, img_height, img_width, res_y, res_x, A.ptr(origins), A.ptr(dirs), A.stream())
    return Rays(origins, dirs, dist_min=near, dist_max=far)
