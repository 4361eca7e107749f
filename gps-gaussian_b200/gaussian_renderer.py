"""Mirror of reference gaussian_renderer/__init__.py:17-67 -- `render(data, idx, pts_xyz, pts_rgb,
rotations, scales, opacity, bg_color)` with the same argument meaning and return value
([3,H,W] image; radii dropped), wired to the sm_90a rasterizer.

Differences that are invisible to the caller: the zero `screenspace_points` tensor is only created
when a gradient is being recorded (it exists upstream solely so autograd can return a means2D
gradient), FoV/size scalars are read without forcing a device sync when they live on the host
(they do in training: reference train_stage2.py:155-157), the background colour stays on the host
(the kernels take it by value) and the autograd function is entered directly instead of through a
freshly constructed `nn.Module` per call.
"""
import math
import os
import sys

import torch

_DROPIN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "dropin")
if _DROPIN not in sys.path:
    sys.path.insert(0, _DROPIN)
import diff_gaussian_rasterization as _dgr  # noqa: E402

_NONE = torch.Tensor([])          # what GaussianRasterizer.forward substitutes for an absent optional argument


def _camera(nv, idx, bg_color):
    """The 12 rasterizer settings of gaussian_renderer/__init__.py:36-49 for novel view `idx`."""
    half_fov = (0.5 * float(nv['FovX'][idx]), 0.5 * float(nv['FovY'][idx]))
    return _dgr.GaussianRasterizationSettings(
        int(nv['height'][idx]), int(nv['width'][idx]), math.tan(half_fov[0]), math.tan(half_fov[1]),
        torch.as_tensor(bg_color, dtype=torch.float32), 1.0, nv['world_view_transform'][idx],
        nv['full_proj_transform'][idx], 3, nv['camera_center'][idx], False, False)


def _grad_sink(pts_xyz):
    """means2D: zeros; a leaf-like tensor with retained grad only when a gradient can flow (upstream's idiom)."""
    sink = torch.zeros_like(pts_xyz, dtype=torch.float32)
    if torch.is_grad_enabled() and pts_xyz.requires_grad:
        sink = sink.requires_grad_(True) + 0
        try:
            sink.retain_grad()
        except Exception:
            pass
    return sink


def render(data, idx, pts_xyz, pts_rgb, rotations, scales, opacity, bg_color):
    settings = _camera(data['novel_view'], idx, bg_color)
    # precomputed colours, scale/rotation pairs: the one combination GPS-Gaussian uses (:54-62)
    image, _radii = _dgr.rasterize_gaussians(pts_xyz, _grad_sink(pts_xyz), _NONE, pts_rgb, opacity, scales, rotations,
                                             _NONE, settings)
    return image
