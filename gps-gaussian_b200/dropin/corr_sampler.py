"""Drop-in `corr_sampler` for GPS-Gaussian, backed by libgpsg_sm90.so (sm_90a).

Put `gps-gaussian_b200/dropin` on PYTHONPATH and the UNMODIFIED reference imports this module at
core/corr.py:5-8 instead of princeton-vl/RAFT-Stereo's `sampler` extension (SURVEY.md Appendix B).

    forward(volume[B,H,W1,W2] fp16|fp32 CUDA, coords[B,C>=1,H,W1] fp32, radius) -> [corr[B,2r+1,H,W1]]
    backward(volume, coords, grad_output (contiguous), radius)                   -> [grad_volume]
(call sites: reference core/corr.py:22 and :28; both unpack a 1-element sequence.)
"""
import ctypes as C
import os
import sys

import torch

_REPO = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
if _REPO not in sys.path:
    sys.path.insert(0, _REPO)
from gps_gaussian_b200 import _lib  # noqa: E402  (raises if the CUDA library is not built)

_DT = {torch.float32: 0, torch.float16: 1}


def _check(volume, coords):
    if not volume.is_cuda:
        raise RuntimeError("corr_sampler (gpsg): volume must be a CUDA tensor")
    if volume.dtype not in _DT:
        raise RuntimeError(f"corr_sampler (gpsg): unsupported volume dtype {volume.dtype}")
    if volume.dim() != 4 or coords.dim() != 4:
        raise RuntimeError("corr_sampler (gpsg): volume must be [B,H,W1,W2] and coords [B,C,H,W1]")
    B, H, W1, _ = volume.shape
    if coords.shape[0] != B or coords.shape[2] != H or coords.shape[3] != W1:
        raise RuntimeError("corr_sampler (gpsg): coords shape does not match volume")


def _coords_x(coords):
    c = coords.detach()
    if c.dtype != torch.float32 or c.stride(3) != 1 or c.stride(2) != c.shape[3]:
        c = c[:, :1].to(torch.float32).contiguous()
    return c, int(c.stride(0))


def _dev_index(t):
    return t.device.index if t.device.index is not None else torch.cuda.current_device()


def forward(volume, coords, radius):
    _check(volume, coords)
    vol = volume.detach()
    if vol.stride(3) != 1:
        vol = vol.contiguous()
    B, H, W1, W2 = vol.shape
    c, csb = _coords_x(coords)
    out = torch.empty((B, 2 * int(radius) + 1, H, W1), dtype=vol.dtype, device=vol.device)
    with torch.cuda.device(vol.device):
        rc = _lib.lib.gpsg_corr_sampler_forward(
            _dev_index(vol), C.c_void_p(torch.cuda.current_stream(vol.device).cuda_stream), _DT[vol.dtype], B, H, W1, W2,
            C.c_void_p(vol.data_ptr()), vol.stride(0), vol.stride(1), vol.stride(2), C.c_void_p(c.data_ptr()), csb,
            int(radius), C.c_void_p(out.data_ptr()))
    _lib.check(rc, "gpsg_corr_sampler_forward")
    return [out]


def backward(volume, coords, grad_output, radius):
    _check(volume, coords)
    B, H, W1, W2 = volume.shape
    c, csb = _coords_x(coords)
    g = grad_output.detach().to(volume.dtype).contiguous()
    gvol = torch.empty((B, H, W1, W2), dtype=volume.dtype, device=volume.device)
    with torch.cuda.device(volume.device):
        rc = _lib.lib.gpsg_corr_sampler_backward(
            _dev_index(volume), C.c_void_p(torch.cuda.current_stream(volume.device).cuda_stream), _DT[volume.dtype],
            B, H, W1, W2, C.c_void_p(c.data_ptr()), csb, C.c_void_p(g.data_ptr()), int(radius),
            C.c_void_p(gvol.data_ptr()))
    _lib.check(rc, "gpsg_corr_sampler_backward")
    return [gvol]
