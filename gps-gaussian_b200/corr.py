"""Mirror of reference core/corr.py:17-61 for the `reg_cuda` path selected at core/raft_stereo_human.py:84-89:
`CorrSampler` (autograd.Function over `corr_sampler.forward/backward`) and `CorrBlockFast1D(fmap1, fmap2,
num_levels=4, radius=4)` with `__call__(coords[B,2,H,W]) -> [B, num_levels*(2r+1), H, W]`.

Same names, ctor kwargs and results; the work is done by sm_90a kernels:
  * ctor: ONE fused launch builds the all-pairs volume, applies 1/sqrt(D) and pools the whole pyramid
    (reference: batched GEMM + divide + 3 avg_pool2d + reshape copies);
  * call: ONE fused launch looks up all levels and writes the concatenated [B,36,H,W] tensor
    (reference: 4 sampler launches + torch.cat); its backward is one launch as well.
"""
import ctypes as C
import math
import os
import sys

import torch

_DROPIN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "dropin")
if _DROPIN not in sys.path:
    sys.path.insert(0, _DROPIN)
import corr_sampler  # noqa: E402
from . import _lib  # noqa: E402

_DT = {torch.float32: 0, torch.float16: 1}


def _dev(t):
    return t.device.index if t.device.index is not None else torch.cuda.current_device()


def _stream(t):
    return C.c_void_p(torch.cuda.current_stream(t.device).cuda_stream)


class CorrSampler(torch.autograd.Function):
    """Per-level sampler, exactly the reference class (core/corr.py:17-29)."""

    @staticmethod
    def forward(ctx, volume, coords, radius):
        ctx.save_for_backward(volume, coords)
        ctx.radius = radius
        corr, = corr_sampler.forward(volume, coords, radius)
        return corr

    @staticmethod
    def backward(ctx, grad_output):
        volume, coords = ctx.saved_tensors
        grad_volume, = corr_sampler.backward(volume, coords, grad_output.contiguous(), ctx.radius)
        return grad_volume, None, None


class _BuildPyramid(torch.autograd.Function):
    """(fmap1, fmap2) -> tuple of `levels` volumes [B,H,W1,W2>>l]  (core/corr.py:31-42,53-61 fused)."""

    @staticmethod
    def forward(ctx, fmap1, fmap2, levels):
        if fmap1.dtype not in _DT or fmap2.dtype != fmap1.dtype or not fmap1.is_cuda:
            raise RuntimeError("CorrBlockFast1D (gpsg): fmaps must be CUDA fp16/fp32 tensors of one dtype")
        f1, f2 = fmap1.detach().contiguous(), fmap2.detach().contiguous()
        B, D, H, W1 = f1.shape
        W2 = f2.shape[3]
        # one allocation for the whole pyramid (each level starts on a 16-byte boundary), carved into per-level views
        sizes = [B * H * W1 * (W2 >> l) for l in range(levels)]
        offs = [0]
        for n in sizes[:-1]:
            offs.append(offs[-1] + ((n + 7) & ~7))
        buf = torch.empty(offs[-1] + sizes[-1], dtype=f1.dtype, device=f1.device)
        vols = [buf[o:o + n].view(B, H, W1, W2 >> l) for l, (o, n) in enumerate(zip(offs, sizes))]
        ptrs = (C.c_void_p * 4)(*[v.data_ptr() if v.numel() else None for v in vols] + [None] * (4 - levels))
        with torch.cuda.device(f1.device):
            rc = _lib.lib.gpsg_corr_build_pyramid(_dev(f1), _stream(f1), _DT[f1.dtype], B, D, H, W1, W2,
                                                  C.c_void_p(f1.data_ptr()), C.c_void_p(f2.data_ptr()), ptrs, levels)
        _lib.check(rc, "gpsg_corr_build_pyramid")
        ctx.save_for_backward(f1, f2)
        ctx.levels = levels
        return tuple(vols)

    @staticmethod
    def backward(ctx, *grads):
        # Chain of avg_pool2d([1,2]) folded back to level 0 (cheap elementwise torch ops), then the two contractions
        # dF1 = F2 g^T, dF2 = F1 g in one sm_90a kernel each (gpsg_corr_build_backward).
        f1, f2 = ctx.saved_tensors
        B, D, H, W1 = f1.shape
        W2 = f2.shape[3]
        g = None                                      # gradient w.r.t. the level currently being folded
        for l in range(ctx.levels - 1, -1, -1):
            gl = grads[l]
            if g is not None:                         # g = d/d(level l+1): each of its elements averaged two of level l
                up = torch.zeros((B, H, W1, W2 >> l), dtype=g.dtype, device=g.device)
                up[..., :2 * g.shape[-1]] = (0.5 * g).repeat_interleave(2, dim=-1)
                g = up if gl is None else gl + up
            else:
                g = gl
        if g is None:
            return None, None, None
        g = g.to(f1.dtype).contiguous()
        d1, d2 = torch.empty_like(f1), torch.empty_like(f2)
        with torch.cuda.device(f1.device):
            rc = _lib.lib.gpsg_corr_build_backward(_dev(f1), _stream(f1), _DT[f1.dtype], B, D, H, W1, W2,
                                                   C.c_void_p(f1.data_ptr()), C.c_void_p(f2.data_ptr()),
                                                   C.c_void_p(g.data_ptr()), C.c_void_p(d1.data_ptr()),
                                                   C.c_void_p(d2.data_ptr()))
        _lib.check(rc, "gpsg_corr_build_backward")
        return d1, d2, None


class _LookupPyramid(torch.autograd.Function):
    """(coords_x[B,1,H,W1], radius, *vols) -> [B, levels*(2r+1), H, W1]  (core/corr.py:44-51 fused)."""

    @staticmethod
    def forward(ctx, coords, radius, *vols):
        v0 = vols[0]
        B, H, W1, _ = v0.shape
        L = len(vols)
        vs = [v.detach().contiguous() for v in vols]
        c = coords.detach()
        if c.dtype != torch.float32 or c.stride(3) != 1 or c.stride(2) != c.shape[3]:
            c = c[:, :1].to(torch.float32).contiguous()
        out = torch.empty((B, L * (2 * radius + 1), H, W1), dtype=v0.dtype, device=v0.device)
        ptrs = (C.c_void_p * 4)(*[v.data_ptr() if v.numel() else None for v in vs] + [None] * (4 - L))
        widths = (C.c_int32 * 4)(*[int(v.shape[3]) for v in vs] + [0] * (4 - L))
        with torch.cuda.device(v0.device):
            rc = _lib.lib.gpsg_corr_lookup_pyramid_forward(_dev(v0), _stream(v0), _DT[v0.dtype], B, H, W1, ptrs, widths, L,
                                                           C.c_void_p(c.data_ptr()), int(c.stride(0)), int(radius),
                                                           C.c_void_p(out.data_ptr()))
        _lib.check(rc, "gpsg_corr_lookup_pyramid_forward")
        ctx.save_for_backward(c)
        ctx.meta = (radius, [tuple(v.shape) for v in vs], v0.dtype)
        return out

    @staticmethod
    def backward(ctx, grad_out):
        c, = ctx.saved_tensors
        radius, shapes, dtype = ctx.meta
        L = len(shapes)
        B, H, W1, _ = shapes[0]
        g = grad_out.detach().to(dtype).contiguous()
        gv = [torch.empty(s, dtype=dtype, device=g.device) for s in shapes]
        ptrs = (C.c_void_p * 4)(*[v.data_ptr() if v.numel() else None for v in gv] + [None] * (4 - L))
        widths = (C.c_int32 * 4)(*[int(s[3]) for s in shapes] + [0] * (4 - L))
        with torch.cuda.device(g.device):
            rc = _lib.lib.gpsg_corr_lookup_pyramid_backward(_dev(g), _stream(g), _DT[dtype], B, H, W1, ptrs, widths, L,
                                                            C.c_void_p(c.data_ptr()), int(c.stride(0)), int(radius),
                                                            C.c_void_p(g.data_ptr()))
        _lib.check(rc, "gpsg_corr_lookup_pyramid_backward")
        return (None, None) + tuple(gv)


class CorrBlockFast1D:
    def __init__(self, fmap1, fmap2, num_levels=4, radius=4):
        if num_levels > 4:
            raise ValueError("CorrBlockFast1D (gpsg): at most 4 pyramid levels")
        self.num_levels = num_levels
        self.radius = radius
        self._vols = _BuildPyramid.apply(fmap1, fmap2, num_levels)
        # same shapes as the reference's views: [B, H, W1, 1, W2 // 2**i]
        self.corr_pyramid = [v.unsqueeze(3) for v in self._vols]

    def __call__(self, coords):
        return _LookupPyramid.apply(coords[:, :1], self.radius, *self._vols)      # x channel as a view (reference copies it)

    @staticmethod
    def corr(fmap1, fmap2):
        """Level-0 volume [B,H,W1,1,W2] (reference CorrBlockFast1D.corr, core/corr.py:53-61)."""
        return _BuildPyramid.apply(fmap1, fmap2, 1)[0].unsqueeze(3)
