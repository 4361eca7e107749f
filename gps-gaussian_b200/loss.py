"""Mirror of the photometric part of reference lib/loss.py:35-72 and its use at train_stage2.py:70-72, on sm_90a.

`l1_loss(network_output, gt)`, `ssim(img1, img2, window_size=11, size_average=True)` keep the reference signatures;
`fused_l1_ssim(img, gt, w_l1=0.8, w_ssim=0.2)` is the whole expression `0.8*Ll1 + 0.2*(1 - ssim)` in one forward and one
backward launch (`gpsg_l1_ssim_forward/backward`, csrc/loss.cu) instead of 5 depthwise 11x11 convolutions + ~15 elementwise
kernels and their autograd mirror.  The returned loss carries `.l1` and `.ssim` (detached 0-dim tensors) for the logging the
reference does (train_stage2.py:76-80).  No CPU fallback: CUDA tensors only.
"""
import ctypes as C

import torch

from . import _lib


def _p(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


def _check_inputs(img, gt):
    if not (img.is_cuda and gt.is_cuda):
        raise RuntimeError("gpsg loss: CUDA tensors required (no CPU fallback)")
    if img.shape != gt.shape or img.dim() < 2:
        raise RuntimeError(f"gpsg loss: shape mismatch {tuple(img.shape)} vs {tuple(gt.shape)}")


class _L1SSIM(torch.autograd.Function):
    """(img, gt, w_l1, w_ssim) -> float32[3] = (w_l1*L1 + w_ssim*(1-SSIM), L1, SSIM); only [0] is differentiable."""

    @staticmethod
    def forward(ctx, img, gt, w_l1, w_ssim):
        _check_inputs(img, gt)
        x, y = img.detach().to(torch.float32).contiguous(), gt.detach().to(torch.float32).contiguous()
        H, W = int(x.shape[-2]), int(x.shape[-1])
        planes = x.numel() // (H * W)
        need = [img.requires_grad, gt.requires_grad]
        out = torch.empty(3, dtype=torch.float32, device=x.device)
        ws = torch.empty(int(_lib.lib.gpsg_l1_ssim_workspace_bytes(planes, H, W)), dtype=torch.uint8, device=x.device)
        maps = [None, None]
        dev_stream = _lib.device_stream(x.device)
        with torch.cuda.device(x.device):
            # SSIM and L1 are symmetric in their two arguments: d/d(gt) is the same kernel with the roles swapped.
            for k, (a, b) in enumerate(((x, y), (y, x))):
                if k == 1 and not need[1]:
                    continue
                maps[k] = torch.empty((3,) + tuple(x.shape), dtype=torch.float32, device=x.device) if need[k] else None
                rc = _lib.lib.gpsg_l1_ssim_forward(*dev_stream, planes, H, W, _p(a), _p(b), float(w_l1), float(w_ssim),
                                                   _p(out), _p(maps[k]), _p(ws))
                _lib.check(rc, "gpsg_l1_ssim_forward")
        ctx.save_for_backward(x, y, *[m for m in maps if m is not None])
        ctx.cfg = (planes, H, W, float(w_l1), float(w_ssim), need, img.dtype, gt.dtype)
        # (loss, l1, ssim): only the loss carries a gradient; l1 / ssim are reporting values -- marked non-differentiable so
        # that building a loss from them raises instead of silently producing zero gradients (ADVICE r1)
        loss, l1, ss = out[0].clone(), out[1].clone(), out[2].clone()
        ctx.mark_non_differentiable(l1, ss)
        return loss, l1, ss

    @staticmethod
    def backward(ctx, grad_out, _g_l1=None, _g_ssim=None):
        planes, H, W, w_l1, w_ssim, need, dt_img, dt_gt = ctx.cfg
        saved = list(ctx.saved_tensors)
        x, y, rest = saved[0], saved[1], saved[2:]
        g = grad_out.detach().to(torch.float32).reshape(1).contiguous()  # d/d(loss), read on the device (no sync)
        res = [None, None]
        dev_stream = _lib.device_stream(x.device)
        with torch.cuda.device(x.device):
            for k, (a, b) in enumerate(((x, y), (y, x))):
                if not need[k]:
                    continue
                m = rest.pop(0)
                d = torch.empty_like(a)
                rc = _lib.lib.gpsg_l1_ssim_backward(*dev_stream, planes, H, W, _p(a), _p(b), _p(m), w_l1, w_ssim, _p(g), _p(d))
                _lib.check(rc, "gpsg_l1_ssim_backward")
                res[k] = d.to(dt_img if k == 0 else dt_gt)
        return res[0], res[1], None, None


def fused_l1_ssim(img, gt, w_l1=0.8, w_ssim=0.2):
    """== w_l1 * l1_loss(img, gt) + w_ssim * (1 - ssim(img, gt))   (reference train_stage2.py:70-72, without flow_loss)."""
    loss, l1, ss = _L1SSIM.apply(img, gt, w_l1, w_ssim)
    loss.l1, loss.ssim = l1, ss
    return loss


def l1_loss(network_output, gt):
    """reference lib/loss.py:35-36."""
    return _L1SSIM.apply(network_output, gt, 1.0, 0.0)[0]


def ssim(img1, img2, window_size=11, size_average=True):
    """reference lib/loss.py:52-72 (the only window the reference ever uses is the default 11 / sigma 1.5)."""
    if window_size != 11:
        raise NotImplementedError("gpsg ssim: window_size is fixed to 11 (reference default, lib/loss.py:52)")
    if size_average:
        return 1.0 - _L1SSIM.apply(img1, img2, 0.0, 1.0)[0]
    if img1.dim() != 4:
        raise RuntimeError("ssim(size_average=False) expects [B,C,H,W]")
    return torch.stack([1.0 - _L1SSIM.apply(img1[i], img2[i], 0.0, 1.0)[0] for i in range(img1.shape[0])])
