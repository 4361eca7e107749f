"""The full-resolution tail of the Gaussian-parameter regressor on sm_90a (csrc/gs_head.cu), forward and backward.

`GSRegresser.forward` (reference lib/gs_parm_network.py) runs at 1/8 to 1/2 resolution up to `decoder1`; its last step
upsamples the 48-channel decoder output x2, concatenates the image and the depth, and runs `out_conv` and the rot /
scale / opacity heads at full resolution, in fp32.  `gs_head` does that step in two TF32 warpgroup-MMA (wgmma)
kernels in place of the upsample / cat / seven convolutions / ReLU / activation chain, reading the half-resolution
decoder output, the image and the depth and writing the three maps.  `gs_head_train` is the same with autograd: its
backward (`gpsg_gs_head_backward`) recomputes the heads from the forward's saved 32-channel intermediate and returns
the gradients of the decoder output, the depth and the 14 weights (not the image's).

`make_regresser_forward(orig)` is `GSRegresser.forward` that hands the decoder1 output to `gs_head` when autograd is off
(the inference scripts and the stage-2 evaluation run under `torch.no_grad()`) and `supported(...)` holds; with grad
enabled (the training step), under autocast, or for inputs the kernels do not cover, it calls `orig`, the reference's
own method, unchanged.  `make_regresser_forward(orig, train=True)` also sends a grad-enabled call to `gs_head_train`
when the image does not require grad.  `make_regresser_forward(orig, tail=..., decoder=True)` also runs `decoder1` on
the kernels of gps_gaussian_b200.decoder (autograd and autocast off, cudnn.allow_tf32 on); it is the one restatement of
the regressor's forward for every combination, and with `tail=False` the tail runs on the module's own layers.  The maps
and gradients differ from cuDNN's TF32 convolutions by TF32
re-association; see include/gpsg.h for the exact semantics.
"""
import ctypes as C

import torch
from torch import nn
from torch.autograd.function import once_differentiable

from . import _lib
from . import decoder as _decoder

SRC_C, RGB_C, DEPTH_C, HEAD_C = 48, 3, 1, 32


def _p(t):
    return C.c_void_p(t.data_ptr())


def params_of(regresser):
    """The 14 weight / bias tensors of the tail, in GpsgGsHeadWeights order (`_lib.GS_HEAD_PARAMS`)."""
    r = regresser
    return (r.out_conv.weight, r.out_conv.bias,
            r.rot_head[0].weight, r.rot_head[0].bias, r.rot_head[2].weight, r.rot_head[2].bias,
            r.scale_head[0].weight, r.scale_head[0].bias, r.scale_head[2].weight, r.scale_head[2].bias,
            r.opacity_head[0].weight, r.opacity_head[0].bias, r.opacity_head[2].weight, r.opacity_head[2].bias)


PARAM_SHAPES = ((HEAD_C, SRC_C + RGB_C + DEPTH_C, 3, 3), (HEAD_C,),
                (HEAD_C, HEAD_C, 3, 3), (HEAD_C,), (4, HEAD_C, 1, 1), (4,),
                (HEAD_C, HEAD_C, 3, 3), (HEAD_C,), (3, HEAD_C, 1, 1), (3,),
                (HEAD_C, HEAD_C, 3, 3), (HEAD_C,), (1, HEAD_C, 1, 1), (1,))


def _conv(m, cin, cout, k):
    return (type(m) is nn.Conv2d and m.in_channels == cin and m.out_channels == cout and m.kernel_size == (k, k)
            and m.stride == (1, 1) and m.padding == ((k - 1) // 2,) * 2 and m.dilation == (1, 1) and m.groups == 1
            and m.padding_mode == "zeros" and m.bias is not None)


def _module_supported(r):
    try:
        heads = (r.rot_head, r.scale_head, r.opacity_head)
        if list(getattr(r, "decoder_dims", ()))[:1] != [SRC_C] or getattr(r, "head_dim", None) != HEAD_C:
            return False
        up = r.up
        if not (type(up) is nn.Upsample and up.scale_factor in (2, 2.0, (2.0, 2.0)) and up.mode == "bilinear"
                and not up.align_corners and up.size is None):
            return False
        if not (_conv(r.out_conv, SRC_C + RGB_C + DEPTH_C, HEAD_C, 3) and type(r.out_relu) is nn.ReLU):
            return False
        tails = ((4, ()), (3, (nn.Softplus,)), (1, (nn.Sigmoid,)))
        for head, (n, act) in zip(heads, tails):
            if type(head) is not nn.Sequential or len(head) != 3 + len(act):
                return False
            if not (_conv(head[0], HEAD_C, HEAD_C, 3) and type(head[1]) is nn.ReLU and _conv(head[2], HEAD_C, n, 1)):
                return False
            if act and type(head[3]) is not act[0]:
                return False
        sp = r.scale_head[3]
        return sp.beta == 100 and sp.threshold == 20
    except (AttributeError, IndexError, TypeError):
        return False


def _tensors_supported(dev, *ts):
    return all(torch.is_tensor(t) and t.is_cuda and t.device == dev and t.dtype == torch.float32 for t in ts)


def supported(regresser, img, depth, up_src):
    """Whether `gs_head` runs these inputs: CUDA fp32 tensors on one device, img [B,3,H,W] and depth [B,1,H,W] with H and W
    even, up_src [B,48,H/2,W/2] (None skips its check), fp32 weights there too, and a module whose tail has the expected
    layers (decoder_dims[0] == 48, head_dim == 32, 3x3 / 1x1 Conv2d with bias and zero padding, bilinear x2 Upsample
    without align_corners, Softplus(beta=100, threshold=20), Sigmoid)."""
    if not (torch.is_tensor(img) and img.is_cuda and _module_supported(regresser)):
        return False
    dev = img.device
    if not _tensors_supported(dev, img, depth, *params_of(regresser)):
        return False
    if img.dim() != 4 or depth.dim() != 4:
        return False
    B, c, H, W = img.shape
    if c != RGB_C or tuple(depth.shape) != (B, DEPTH_C, H, W) or H % 2 or W % 2:
        return False
    if up_src is not None:
        return _tensors_supported(dev, up_src) and tuple(up_src.shape) == (B, SRC_C, H // 2, W // 2)
    return True


def _check_args(up_src, img, depth, params):
    B, _, H, W = (int(s) for s in img.shape)
    dev = img.device
    if not (_tensors_supported(dev, up_src, img, depth, *params) and tuple(up_src.shape) == (B, SRC_C, H // 2, W // 2)
            and tuple(depth.shape) == (B, DEPTH_C, H, W) and img.shape[1] == RGB_C and H % 2 == 0 and W % 2 == 0
            and all(tuple(p.shape) == s for p, s in zip(params, PARAM_SHAPES)) and len(params) == len(PARAM_SHAPES)):
        raise RuntimeError(
            f"gs_head (gpsg): needs CUDA fp32 up_src [B,48,H/2,W/2], img [B,3,H,W], depth [B,1,H,W] with even H, W and "
            f"the 14 tail parameters on one device; got up_src {tuple(up_src.shape)} {up_src.dtype} {up_src.device}, "
            f"img {tuple(img.shape)} {img.dtype} {img.device}, depth {tuple(depth.shape)} {depth.dtype}")
    return B, H, W, dev


def forward_with_mid(up_src, img, depth, params):
    """`run`, and the forward's workspace: (rot, scale, opacity, mid) with mid the 32-channel intermediate, a flat fp32
    tensor holding NHWC [B,H,W,32] (TF32 values), as the backward takes it."""
    B, H, W, dev = _check_args(up_src, img, depth, params)
    with torch.no_grad():
        src, im, dp = (t.detach().contiguous() for t in (up_src, img, depth))
        ps = [p.detach().contiguous() for p in params]
        rot = torch.empty((B, 4, H, W), dtype=torch.float32, device=dev)
        scale = torch.empty((B, 3, H, W), dtype=torch.float32, device=dev)
        opacity = torch.empty((B, 1, H, W), dtype=torch.float32, device=dev)
        ws = torch.empty(max(int(_lib.lib.gpsg_gs_head_workspace_bytes(B, H, W)) // 4, 1), dtype=torch.float32,
                         device=dev)
        wt = _lib.GsHeadWeights(*[p.data_ptr() for p in ps])
        with torch.cuda.device(dev):
            rc = _lib.lib.gpsg_gs_head_forward(*_lib.device_stream(dev), B, H, W, _p(src), _p(im), _p(dp), _p(rot),
                                               _p(scale), _p(opacity), wt, _p(ws))
        _lib.check(rc, "gpsg_gs_head_forward")
    return rot, scale, opacity, ws


def run(up_src, img, depth, params):
    """The kernels on raw tensors: up_src [B,48,H/2,W/2], img [B,3,H,W], depth [B,1,H,W] and the 14 parameters in
    `params_of` order, all CUDA fp32 on one device -> (rot [B,4,H,W], scale [B,3,H,W], opacity [B,1,H,W])."""
    return forward_with_mid(up_src, img, depth, params)[:3]


_COUNTS = {"backward": 0}


def counts():
    """{'backward': n}: calls of the backward kernels in this process."""
    return dict(_COUNTS)


def reset_counts():
    _COUNTS["backward"] = 0


def backward(up_src, img, depth, params, mid, g_rot, g_scale, g_opacity, need_src=True, need_depth=True,
             workspace=None):
    """The backward kernels: (d_src or None, d_depth or None, [14 parameter gradients]) from the forward's inputs, its
    workspace `mid` (`forward_with_mid`) and the upstream gradients of rot, scale and opacity.  `workspace`: an fp32
    CUDA tensor of at least gpsg_gs_head_backward_workspace_bytes to use as scratch (allocated here when None); after
    the call its first B*H*W*48 floats hold dcat[:, :48] NHWC when d_src or d_depth was computed."""
    B, H, W, dev = _check_args(up_src, img, depth, params)
    gs = [g.detach().to(torch.float32).contiguous() for g in (g_rot, g_scale, g_opacity)]
    if not (_tensors_supported(dev, mid, *gs) and mid.numel() * 4 >= _lib.lib.gpsg_gs_head_workspace_bytes(B, H, W)
            and [tuple(g.shape) for g in gs] == [(B, 4, H, W), (B, 3, H, W), (B, 1, H, W)]):
        raise RuntimeError("gs_head backward (gpsg): needs the forward's workspace and fp32 gradients of the three maps")
    with torch.no_grad():
        src, im, dp = (t.detach().contiguous() for t in (up_src, img, depth))
        ps = [p.detach().contiguous() for p in params]
        d_src = torch.empty((B, SRC_C, H // 2, W // 2), dtype=torch.float32, device=dev) if need_src else None
        d_depth = torch.empty((B, DEPTH_C, H, W), dtype=torch.float32, device=dev) if need_depth else None
        grads = [torch.empty(s, dtype=torch.float32, device=dev) for s in PARAM_SHAPES]
        nbytes = int(_lib.lib.gpsg_gs_head_backward_workspace_bytes(B, H, W))
        ws = workspace
        if ws is None:
            ws = torch.empty(max(nbytes // 4, 1), dtype=torch.float32, device=dev)
        elif not (_tensors_supported(dev, ws) and ws.is_contiguous() and ws.numel() * 4 >= nbytes):
            raise RuntimeError("gs_head backward (gpsg): workspace must be a contiguous fp32 tensor on the device of "
                               f"at least {nbytes} bytes")
        wt = _lib.GsHeadWeights(*[p.data_ptr() for p in ps])
        gr = _lib.GsHeadGrads(*[g.data_ptr() for g in grads])
        opt = lambda t: _p(t) if t is not None else None
        with torch.cuda.device(dev):
            rc = _lib.lib.gpsg_gs_head_backward(*_lib.device_stream(dev), B, H, W, _p(src), _p(im), _p(dp), _p(mid),
                                                *[_p(g) for g in gs], opt(d_src), opt(d_depth), wt, gr, _p(ws))
        _lib.check(rc, "gpsg_gs_head_backward")
    _COUNTS["backward"] += 1
    return d_src, d_depth, grads


class _Tail(torch.autograd.Function):
    """The tail with autograd over (up_src, img, depth, *params); the image's gradient is not computed."""

    @staticmethod
    def forward(ctx, up_src, img, depth, *params):
        rot, scale, opacity, mid = forward_with_mid(up_src, img, depth, params)
        ctx.save_for_backward(up_src, img, depth, mid, *params)
        return rot, scale, opacity

    @staticmethod
    @once_differentiable
    def backward(ctx, g_rot, g_scale, g_opacity):
        up_src, img, depth, mid, *params = ctx.saved_tensors
        if ctx.needs_input_grad[1]:
            raise RuntimeError("gs_head_train (gpsg): the image's gradient is not computed")
        outs = []
        for g, c in zip((g_rot, g_scale, g_opacity), (4, 3, 1)):
            B, _, H, W = img.shape
            outs.append(g if g is not None else torch.zeros((B, c, H, W), dtype=torch.float32, device=img.device))
        need = ctx.needs_input_grad
        d_src, d_depth, grads = backward(up_src, img, depth, params, mid, *outs, need_src=need[0], need_depth=need[2])
        return (d_src, None, d_depth) + tuple(g if n else None for g, n in zip(grads, need[3:]))


def gs_head(up_src, img, depth, regresser):
    """(rot [B,4,H,W], scale [B,3,H,W], opacity [B,1,H,W]) of `regresser`'s tail from its decoder1 output up_src
    [B,48,H/2,W/2], the image [B,3,H,W] and the depth [B,1,H,W]: forward only, no autograd."""
    if not supported(regresser, img, depth, up_src):
        raise RuntimeError("gs_head (gpsg): inputs or module not supported; see gs_head.supported")
    return run(up_src, img, depth, params_of(regresser))


def gs_head_train(up_src, img, depth, regresser):
    """`gs_head` with autograd: gradients reach up_src, depth and the tail's 14 parameters through the backward kernels.
    The image must not require grad (its gradient is not computed)."""
    if not supported(regresser, img, depth, up_src):
        raise RuntimeError("gs_head (gpsg): inputs or module not supported; see gs_head.supported")
    if img.requires_grad and torch.is_grad_enabled():
        raise RuntimeError("gs_head_train (gpsg): the image's gradient is not computed; img must not require grad")
    return _Tail.apply(up_src, img, depth, *params_of(regresser))


def make_regresser_forward(orig, train=False, tail=True, decoder=False, deep=False):
    """`GSRegresser.forward` with parts of it on the kernels; otherwise `orig`, the reference's own method.

    tail: the full-resolution tail runs on the kernels when grad is disabled and the inputs are supported; with `train`,
    also when grad is enabled and the image does not require grad (`gs_head_train`).
    decoder: `decoder1` runs on the kernels (gps_gaussian_b200.decoder) when grad and autocast are off, cudnn.allow_tf32
    is on and `decoder.supported(...)` holds; the tail then runs on the kernels (with `tail`) or on the module's own
    layers.  With grad enabled decoder1 always stays the module's.
    deep: under the same conditions `decoder3` and `decoder2` run on the kernels (`decoder.run3`, `decoder.run2`) where
    `decoder.deep_supported(...)` holds; their output feeds decoder1 (kernels or module) as it is.  Otherwise they run
    on the module's own layers."""
    def forward(self, img, depth, img_feat):
        grad = torch.is_grad_enabled()
        autocast = torch.is_autocast_enabled()
        on_tail = (tail and not (grad and not (train and torch.is_tensor(img) and not img.requires_grad))
                   and not autocast and supported(self, img, depth, None))
        on_dec = (decoder and not grad and not autocast and torch.backends.cudnn.allow_tf32
                  and _decoder.supported(self, None, img_feat[0], None))
        on_deep = (deep and not grad and not autocast and torch.backends.cudnn.allow_tf32 and torch.is_tensor(img_feat[2])
                   and img_feat[2].is_cuda and _decoder._deep_module_supported(self))
        if not (on_tail or on_dec or on_deep):
            return orig(self, img, depth, img_feat)
        img_feat1, img_feat2, img_feat3 = img_feat
        depth_feat1, depth_feat2, depth_feat3 = self.depth_encoder(depth)
        if on_deep and _decoder.deep_supported(self, img_feat3, depth_feat3, img_feat2, depth_feat2):
            p3, p2 = _decoder.deep_params_of(self)
            x = _decoder.run2(_decoder.run3(img_feat3, depth_feat3, p3), img_feat2, depth_feat2, p2)
        else:
            x = self.decoder3(torch.cat([img_feat3, depth_feat3], dim=1))
            x = self.decoder2(torch.cat([self.up(x), img_feat2, depth_feat2], dim=1))
        decoded = on_dec and _decoder.supported(self, x, img_feat1, depth_feat1)
        if decoded:
            x = _decoder.run(x, img_feat1, depth_feat1, _decoder.params_of(self))
        else:
            x = self.decoder1(torch.cat([self.up(x), img_feat1, depth_feat1], dim=1))
        if on_tail and supported(self, img, depth, x):
            if grad:
                return _Tail.apply(x, img, depth, *params_of(self))
            return run(x, img, depth, params_of(self))
        if on_tail and not decoded:                   # e.g. fp16 image features: the decoders ran in fp16
            return orig(self, img, depth, img_feat)
        # the reference's tail (lib/gs_parm_network.py) on the module's own layers
        out = self.out_relu(self.out_conv(torch.cat([self.up(x), img, depth], dim=1)))
        rot_out = torch.nn.functional.normalize(self.rot_head(out), dim=1)
        scale_out = torch.clamp_max(self.scale_head(out), 0.01)
        opacity_out = self.opacity_head(out)
        return rot_out, scale_out, opacity_out
    forward.__doc__ = orig.__doc__
    return forward
