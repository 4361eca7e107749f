"""The UnetExtractor's half-resolution stem on sm_90a (csrc/encoder_stem.cu), for inference.

`UnetExtractor.forward` (reference core/extractor.py) runs `in_ds` (a 5x5 stride-2 convolution to 32 channels,
GroupNorm(8, 32), ReLU) and `res1` (two ResidualBlock(32, 32) with GroupNorm(4, 32)) at half resolution before `res2`
and `res3`.  It is the image encoder of RtStereoHumanModel (two source images, usually under fp16 autocast) and the depth
encoder of GSRegresser (two depth maps, fp32).  `run` computes the stem's output x1 in five kernels that write each raw
convolution output once and apply GroupNorm, ReLU and the residual while the next convolution stages its input.

Two precisions, as the reference's convolutions run them: "tf32" (autocast off with cudnn.allow_tf32, every
convolution operand rounded to TF32) and "fp16" (CUDA autocast in fp16: operands and biases rounded to fp16, each
convolution's output rounded to fp16, GroupNorm / ReLU / residual in fp32).  x1 differs from cuDNN's by TF32 or fp16
re-association; see include/gpsg.h for the exact semantics.

`run_down` computes one of the two stride-2 residual stages that follow (`res2`: 32 -> 48 channels, `res3`: 48 -> 96,
csrc/encoder_down.cu) in the same two precisions, from the previous stage's NCHW output to its own.

`make_extractor_forward(orig)` is `UnetExtractor.forward` that computes x1 on the kernels when autograd is off, the
precision is one of the two above and `supported(...)` holds, then runs the module's own `res2` and `res3` on it in the
caller's autocast context; with `deep=True` and res2 / res3 the reference's stages it computes x2 and x3 on the kernels too.  In every
other case (grad enabled, bf16 autocast, allow_tf32 off, CPU or non-fp32 input, another channel count, norm or layer
configuration) it calls `orig`, the reference's own method, unchanged.
"""
import ctypes as C
import sys

import torch
from torch import nn

from . import _lib

STEM_C = 32
PRECISIONS = {"tf32": _lib.ENCODER_STEM_TF32, "fp16": _lib.ENCODER_STEM_FP16}


def _p(t):
    return C.c_void_p(t.data_ptr())


def params_of(extractor):
    """The 20 stem tensors in GpsgEncoderStemWeights order (`_lib.ENCODER_STEM_PARAMS`)."""
    e = extractor
    out = [e.in_ds[0].weight, e.in_ds[0].bias, e.in_ds[1].weight, e.in_ds[1].bias]
    for blk in e.res1:
        out += [blk.conv1.weight, blk.conv1.bias, blk.norm1.weight, blk.norm1.bias,
                blk.conv2.weight, blk.conv2.bias, blk.norm2.weight, blk.norm2.bias]
    return tuple(out)


def param_shapes(cin):
    blk = ((STEM_C, STEM_C, 3, 3), (STEM_C,), (STEM_C,), (STEM_C,)) * 2
    return ((STEM_C, cin, 5, 5), (STEM_C,), (STEM_C,), (STEM_C,)) + blk * 2


def _conv(m, cin, cout, k, stride, pad):
    return (type(m) is nn.Conv2d and m.in_channels == cin and m.out_channels == cout and m.kernel_size == (k, k)
            and m.stride == (stride, stride) and m.padding == (pad, pad) and m.dilation == (1, 1) and m.groups == 1
            and m.padding_mode == "zeros" and m.bias is not None)


def _gn(m, groups):
    return (type(m) is nn.GroupNorm and m.num_groups == groups and m.num_channels == STEM_C and m.eps == 1e-5
            and m.affine)


def _module_supported(e, cin):
    try:
        ds = e.in_ds
        if not (type(ds) is nn.Sequential and len(ds) == 3 and _conv(ds[0], cin, STEM_C, 5, 2, 2) and _gn(ds[1], 8)
                and type(ds[2]) is nn.ReLU):
            return False
        block_cls = getattr(sys.modules.get(type(e).__module__), "ResidualBlock", None)
        if not (type(e.res1) is nn.Sequential and len(e.res1) == 2 and block_cls is not None):
            return False
        for blk in e.res1:
            if not (type(blk) is block_cls and blk.downsample is None and type(blk.relu) is nn.ReLU
                    and _conv(blk.conv1, STEM_C, STEM_C, 3, 1, 1) and _conv(blk.conv2, STEM_C, STEM_C, 3, 1, 1)
                    and _gn(blk.norm1, 4) and _gn(blk.norm2, 4)):
                return False
        return True
    except (AttributeError, IndexError, TypeError):
        return False


def _tensors_supported(dev, *ts):
    return all(torch.is_tensor(t) and t.is_cuda and t.device == dev and t.dtype == torch.float32 for t in ts)


def supported(extractor, x):
    """Whether the kernels run this module on x: x a CUDA fp32 tensor [B,Cin,H,W] with Cin 1 or 3 and H, W >= 1, the
    module's stem the reference's layers (Conv2d(Cin, 32, 5, stride 2, padding 2), GroupNorm(8, 32), ReLU, then two
    ResidualBlock(32, 32) without downsample, GroupNorm(4, 32), default eps, affine) with fp32 parameters on x's
    device."""
    if not (torch.is_tensor(x) and x.is_cuda and x.dtype == torch.float32 and x.dim() == 4):
        return False
    B, cin, H, W = x.shape
    if cin not in (1, 3) or H < 1 or W < 1 or B < 1 or not _module_supported(extractor, cin):
        return False
    return _tensors_supported(x.device, *params_of(extractor))


def precision_now():
    """The kernels' precision for the reference's convolutions in the current context: "fp16" under CUDA autocast in
    fp16, "tf32" with autocast off and cudnn.allow_tf32, otherwise None (bf16 autocast, TF32 off)."""
    if torch.is_autocast_enabled("cuda"):
        return "fp16" if torch.get_autocast_dtype("cuda") == torch.float16 else None
    return "tf32" if torch.backends.cudnn.allow_tf32 else None


def forward_with_workspace(x, params, precision, keep=True):
    """`run`, and the convolutions' raw outputs the kernels kept: (x1, [y0, y1, y2, y3, y4]) with y_i the i-th
    convolution's output, bias included, as fp32 NCHW [B,32,Ho,Wo] copies from the workspace (fp16 values in "fp16").
    keep=False skips the copies and returns an empty list."""
    if precision not in PRECISIONS:
        raise ValueError(f"encoder_stem (gpsg): precision must be 'tf32' or 'fp16', got {precision!r}")
    if not (torch.is_tensor(x) and x.dim() == 4):
        raise RuntimeError("encoder_stem (gpsg): x must be a 4-D tensor")
    B, cin, H, W = (int(s) for s in x.shape)
    dev = x.device
    if not (_tensors_supported(dev, x, *params) and cin in (1, 3) and H >= 1 and W >= 1
            and len(params) == 20 and all(tuple(p.shape) == s for p, s in zip(params, param_shapes(cin)))):
        raise RuntimeError(
            f"encoder_stem (gpsg): needs CUDA fp32 x [B,1 or 3,H,W] and the 20 stem parameters on one device; got x "
            f"{tuple(x.shape)} {x.dtype} {x.device}")
    prec = PRECISIONS[precision]
    Ho, Wo = (H + 1) // 2, (W + 1) // 2
    with torch.no_grad():
        xc = x.detach().contiguous()
        ps = [p.detach().contiguous() for p in params]
        out = torch.empty((B, STEM_C, Ho, Wo), dtype=torch.float32, device=dev)
        if B == 0:
            return out, []
        nbytes = int(_lib.lib.gpsg_encoder_stem_workspace_bytes(B, cin, H, W, prec))
        ws = torch.empty(max(nbytes, 1), dtype=torch.uint8, device=dev)
        wt = _lib.EncoderStemWeights(*[p.data_ptr() for p in ps])
        with torch.cuda.device(dev):
            rc = _lib.lib.gpsg_encoder_stem_forward(*_lib.device_stream(dev), B, cin, H, W, prec, _p(xc), wt, _p(out),
                                                    _p(ws))
        _lib.check(rc, "gpsg_encoder_stem_forward")
        # workspace layout (include/gpsg.h): y0 .. y4 NHWC, each at a multiple of its 256-byte-aligned size
        dt = torch.float16 if precision == "fp16" else torch.float32
        size = B * Ho * Wo * STEM_C * (2 if precision == "fp16" else 4)
        stride = (size + 255) // 256 * 256
        raws = [ws[i * stride:i * stride + size].view(dt).view(B, Ho, Wo, STEM_C).permute(0, 3, 1, 2).float()
                for i in range(5)] if keep else []
    _COUNTS[precision] += 1
    return out, raws


def run(x, params, precision):
    """The kernels on raw tensors: x [B,Cin,H,W] (Cin 1 or 3) and the 20 parameters in `params_of` order, all CUDA fp32
    on one device; precision "tf32" or "fp16" -> x1 [B,32,ceil(H/2),ceil(W/2)] fp32, no autograd."""
    return forward_with_workspace(x, params, precision, keep=False)[0]


_COUNTS = {"tf32": 0, "fp16": 0}


def counts():
    """{'tf32': n, 'fp16': m}: calls of the stem kernels in this process, per precision."""
    return dict(_COUNTS)


def reset_counts():
    for k in _COUNTS:
        _COUNTS[k] = 0


# ---- res2 / res3 ------------------------------------------------------------------------------------------------------
DOWN_DIMS = ((32, 48), (48, 96))       # (Cin, C) of res2 and res3 with encoder_dims [32, 48, 96]


def down_params_of(stage):
    """The 20 tensors of a down stage (`res2` or `res3`, two ResidualBlocks) in GpsgEncoderDownWeights order
    (`_lib.DECODER1_PARAMS`): block 0's conv1, norm1, conv2, norm2, downsample conv, norm3, then block 1's."""
    b0, b1 = stage[0], stage[1]
    return (b0.conv1.weight, b0.conv1.bias, b0.norm1.weight, b0.norm1.bias,
            b0.conv2.weight, b0.conv2.bias, b0.norm2.weight, b0.norm2.bias,
            b0.downsample[0].weight, b0.downsample[0].bias, b0.norm3.weight, b0.norm3.bias,
            b1.conv1.weight, b1.conv1.bias, b1.norm1.weight, b1.norm1.bias,
            b1.conv2.weight, b1.conv2.bias, b1.norm2.weight, b1.norm2.bias)


def down_param_shapes(cin, c):
    v, k3 = (c,), (c, c, 3, 3)
    return ((c, cin, 3, 3), v, v, v, k3, v, v, v, (c, cin, 1, 1), v, v, v) + (k3, v, v, v) * 2


def _gn_c(m, c):
    return type(m) is nn.GroupNorm and m.num_groups == c // 8 and m.num_channels == c and m.eps == 1e-5 and m.affine


def _stage_supported(stage, block_cls, cin, c):
    try:
        if not (type(stage) is nn.Sequential and len(stage) == 2 and block_cls is not None):
            return False
        b0, b1 = stage
        if not (type(b0) is block_cls and type(b1) is block_cls and type(b0.relu) is nn.ReLU
                and type(b1.relu) is nn.ReLU and b1.downsample is None):
            return False
        ds = b0.downsample
        if not (type(ds) is nn.Sequential and len(ds) == 2 and _conv(ds[0], cin, c, 1, 2, 0) and ds[1] is b0.norm3
                and _gn_c(b0.norm3, c)):
            return False
        return (_conv(b0.conv1, cin, c, 3, 2, 1) and _conv(b0.conv2, c, c, 3, 1, 1) and _conv(b1.conv1, c, c, 3, 1, 1)
                and _conv(b1.conv2, c, c, 3, 1, 1) and all(_gn_c(m, c) for m in (b0.norm1, b0.norm2, b1.norm1,
                                                                                   b1.norm2)))
    except (AttributeError, IndexError, TypeError):
        return False


def down_supported(stage, x):
    """Whether the kernels run this down stage on x: x a CUDA fp32 tensor [B,Cin,H,W] with H, W >= 1, (Cin, C) one of
    `DOWN_DIMS`, the stage the reference's two ResidualBlocks (the first Conv2d(Cin, C, 3, stride 2, padding 1) with the
    1x1 stride-2 downsample and its norm3, the second without downsample), GroupNorm(C/8, C) with eps 1e-5 and affine,
    with fp32 parameters on x's device."""
    if not (torch.is_tensor(x) and x.is_cuda and x.dtype == torch.float32 and x.dim() == 4):
        return False
    B, cin, H, W = x.shape
    dims = [d for d in DOWN_DIMS if d[0] == cin]
    if not dims or H < 1 or W < 1 or B < 1:
        return False
    try:
        block_cls = getattr(sys.modules.get(type(stage[0]).__module__), "ResidualBlock", None)
    except (IndexError, KeyError, TypeError):
        return False
    if not _stage_supported(stage, block_cls, *dims[0]):
        return False
    return _tensors_supported(x.device, *down_params_of(stage))


def down_forward_with_workspace(x, params, precision, keep=True):
    """`run_down`, and the convolutions' raw outputs the kernels kept: (out, [ya, yd, yb, yc, ye]) as fp32 NCHW
    [B,C,Ho,Wo] copies from the workspace (fp16 values in "fp16").  keep=False skips the copies and returns []."""
    if precision not in PRECISIONS:
        raise ValueError(f"encoder_down (gpsg): precision must be 'tf32' or 'fp16', got {precision!r}")
    if not (torch.is_tensor(x) and x.dim() == 4):
        raise RuntimeError("encoder_down (gpsg): x must be a 4-D tensor")
    B, cin, H, W = (int(s) for s in x.shape)
    dims = [d for d in DOWN_DIMS if d[0] == cin]
    c = dims[0][1] if dims else 0
    if not (dims and _tensors_supported(x.device, x, *params) and H >= 1 and W >= 1 and len(params) == 20
            and all(tuple(p.shape) == s for p, s in zip(params, down_param_shapes(cin, c)))):
        raise RuntimeError(
            f"encoder_down (gpsg): needs CUDA fp32 x [B,32 or 48,H,W] and the 20 stage parameters on one device; got x "
            f"{tuple(x.shape)} {x.dtype} {x.device}")
    prec = PRECISIONS[precision]
    Ho, Wo = (H + 1) // 2, (W + 1) // 2
    dev = x.device
    with torch.no_grad():
        xc = x.detach().contiguous()
        ps = [p.detach().contiguous() for p in params]
        out = torch.empty((B, c, Ho, Wo), dtype=torch.float32, device=dev)
        if B == 0:
            return out, []
        nbytes = int(_lib.lib.gpsg_encoder_down_workspace_bytes(B, cin, c, H, W, prec))
        ws = torch.empty(max(nbytes, 1), dtype=torch.uint8, device=dev)
        wt = _lib.EncoderDownWeights(*[p.data_ptr() for p in ps])
        with torch.cuda.device(dev):
            rc = _lib.lib.gpsg_encoder_down_forward(*_lib.device_stream(dev), B, cin, c, H, W, prec, _p(xc), wt,
                                                    _p(out), _p(ws))
        _lib.check(rc, "gpsg_encoder_down_forward")
        # workspace layout (include/gpsg.h): ya, yd, yb, yc, ye NHWC, each at a multiple of its 256-byte-aligned size
        dt = torch.float16 if precision == "fp16" else torch.float32
        size = B * Ho * Wo * c * (2 if precision == "fp16" else 4)
        stride = (size + 255) // 256 * 256
        raws = [ws[i * stride:i * stride + size].view(dt).view(B, Ho, Wo, c).permute(0, 3, 1, 2).float()
                for i in range(5)] if keep else []
    _DOWN_COUNTS[precision] += 1
    return out, raws


def run_down(x, params, precision):
    """One down stage on raw tensors: x [B,Cin,H,W] with Cin 32 (res2) or 48 (res3) and the 20 parameters in
    `down_params_of` order, all CUDA fp32 on one device; precision "tf32" or "fp16" -> [B,C,ceil(H/2),ceil(W/2)] fp32,
    no autograd."""
    return down_forward_with_workspace(x, params, precision, keep=False)[0]


_DOWN_COUNTS = {"tf32": 0, "fp16": 0}


def down_counts():
    """{'tf32': n, 'fp16': m}: calls of the res2 / res3 kernels in this process, per precision."""
    return dict(_DOWN_COUNTS)


def reset_down_counts():
    for k in _DOWN_COUNTS:
        _DOWN_COUNTS[k] = 0


def _down_stages_supported(extractor, dev):
    """For a module that `supported` accepted: whether its res2 and res3 are the reference's stages with encoder_dims
    [32, 48, 96] and fp32 parameters on `dev`.  `supported` has checked res1's blocks, so their class is the module's
    ResidualBlock."""
    try:
        block_cls, res2, res3 = type(extractor.res1[0]), extractor.res2, extractor.res3
    except (AttributeError, IndexError, TypeError):
        return False
    return (_stage_supported(res2, block_cls, *DOWN_DIMS[0]) and _stage_supported(res3, block_cls, *DOWN_DIMS[1])
            and _tensors_supported(dev, *down_params_of(res2), *down_params_of(res3)))


def make_extractor_forward(orig, deep=False):
    """`UnetExtractor.forward` with the stem (in_ds + res1) on the kernels when grad is disabled, the precision is
    TF32 or fp16 autocast (`precision_now`) and the module and input are `supported`; otherwise `orig`.  With deep=True
    and res2 / res3 the reference's stages with encoder_dims [32, 48, 96], they run on the kernels too (`run_down`)."""
    def forward(self, x):
        prec = None if torch.is_grad_enabled() else precision_now()
        if prec is None or not supported(self, x):
            return orig(self, x)
        if deep and _down_stages_supported(self, x.device):
            x1 = run(x, params_of(self), prec)
            x2 = run_down(x1, down_params_of(self.res2), prec)
            return x1, x2, run_down(x2, down_params_of(self.res3), prec)
        x1 = run(x, params_of(self), prec)
        x2 = self.res2(x1)
        x3 = self.res3(x2)
        return x1, x2, x3
    forward.__doc__ = orig.__doc__
    return forward
