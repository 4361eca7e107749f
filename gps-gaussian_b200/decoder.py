"""The decoders of the Gaussian-parameter regressor on sm_90a, for inference in TF32: `decoder1` (csrc/decoder1.cu) and
`decoder3` / `decoder2` (csrc/decoder23.cu).

`GSRegresser.forward` (reference lib/gs_parm_network.py) runs `decoder1`, two ResidualBlocks (core/extractor.py) with
GroupNorm(6, 48), on cat(up(decoder2 output), img_feat1, depth_feat1) at half resolution: an upsample, a 128-channel
concat, five convolutions, five GroupNorms, ReLUs and two residual adds, each its own pass over tensors of 100 MB and
more at 1024^2.  `run` computes the same output in a chain of kernels that stage the concatenated input (the upsample
computed on the fly) and each normalized tensor while they load their input tile, so only the raw convolution outputs
reach memory.

Precision: TF32 as cuDNN with `allow_tf32` (autocast off; the regressor runs outside autocast).  The output differs
from cuDNN's by TF32 re-association; see include/gpsg.h for the exact semantics.  The regressor's forward with this
stage on the kernels is built by `gs_head.make_regresser_forward(orig, decoder=True)`.

`decoder3` (cat(img_feat3, depth_feat3) -> 96 channels at 1/8 resolution) and `decoder2` (cat(up(decoder3 output),
img_feat2, depth_feat2) -> 64 channels at 1/4) are the same ResidualBlock pair with GroupNorm(12, 96) and GroupNorm(8, 64);
`run3` / `run2` compute them the same way, and `make_regresser_forward(orig, decoder=True, deep=True)` puts them on the
kernels in front of decoder1.  `deep_counts()` counts their calls apart from decoder1's `counts()`.
"""
import ctypes as C
import sys

import torch
from torch import nn

from . import _lib

OUT_C, S_C, FEAT_C, GROUPS = 48, 64, 32, 6
IN_C = S_C + 2 * FEAT_C

PARAM_SHAPES = ((OUT_C, IN_C, 3, 3), (OUT_C,), (OUT_C,), (OUT_C,),
                (OUT_C, OUT_C, 3, 3), (OUT_C,), (OUT_C,), (OUT_C,),
                (OUT_C, IN_C, 1, 1), (OUT_C,), (OUT_C,), (OUT_C,),
                (OUT_C, OUT_C, 3, 3), (OUT_C,), (OUT_C,), (OUT_C,),
                (OUT_C, OUT_C, 3, 3), (OUT_C,), (OUT_C,), (OUT_C,))


def _p(t):
    return C.c_void_p(t.data_ptr())


def params_of(regresser):
    """The 20 tensors of `regresser.decoder1` in GpsgDecoder1Weights order (`_lib.DECODER1_PARAMS`): block 0's conv1,
    norm1, conv2, norm2, downsample conv and norm3, then block 1's conv1, norm1, conv2, norm2 (weight, bias each)."""
    b0, b1 = regresser.decoder1
    return (b0.conv1.weight, b0.conv1.bias, b0.norm1.weight, b0.norm1.bias,
            b0.conv2.weight, b0.conv2.bias, b0.norm2.weight, b0.norm2.bias,
            b0.downsample[0].weight, b0.downsample[0].bias, b0.norm3.weight, b0.norm3.bias,
            b1.conv1.weight, b1.conv1.bias, b1.norm1.weight, b1.norm1.bias,
            b1.conv2.weight, b1.conv2.bias, b1.norm2.weight, b1.norm2.bias)


def _conv(m, cin, cout, k):
    return (type(m) is nn.Conv2d and m.in_channels == cin and m.out_channels == cout and m.kernel_size == (k, k)
            and m.stride == (1, 1) and m.padding == ((k - 1) // 2,) * 2 and m.dilation == (1, 1) and m.groups == 1
            and m.padding_mode == "zeros" and m.bias is not None)


def _gn(m):
    return (type(m) is nn.GroupNorm and m.num_groups == GROUPS and m.num_channels == OUT_C and m.eps == 1e-5
            and m.affine)


def _module_supported(r):
    """The reference's stage-2 decoder1 exactly: ResidualBlock(128, 48) with a 1x1 downsample and GroupNorm(6, 48)
    everywhere, then ResidualBlock(48, 48) without one, and `up` a bilinear x2 Upsample without align_corners."""
    try:
        if list(getattr(r, "decoder_dims", ()))[:2] != [OUT_C, S_C]:
            return False
        up = r.up
        if not (type(up) is nn.Upsample and up.scale_factor in (2, 2.0, (2.0, 2.0)) and up.mode == "bilinear"
                and not up.align_corners and up.size is None):
            return False
        block_cls = getattr(sys.modules.get(type(r).__module__), "ResidualBlock", None)
        dec = r.decoder1
        if not (type(dec) is nn.Sequential and len(dec) == 2 and block_cls is not None):
            return False
        for blk, cin in zip(dec, (IN_C, OUT_C)):
            if not (type(blk) is block_cls and type(blk.relu) is nn.ReLU and _conv(blk.conv1, cin, OUT_C, 3)
                    and _conv(blk.conv2, OUT_C, OUT_C, 3) and _gn(blk.norm1) and _gn(blk.norm2)):
                return False
        b0, b1 = dec
        ds = b0.downsample
        if not (type(ds) is nn.Sequential and len(ds) == 2 and _conv(ds[0], IN_C, OUT_C, 1) and ds[1] is b0.norm3
                and _gn(b0.norm3)):
            return False
        return b1.downsample is None
    except (AttributeError, IndexError, TypeError, ValueError):
        return False


def _tensors_supported(dev, *ts):
    return all(torch.is_tensor(t) and t.is_cuda and t.device == dev and t.dtype == torch.float32 for t in ts)


def supported(regresser, s, f_i, f_d):
    """Whether the kernels run decoder1 of `regresser` on these inputs: CUDA fp32 tensors on one device, s [B,64,Hs,Ws]
    (the decoder2 output), f_i and f_d [B,32,2Hs,2Ws] (img_feat1, depth_feat1), B, Hs, Ws >= 1, the module's decoder1
    and upsample the reference's layers (see _module_supported) with fp32 parameters there too.  s or f_d None skips
    that tensor's checks (the shapes are then checked against f_i alone)."""
    if not (torch.is_tensor(f_i) and f_i.is_cuda and f_i.dim() == 4 and _module_supported(regresser)):
        return False
    dev = f_i.device
    B, c, H, W = f_i.shape
    if c != FEAT_C or B < 1 or H < 2 or W < 2 or H % 2 or W % 2:
        return False
    if not _tensors_supported(dev, f_i, *params_of(regresser)):
        return False
    if f_d is not None and not (_tensors_supported(dev, f_d) and tuple(f_d.shape) == (B, FEAT_C, H, W)):
        return False
    return s is None or (_tensors_supported(dev, s) and tuple(s.shape) == (B, S_C, H // 2, W // 2))


def forward_with_workspace(s, f_i, f_d, params, keep=True):
    """`run`, and the raw convolution outputs the kernels kept: (out, [y1, yd, y2, y3, y4]) with block 0's conv1,
    downsample and conv2 and block 1's conv1 and conv2 outputs, bias included, as fp32 NCHW [B,48,H,W] copies from the
    workspace.  keep=False skips the copies and returns an empty list."""
    if not all(torch.is_tensor(t) and t.dim() == 4 for t in (s, f_i, f_d)):
        raise RuntimeError("decoder1 (gpsg): s, f_i and f_d must be 4-D tensors")
    B, _, Hs, Ws = (int(v) for v in s.shape)
    H, W = 2 * Hs, 2 * Ws
    dev = s.device
    if not (_tensors_supported(dev, s, f_i, f_d, *params) and s.shape[1] == S_C and Hs >= 1 and Ws >= 1
            and tuple(f_i.shape) == (B, FEAT_C, H, W) and tuple(f_d.shape) == (B, FEAT_C, H, W)
            and len(params) == len(PARAM_SHAPES) and all(tuple(p.shape) == sh for p, sh in zip(params, PARAM_SHAPES))):
        raise RuntimeError(
            f"decoder1 (gpsg): needs CUDA fp32 s [B,64,Hs,Ws], f_i and f_d [B,32,2Hs,2Ws] and the 20 decoder1 parameters "
            f"on one device; got s {tuple(s.shape)} {s.dtype} {s.device}, f_i {tuple(f_i.shape)} {f_i.dtype}, f_d "
            f"{tuple(f_d.shape)} {f_d.dtype}")
    with torch.no_grad():
        sc, fi, fd = (t.detach().contiguous() for t in (s, f_i, f_d))
        ps = [p.detach().contiguous() for p in params]
        out = torch.empty((B, OUT_C, H, W), dtype=torch.float32, device=dev)
        if B == 0:
            return out, []
        nbytes = int(_lib.lib.gpsg_decoder1_workspace_bytes(B, Hs, Ws))
        ws = torch.empty(max(nbytes, 1), dtype=torch.uint8, device=dev)
        wt = _lib.Decoder1Weights(*[p.data_ptr() for p in ps])
        with torch.cuda.device(dev):
            rc = _lib.lib.gpsg_decoder1_forward(*_lib.device_stream(dev), B, Hs, Ws, _p(sc), _p(fi), _p(fd), wt,
                                                _p(out), _p(ws))
        _lib.check(rc, "gpsg_decoder1_forward")
        # workspace layout (include/gpsg.h): y1, yd, y2, y3, y4 NHWC, each at a multiple of its 256-byte-aligned size
        size = B * H * W * OUT_C * 4
        stride = (size + 255) // 256 * 256
        raws = [ws[i * stride:i * stride + size].view(torch.float32).view(B, H, W, OUT_C).permute(0, 3, 1, 2)
                .contiguous() for i in range(5)] if keep else []
    _COUNTS["forward"] += 1
    return out, raws


def run(s, f_i, f_d, params):
    """The kernels on raw tensors: s [B,64,Hs,Ws], f_i and f_d [B,32,2Hs,2Ws] and the 20 parameters in `params_of`
    order, all CUDA fp32 on one device -> decoder1's output [B,48,2Hs,2Ws] fp32, no autograd."""
    return forward_with_workspace(s, f_i, f_d, params, keep=False)[0]


_COUNTS = {"forward": 0}


def counts():
    """{'forward': n}: calls of the decoder1 kernels in this process."""
    return dict(_COUNTS)


def reset_counts():
    _COUNTS["forward"] = 0


# ---- decoder3 and decoder2 (csrc/decoder23.cu) ------------------------------------------------------------------------
# decoder3: cat(img_feat3, depth_feat3) [B,96+96,H,W] -> [B,96,H,W], GroupNorm(12, 96);
# decoder2: cat(up(decoder3 out), img_feat2, depth_feat2) [B,96+48+48,2H,2W] -> [B,64,2H,2W], GroupNorm(8, 64).
DEEP_IN_C = 192
D3_C, D2_C, FEAT3_C, FEAT2_C = 96, 64, 96, 48
DECODER_DIMS = [OUT_C, S_C, D3_C]            # the reference's stage-2 gsnet.decoder_dims
FEAT_DIMS = [FEAT_C, FEAT2_C, FEAT3_C]       # raft.encoder_dims = gsnet.encoder_dims


def _stage_shapes(cout):
    c, k = cout, DEEP_IN_C
    return ((c, k, 3, 3), (c,), (c,), (c,), (c, c, 3, 3), (c,), (c,), (c,), (c, k, 1, 1), (c,), (c,), (c,),
            (c, c, 3, 3), (c,), (c,), (c,), (c, c, 3, 3), (c,), (c,), (c,))


D3_PARAM_SHAPES, D2_PARAM_SHAPES = _stage_shapes(D3_C), _stage_shapes(D2_C)


def _stage_params(dec):
    b0, b1 = dec
    return (b0.conv1.weight, b0.conv1.bias, b0.norm1.weight, b0.norm1.bias,
            b0.conv2.weight, b0.conv2.bias, b0.norm2.weight, b0.norm2.bias,
            b0.downsample[0].weight, b0.downsample[0].bias, b0.norm3.weight, b0.norm3.bias,
            b1.conv1.weight, b1.conv1.bias, b1.norm1.weight, b1.norm1.bias,
            b1.conv2.weight, b1.conv2.bias, b1.norm2.weight, b1.norm2.bias)


def deep_params_of(regresser):
    """(decoder3's 20 tensors, decoder2's 20 tensors), each in GpsgDecoder23Weights order (`params_of`'s order)."""
    return _stage_params(regresser.decoder3), _stage_params(regresser.decoder2)


def _gn_of(m, c):
    return (type(m) is nn.GroupNorm and m.num_groups == c // 8 and m.num_channels == c and m.eps == 1e-5 and m.affine)


def _stage_supported(dec, block_cls, cin, c):
    """ResidualBlock(cin, c) with a 1x1 downsample, then ResidualBlock(c, c) without one, GroupNorm(c/8, c) everywhere."""
    if not (type(dec) is nn.Sequential and len(dec) == 2 and block_cls is not None):
        return False
    for blk, ci in zip(dec, (cin, c)):
        if not (type(blk) is block_cls and type(blk.relu) is nn.ReLU and _conv(blk.conv1, ci, c, 3)
                and _conv(blk.conv2, c, c, 3) and _gn_of(blk.norm1, c) and _gn_of(blk.norm2, c)):
            return False
    b0, b1 = dec
    ds = b0.downsample
    if not (type(ds) is nn.Sequential and len(ds) == 2 and _conv(ds[0], cin, c, 1) and ds[1] is b0.norm3
            and _gn_of(b0.norm3, c)):
        return False
    return b1.downsample is None


def _deep_module_supported(r):
    """The reference's stage-2 decoder3 and decoder2 exactly: decoder_dims [48, 64, 96], rgb and depth dims
    [32, 48, 96], norm_fn='group' (GroupNorm(c/8, c), eps 1e-5, affine) and `up` a bilinear x2 Upsample without
    align_corners."""
    try:
        if not (list(getattr(r, "decoder_dims", ())) == DECODER_DIMS and list(getattr(r, "rgb_dims", ())) == FEAT_DIMS
                and list(getattr(r, "depth_dims", ())) == FEAT_DIMS):
            return False
        up = r.up
        if not (type(up) is nn.Upsample and up.scale_factor in (2, 2.0, (2.0, 2.0)) and up.mode == "bilinear"
                and not up.align_corners and up.size is None):
            return False
        block_cls = getattr(sys.modules.get(type(r).__module__), "ResidualBlock", None)
        return (_stage_supported(r.decoder3, block_cls, DEEP_IN_C, D3_C)
                and _stage_supported(r.decoder2, block_cls, DEEP_IN_C, D2_C))
    except (AttributeError, IndexError, TypeError, ValueError):
        return False


def deep_supported(regresser, f3_i, f3_d, f2_i, f2_d):
    """Whether the kernels run decoder3 and decoder2 of `regresser` on these inputs: CUDA fp32 tensors on one device,
    f3_i and f3_d [B,96,H,W] (img_feat3, depth_feat3), f2_i and f2_d [B,48,2H,2W] (img_feat2, depth_feat2), B, H, W
    >= 1, both stages and the upsample the reference's layers (see _deep_module_supported) with fp32 parameters on the
    same device."""
    if not (all(torch.is_tensor(t) and t.dim() == 4 for t in (f3_i, f3_d, f2_i, f2_d)) and f3_i.is_cuda
            and _deep_module_supported(regresser)):
        return False
    dev = f3_i.device
    B, c, H, W = f3_i.shape
    if c != FEAT3_C or B < 1 or H < 1 or W < 1:
        return False
    p3, p2 = deep_params_of(regresser)
    if not _tensors_supported(dev, f3_i, f3_d, f2_i, f2_d, *p3, *p2):
        return False
    return (tuple(f3_d.shape) == (B, FEAT3_C, H, W) and tuple(f2_i.shape) == (B, FEAT2_C, 2 * H, 2 * W)
            and tuple(f2_d.shape) == (B, FEAT2_C, 2 * H, 2 * W))


def _raws(ws, B, H, W, c):
    # workspace layout (include/gpsg.h): ya, yd, yb, yc, ye NHWC, each at a multiple of its 256-byte-aligned size
    size = B * H * W * c * 4
    stride = (size + 255) // 256 * 256
    return [ws[i * stride:i * stride + size].view(torch.float32).view(B, H, W, c).permute(0, 3, 1, 2).contiguous()
            for i in range(5)]


def _check_params(params, shapes):
    return len(params) == len(shapes) and all(tuple(p.shape) == sh for p, sh in zip(params, shapes))


def forward3_with_workspace(f_i, f_d, params, keep=True):
    """`run3`, and the raw convolution outputs the kernels kept: (out, [ya, yd, yb, yc, ye]) as fp32 NCHW [B,96,H,W]
    copies from the workspace (bias included).  keep=False skips the copies and returns an empty list."""
    if not all(torch.is_tensor(t) and t.dim() == 4 for t in (f_i, f_d)):
        raise RuntimeError("decoder3 (gpsg): f_i and f_d must be 4-D tensors")
    B, _, H, W = (int(v) for v in f_i.shape)
    dev = f_i.device
    if not (_tensors_supported(dev, f_i, f_d, *params) and f_i.shape[1] == FEAT3_C and H >= 1 and W >= 1
            and tuple(f_d.shape) == (B, FEAT3_C, H, W) and _check_params(params, D3_PARAM_SHAPES)):
        raise RuntimeError(
            f"decoder3 (gpsg): needs CUDA fp32 f_i and f_d [B,96,H,W] and the 20 decoder3 parameters on one device; got "
            f"f_i {tuple(f_i.shape)} {f_i.dtype} {f_i.device}, f_d {tuple(f_d.shape)} {f_d.dtype}")
    with torch.no_grad():
        fi, fd = (t.detach().contiguous() for t in (f_i, f_d))
        ps = [p.detach().contiguous() for p in params]
        out = torch.empty((B, D3_C, H, W), dtype=torch.float32, device=dev)
        if B == 0:
            return out, []
        nbytes = int(_lib.lib.gpsg_decoder3_workspace_bytes(B, H, W))
        ws = torch.empty(max(nbytes, 1), dtype=torch.uint8, device=dev)
        wt = _lib.Decoder23Weights(*[p.data_ptr() for p in ps])
        with torch.cuda.device(dev):
            rc = _lib.lib.gpsg_decoder3_forward(*_lib.device_stream(dev), B, H, W, _p(fi), _p(fd), wt, _p(out), _p(ws))
        _lib.check(rc, "gpsg_decoder3_forward")
        raws = _raws(ws, B, H, W, D3_C) if keep else []
    _DEEP_COUNTS["decoder3"] += 1
    return out, raws


def forward2_with_workspace(s, f_i, f_d, params, keep=True):
    """`run2`, and the raw convolution outputs the kernels kept: (out, [ya, yd, yb, yc, ye]) as fp32 NCHW
    [B,64,2Hs,2Ws] copies from the workspace (bias included).  keep=False skips the copies and returns an empty list."""
    if not all(torch.is_tensor(t) and t.dim() == 4 for t in (s, f_i, f_d)):
        raise RuntimeError("decoder2 (gpsg): s, f_i and f_d must be 4-D tensors")
    B, _, Hs, Ws = (int(v) for v in s.shape)
    H, W = 2 * Hs, 2 * Ws
    dev = s.device
    if not (_tensors_supported(dev, s, f_i, f_d, *params) and s.shape[1] == D3_C and Hs >= 1 and Ws >= 1
            and tuple(f_i.shape) == (B, FEAT2_C, H, W) and tuple(f_d.shape) == (B, FEAT2_C, H, W)
            and _check_params(params, D2_PARAM_SHAPES)):
        raise RuntimeError(
            f"decoder2 (gpsg): needs CUDA fp32 s [B,96,Hs,Ws], f_i and f_d [B,48,2Hs,2Ws] and the 20 decoder2 "
            f"parameters on one device; got s {tuple(s.shape)} {s.dtype} {s.device}, f_i {tuple(f_i.shape)} "
            f"{f_i.dtype}, f_d {tuple(f_d.shape)} {f_d.dtype}")
    with torch.no_grad():
        sc, fi, fd = (t.detach().contiguous() for t in (s, f_i, f_d))
        ps = [p.detach().contiguous() for p in params]
        out = torch.empty((B, D2_C, H, W), dtype=torch.float32, device=dev)
        if B == 0:
            return out, []
        nbytes = int(_lib.lib.gpsg_decoder2_workspace_bytes(B, Hs, Ws))
        ws = torch.empty(max(nbytes, 1), dtype=torch.uint8, device=dev)
        wt = _lib.Decoder23Weights(*[p.data_ptr() for p in ps])
        with torch.cuda.device(dev):
            rc = _lib.lib.gpsg_decoder2_forward(*_lib.device_stream(dev), B, Hs, Ws, _p(sc), _p(fi), _p(fd), wt,
                                                _p(out), _p(ws))
        _lib.check(rc, "gpsg_decoder2_forward")
        raws = _raws(ws, B, H, W, D2_C) if keep else []
    _DEEP_COUNTS["decoder2"] += 1
    return out, raws


def run3(f_i, f_d, params):
    """decoder3 on the kernels: f_i and f_d [B,96,H,W] and the 20 parameters (deep_params_of(...)[0]), all CUDA fp32 on
    one device -> [B,96,H,W] fp32, no autograd."""
    return forward3_with_workspace(f_i, f_d, params, keep=False)[0]


def run2(s, f_i, f_d, params):
    """decoder2 on the kernels: s [B,96,Hs,Ws] (the decoder3 output), f_i and f_d [B,48,2Hs,2Ws] and the 20 parameters
    (deep_params_of(...)[1]), all CUDA fp32 on one device -> [B,64,2Hs,2Ws] fp32, no autograd."""
    return forward2_with_workspace(s, f_i, f_d, params, keep=False)[0]


_DEEP_COUNTS = {"decoder3": 0, "decoder2": 0}


def deep_counts():
    """{'decoder3': n, 'decoder2': m}: calls of the decoder3 / decoder2 kernels in this process (`counts()` counts
    decoder1's)."""
    return dict(_DEEP_COUNTS)


def reset_deep_counts():
    for k in _DEEP_COUNTS:
        _DEEP_COUNTS[k] = 0
