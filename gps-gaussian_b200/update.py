"""The disparity update block on sm_90a (csrc/update_block.cu), for inference under fp16 autocast.

`FlowUpdateModule.forward` (reference core/raft_stereo_human.py) runs, per RAFT iteration, the corr lookup and then
`BasicMultiUpdateBlock` (core/update.py): the motion encoder, the ConvGRU and the flow and mask heads, twelve
convolutions and their elementwise glue.  `step` runs that block in six or seven kernels on fp16 wgmma with the hidden
state kept NHWC fp16 across iterations, `cz / cr / cq` read in place from the context tensor they were split from, and
coords1 updated in place.  The fp16 rounding points are autocast's (include/gpsg.h), so the results differ from cuDNN's
by the convolutions' accumulation order only, compounded over the iterations through the lookup.

`make_update_forward(orig)` is `FlowUpdateModule.forward` on the kernels when autograd is off, `args.mixed_precision`
is set and `supported(...)` holds; it builds the corr block through the module's own corr class, honours `flow_init`,
computes the mask only on iterations whose upsampled flow is returned and upsamples with `self.upsample_flow`.  In every
other case (grad enabled, fp32 eval, other GRU / hidden / corr / downsample configurations, foreign layers, CPU tensors
or other dtypes) it calls `orig`, the reference's own method, unchanged.
"""
import ctypes as C
import sys

import torch
from torch import nn

from . import _lib

HID, CORR_C, MASK_C = 96, 36, 576
PARAM_SHAPES = ((64, 36, 1, 1), (64,), (64, 64, 3, 3), (64,), (64, 2, 7, 7), (64,), (64, 64, 3, 3), (64,),
                (126, 128, 3, 3), (126,), (96, 224, 3, 3), (96,), (96, 224, 3, 3), (96,), (96, 224, 3, 3), (96,),
                (256, 96, 3, 3), (256,), (2, 256, 3, 3), (2,), (256, 96, 3, 3), (256,), (576, 256, 1, 1), (576,))
# workspace regions (include/gpsg.h): name -> channels, in order
REGIONS = (("h", 96), ("x", 128), ("cf1", 128), ("cf2", 128), ("z", 96), ("rh", 96), ("hid", 512), ("delta", 2))


def _p(t):
    return C.c_void_p(t.data_ptr() if t is not None else None)


def params_of(block):
    """The 24 tensors of a BasicMultiUpdateBlock in GpsgUpdateWeights order (`_lib.UPDATE_PARAMS`)."""
    e, g, f = block.encoder, block.gru08, block.flow_head
    out = []
    for m in (e.convc1, e.convc2, e.convf1, e.convf2, e.conv, g.convz, g.convr, g.convq, f.conv1, f.conv2,
              block.mask[0], block.mask[2]):
        out += [m.weight, m.bias]
    return tuple(out)


def _conv(m, cin, cout, k, pad):
    return (type(m) is nn.Conv2d and m.in_channels == cin and m.out_channels == cout and m.kernel_size == (k, k)
            and m.stride == (1, 1) and m.padding == (pad, pad) and m.dilation == (1, 1) and m.groups == 1
            and m.padding_mode == "zeros" and m.bias is not None)


def _block_supported(blk, mod):
    """blk is the reference's BasicMultiUpdateBlock of classes from `mod` (core.update) with the reference's layers."""
    try:
        cls = {n: getattr(mod, n) for n in ("BasicMultiUpdateBlock", "BasicMotionEncoder", "ConvGRU", "FlowHead")}
        e, g, f, m = blk.encoder, blk.gru08, blk.flow_head, blk.mask
        return (type(blk) is cls["BasicMultiUpdateBlock"] and type(e) is cls["BasicMotionEncoder"]
                and type(g) is cls["ConvGRU"] and type(f) is cls["FlowHead"]
                and _conv(e.convc1, CORR_C, 64, 1, 0) and _conv(e.convc2, 64, 64, 3, 1) and _conv(e.convf1, 2, 64, 7, 3)
                and _conv(e.convf2, 64, 64, 3, 1) and _conv(e.conv, 128, 126, 3, 1)
                and all(_conv(c, 224, HID, 3, 1) for c in (g.convz, g.convr, g.convq))
                and _conv(f.conv1, HID, 256, 3, 1) and _conv(f.conv2, 256, 2, 3, 1) and type(f.relu) is nn.ReLU
                and type(m) is nn.Sequential and len(m) == 3 and _conv(m[0], HID, 256, 3, 1)
                and type(m[1]) is nn.ReLU and _conv(m[2], 256, MASK_C, 1, 0))
    except (AttributeError, IndexError, TypeError, KeyError):
        return False


def _args_supported(a):
    try:
        return (bool(a.mixed_precision) and a.n_gru_layers == 1 and not a.slow_fast_gru
                and list(a.hidden_dims)[2] == HID and a.corr_levels == 4 and a.corr_radius == 4
                and a.n_downsample == 3 and a.corr_implementation in ("reg", "reg_cuda"))
    except (AttributeError, IndexError, TypeError):
        return False


def czrq_stride(inp0, B, H, W):
    """The batch stride (elements) of the [B,288,H,W] fp16 tensor that `split` made cz, cr, cq of, or None when the
    three are not such views."""
    try:
        cz, cr, cq = inp0
    except (TypeError, ValueError):
        return None
    hw = H * W
    if not all(torch.is_tensor(t) and t.dtype == torch.float16 and t.is_cuda and tuple(t.shape) == (B, HID, H, W)
               for t in (cz, cr, cq)):
        return None
    s = cz.stride()
    if any(t.stride() != s for t in (cr, cq)) or s[1:] != (hw, W, 1) or (B > 1 and s[0] < 3 * HID * hw):
        return None
    es = cz.element_size()
    if cr.data_ptr() != cz.data_ptr() + HID * hw * es or cq.data_ptr() != cz.data_ptr() + 2 * HID * hw * es:
        return None
    return s[0] if B > 1 else 3 * HID * hw


def supported(module, fmap1, net_list, inp_list):
    """Whether the kernels run this FlowUpdateModule: its args the stage-2 configuration (mixed precision, one GRU
    layer without slow-fast, hidden dim 96, corr levels / radius 4 / 4, n_downsample 3, corr "reg" or "reg_cuda"), its
    update block the reference's classes and layers with fp32 parameters on the device of net, net [B,96,H,W] fp16
    CUDA contiguous, cz / cr / cq the split of one [B,288,H,W] fp16 tensor, fmap1 a CUDA fp16 or fp32 tensor."""
    if not _args_supported(getattr(module, "args", None)):
        return False
    mod = sys.modules.get(type(getattr(module, "update_block", None)).__module__)
    if mod is None or not _block_supported(module.update_block, mod):
        return False
    try:
        net = net_list[0]
    except (TypeError, IndexError):
        return False
    if not (torch.is_tensor(net) and net.is_cuda and net.dtype == torch.float16 and net.dim() == 4
            and net.shape[1] == HID and net.is_contiguous() and min(net.shape) >= 1):
        return False
    if not (torch.is_tensor(fmap1) and fmap1.is_cuda and fmap1.dtype in (torch.float16, torch.float32)):
        return False
    B, _, H, W = net.shape
    try:
        if czrq_stride(inp_list[0], B, H, W) is None:
            return False
    except (TypeError, IndexError):
        return False
    ps = params_of(module.update_block)
    return all(p.is_cuda and p.device == net.device and p.dtype == torch.float32 for p in ps)


def pack(params):
    """The 24 parameters (`params_of` order, CUDA fp32) packed for the kernels (gpsg_update_pack): a uint8 tensor."""
    dev = params[0].device
    if not (len(params) == 24 and all(torch.is_tensor(p) and p.is_cuda and p.device == dev and p.dtype == torch.float32
                                      and tuple(p.shape) == s for p, s in zip(params, PARAM_SHAPES))):
        raise RuntimeError("update (gpsg): needs the 24 update-block parameters, CUDA fp32 on one device, in "
                           "params_of order and shapes")
    ps = [p.detach().contiguous() for p in params]
    out = torch.empty(int(_lib.lib.gpsg_update_packed_bytes()), dtype=torch.uint8, device=dev)
    with torch.cuda.device(dev):
        rc = _lib.lib.gpsg_update_pack(*_lib.device_stream(dev), _lib.UpdateWeights(*[p.data_ptr() for p in ps]),
                                       _p(out))
    _lib.check(rc, "gpsg_update_pack")
    out._gpsg_keep = ps                      # the pack kernel reads them asynchronously
    return out


def workspace(B, H, W, device):
    n = int(_lib.lib.gpsg_update_workspace_bytes(B, H, W))
    if n == 0:
        raise RuntimeError(f"update (gpsg): unsupported shape B={B} H={H} W={W}")
    return torch.empty(n, dtype=torch.uint8, device=device)


def regions(ws, B, H, W):
    """The workspace's NHWC fp16 regions as views: {name: [B,H,W,C]} (include/gpsg.h)."""
    out, off = {}, 0
    for name, c in REGIONS:
        size = B * H * W * c * 2
        out[name] = ws[off:off + size].view(torch.float16).view(B, H, W, c)
        off += (size + 255) // 256 * 256
    return out


def step(corr, coords1, net, czrq, czrq_bs, packed, ws, mask=None):
    """One iteration on raw tensors: corr [B,36,H,W] fp16 or fp32, coords1 [B,2,H,W] fp32 (updated in place), net
    [B,96,H,W] fp16 NCHW to load the hidden state from (None: the workspace's h from the previous step), czrq the cz
    view (cr, cq at 96 / 192 planes further), packed from `pack`, ws from `workspace`, mask None or [B,576,H,W] fp16
    (written).  No autograd."""
    B, _, H, W = coords1.shape
    dev = coords1.device
    if not (corr.is_contiguous() and tuple(corr.shape) == (B, CORR_C, H, W) and corr.dtype in (torch.float16, torch.float32)
            and coords1.is_contiguous() and coords1.dtype == torch.float32
            and (net is None or (net.is_contiguous() and net.dtype == torch.float16 and tuple(net.shape) == (B, HID, H, W)))
            and (mask is None or (mask.is_contiguous() and mask.dtype == torch.float16
                                  and tuple(mask.shape) == (B, MASK_C, H, W)))):
        raise RuntimeError("update (gpsg): corr [B,36,H,W] fp16/fp32, coords1 [B,2,H,W] fp32, net [B,96,H,W] fp16 and "
                           "mask [B,576,H,W] fp16, contiguous")
    with torch.cuda.device(dev):
        rc = _lib.lib.gpsg_update_step(*_lib.device_stream(dev), B, H, W, 1 if corr.dtype == torch.float16 else 0,
                                       _p(corr), _p(coords1), _p(net), _p(czrq), int(czrq_bs), _p(mask), _p(packed),
                                       _p(ws))
    _lib.check(rc, "gpsg_update_step")
    _COUNTS["steps"] += 1


def step_with_workspace(corr, coords1, net, czrq, params, mask=True):
    """One iteration from the caller's NCHW hidden state, returning every stage: a dict with the inputs the stages read
    (h_in, corr, coords1_in), the workspace regions after the step as fp32 NCHW (x, cf1, cf2, z, rh, h, fh1, m1, delta)
    and the outputs (coords1, mask).  czrq is the [B,288,H,W] fp16 context tensor.  Copies everything; for checks."""
    B, _, H, W = coords1.shape
    with torch.no_grad():
        packed = pack(params)
        ws = workspace(B, H, W, coords1.device)
        c1 = coords1.clone().contiguous()
        mk = torch.empty((B, MASK_C, H, W), dtype=torch.float16, device=coords1.device) if mask else None
        step(corr.contiguous(), c1, net.contiguous(), czrq, czrq.stride(0), packed, ws, mk)
        r = {k: v.permute(0, 3, 1, 2).float() for k, v in regions(ws, B, H, W).items()}
        out = dict(h_in=net.float(), corr=corr.float(), coords1_in=coords1.clone(), x=r["x"], cf1=r["cf1"],
                   cf2=r["cf2"], z=r["z"], rh=r["rh"], h=r["h"], fh1=r["hid"][:, :256], delta=r["delta"], coords1=c1)
        if mask:
            out["m1"], out["mask"] = r["hid"][:, 256:], mk.float()
    return out


_COUNTS = {"steps": 0, "forwards": 0}


def update_counts():
    """{'steps': n, 'forwards': m}: update-block iterations and FlowUpdateModule forwards run on the kernels."""
    return dict(_COUNTS)


def reset_update_counts():
    for k in _COUNTS:
        _COUNTS[k] = 0


def make_update_forward(orig):
    """`FlowUpdateModule.forward` with the update block on the kernels when grad is disabled and `supported` holds;
    otherwise `orig`.  Same signature and results: flow_up in test mode, the list of upsampled predictions otherwise."""
    def forward(self, fmap1, fmap2, net_list, inp_list, iters=12, flow_init=None, test_mode=False):
        if torch.is_grad_enabled() or iters < 1 or not supported(self, fmap1, net_list, inp_list):
            return orig(self, fmap1, fmap2, net_list, inp_list, iters, flow_init, test_mode)
        mod = sys.modules[type(self).__module__]
        if self.args.corr_implementation == "reg":
            corr_block = mod.CorrBlock1D
            fmap1, fmap2 = fmap1.float(), fmap2.float()
        else:
            corr_block = mod.CorrBlockFast1D
        corr_fn = corr_block(fmap1, fmap2, radius=self.args.corr_radius, num_levels=self.args.corr_levels)
        net = net_list[0]
        B, _, H, W = net.shape
        coords0, coords1 = self.initialize_flow(net)
        if flow_init is not None:
            coords1 = coords1 + flow_init
        coords1 = coords1.float().contiguous()          # a fresh tensor: the kernels update it in place
        cz = inp_list[0][0]
        czrq_bs = czrq_stride(inp_list[0], B, H, W)
        packed = pack(params_of(self.update_block))
        ws = workspace(B, H, W, net.device)
        flow_predictions, flow_up = [], None
        for itr in range(iters):
            corr = corr_fn(coords1)
            if corr.dtype not in (torch.float16, torch.float32) or tuple(corr.shape) != (B, CORR_C, H, W):
                raise RuntimeError(f"update (gpsg): the corr block returned {tuple(corr.shape)} {corr.dtype}")
            want = not test_mode or itr == iters - 1
            mask = torch.empty((B, MASK_C, H, W), dtype=torch.float16, device=net.device) if want else None
            step(corr.contiguous(), coords1, net if itr == 0 else None, cz, czrq_bs, packed, ws, mask)
            if not want:
                continue
            flow_up = self.upsample_flow(coords1 - coords0, mask)[:, :1]
            flow_predictions.append(flow_up)
        if iters > 0:
            net_list[0] = regions(ws, B, H, W)["h"].permute(0, 3, 1, 2)
        _COUNTS["forwards"] += 1
        if test_mode:
            return flow_up
        return flow_predictions
    forward.__doc__ = orig.__doc__
    return forward
