"""Fused unprojection in front of the rasterizer -- mirror of reference lib/network.py:64-69 (`flow2gsparms`, first
loop) built on lib/utils.py:87-119 (`flow2depth`, `depth2pc`): flow -> depth -> xyz + pts_valid in ONE sm_90a kernel
(and one for the backward), instead of ~12 elementwise / bmm torch kernels with repeat/cat copies."""
import ctypes as C

import torch

from . import _lib


class _Unproject(torch.autograd.Function):
    @staticmethod
    def forward(ctx, flow_pred, mask, intr, extr, ref_intr, tf_x):
        if not flow_pred.is_cuda:
            raise RuntimeError("unproject (gpsg): flow_pred must be a CUDA tensor")
        dev = flow_pred.device
        f32 = lambda t: t.detach().to(device=dev, dtype=torch.float32).contiguous()
        flow, m, K, E, Kr, tf = f32(flow_pred), f32(mask), f32(intr), f32(extr), f32(ref_intr), f32(tf_x).reshape(-1)
        # the kernels index every input by batch item and pixel without bounds: refuse any shape they would read past
        if flow.dim() != 4 or flow.shape[1] != 1 or flow.shape[2] != flow.shape[3]:
            raise RuntimeError(f"unproject (gpsg): flow_pred must be [B,1,S,S], got {tuple(flow.shape)}")
        B, _, S, _ = flow.shape
        if m.dim() != 4 or m.shape[0] != B or m.shape[1] < 1 or m.shape[2] != S or m.shape[3] != S:
            raise RuntimeError(f"unproject (gpsg): mask must be [{B},C,{S},{S}], got {tuple(m.shape)}")
        for name, t in (("intr", K), ("ref_intr", Kr)):
            if tuple(t.shape) != (B, 3, 3):
                raise RuntimeError(f"unproject (gpsg): {name} must be [{B},3,3], got {tuple(t.shape)}")
        if E.dim() != 3 or E.shape[0] != B or E.shape[1] < 3 or E.shape[2] != 4:
            raise RuntimeError(f"unproject (gpsg): extr must be [{B},>=3,4], got {tuple(E.shape)}")
        if tf.numel() != B:
            raise RuntimeError(f"unproject (gpsg): Tf_x must have {B} elements, got {tf.numel()}")
        depth = torch.empty((B, 1, S, S), dtype=torch.float32, device=dev)
        xyz = torch.empty((B, S * S, 3), dtype=torch.float32, device=dev)
        valid = torch.empty((B, S * S), dtype=torch.bool, device=dev)
        p = lambda t: C.c_void_p(t.data_ptr())
        with torch.cuda.device(dev):
            rc = _lib.lib.gpsg_unproject_forward(*_lib.device_stream(dev), B, S, p(flow),
                                                 p(m), int(m.stride(0)), p(K), p(E), int(E.shape[-2]), p(Kr), p(tf),
                                                 p(depth), p(xyz), p(valid))
        _lib.check(rc, "gpsg_unproject_forward")
        ctx.save_for_backward(depth, m, K, E, Kr, tf)
        ctx.meta = (B, S)
        ctx.mark_non_differentiable(valid)
        return depth, xyz, valid

    @staticmethod
    def backward(ctx, g_depth, g_xyz, _g_valid):
        depth, m, K, E, Kr, tf = ctx.saved_tensors
        B, S = ctx.meta
        dev = depth.device
        gx = g_xyz.detach().to(torch.float32).contiguous() if g_xyz is not None else None
        gd = g_depth.detach().to(torch.float32).contiguous() if g_depth is not None else None
        dflow = torch.empty((B, 1, S, S), dtype=torch.float32, device=dev)
        p = lambda t: C.c_void_p(t.data_ptr()) if t is not None else None
        with torch.cuda.device(dev):
            rc = _lib.lib.gpsg_unproject_backward(*_lib.device_stream(dev), B, S, p(depth),
                                                  p(m), int(m.stride(0)), p(K), p(E), int(E.shape[-2]), p(Kr), p(tf),
                                                  p(gx), p(gd), p(dflow))
        _lib.check(rc, "gpsg_unproject_backward")
        return dflow, None, None, None, None, None


def unproject_view(view):
    """`view` = data['lmain'] / data['rmain'] with keys flow_pred, mask, intr, extr, ref_intr, Tf_x.
    Returns (depth[B,1,S,S], xyz[B,S*S,3], pts_valid[B,S*S]) == flow2depth / depth2pc / `depth != 0`."""
    return _Unproject.apply(view['flow_pred'], view['mask'], view['intr'], view['extr'], view['ref_intr'], view['Tf_x'])


def flow2xyz(data):
    """The first loop of reference RtStereoHumanModel.flow2gsparms (lib/network.py:64-69), in place on `data`."""
    for name in ('lmain', 'rmain'):
        depth, xyz, valid = unproject_view(data[name])
        data[name]['depth'], data[name]['xyz'], data[name]['pts_valid'] = depth, xyz, valid
    return data
