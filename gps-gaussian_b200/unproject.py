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
        B, _, S, S2 = flow.shape
        if S != S2 or m.shape[0] != B or m.shape[-1] != S or E.shape[-1] != 4 or E.shape[-2] < 3:
            raise RuntimeError("unproject (gpsg): unexpected input shapes")
        depth = torch.empty((B, 1, S, S), dtype=torch.float32, device=dev)
        xyz = torch.empty((B, S * S, 3), dtype=torch.float32, device=dev)
        valid = torch.empty((B, S * S), dtype=torch.bool, device=dev)
        idx = dev.index if dev.index is not None else torch.cuda.current_device()
        p = lambda t: C.c_void_p(t.data_ptr())
        with torch.cuda.device(dev):
            rc = _lib.lib.gpsg_unproject_forward(idx, C.c_void_p(torch.cuda.current_stream(dev).cuda_stream), B, S, p(flow),
                                                 p(m), int(m.stride(0)), p(K), p(E), int(E.shape[-2]), p(Kr), p(tf),
                                                 p(depth), p(xyz), p(valid))
        _lib.check(rc, "gpsg_unproject_forward")
        ctx.save_for_backward(depth, m, K, E, Kr, tf)
        ctx.meta = (B, S, idx)
        ctx.mark_non_differentiable(valid)
        return depth, xyz, valid

    @staticmethod
    def backward(ctx, g_depth, g_xyz, _g_valid):
        depth, m, K, E, Kr, tf = ctx.saved_tensors
        B, S, idx = ctx.meta
        dev = depth.device
        gx = g_xyz.detach().to(torch.float32).contiguous() if g_xyz is not None else None
        gd = g_depth.detach().to(torch.float32).contiguous() if g_depth is not None else None
        dflow = torch.empty((B, 1, S, S), dtype=torch.float32, device=dev)
        p = lambda t: C.c_void_p(t.data_ptr()) if t is not None else None
        with torch.cuda.device(dev):
            rc = _lib.lib.gpsg_unproject_backward(idx, C.c_void_p(torch.cuda.current_stream(dev).cuda_stream), B, S, p(depth),
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
