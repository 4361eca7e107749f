"""Mirror of reference lib/GaussianRender.py:5-39 -- `pts2render(data, bg_color)`: per sample, render the novel view
from the valid pixel-aligned Gaussians of both source views into data['novel_view']['img_pred'] [B,3,H,W].

The reference boolean-mask-gathers ten maps per sample (each gather is a `nonzero` + index_select, i.e. a host sync),
concatenates the two views, rescales the colours and only then calls `render`.  Here the sm_90a rasterizer reads the
maps in place (`gpsg_rasterize_forward_maps`): invalid pixels are culled inside the projection kernel, colours are
img*0.5+0.5 on the fly, and the backward writes gradients directly in map layout.  Same signature, same result
(Gaussian order = lmain pixels then rmain pixels, exactly the order of the reference's gather + concat).
`pts2render_gather` keeps the reference's op-by-op data flow (gather -> `render`) for comparison.
"""
import ctypes as C
import math

import torch

from . import _lib
from .gaussian_renderer import render

_VIEWS = ('lmain', 'rmain')


def _f32(t):
    return t.to(torch.float32).contiguous()


def _ptrs(ts):
    return (C.c_void_p * 2)(*[t.data_ptr() for t in ts])


class _RasterizeMaps(torch.autograd.Function):
    """(settings, valid_l, xyz_l, img_l, rot_l, scale_l, op_l, valid_r, xyz_r, img_r, rot_r, scale_r, op_r) -> image"""

    @staticmethod
    def forward(ctx, settings, *maps):
        vl, xl, il, rl, sl, ol, vr, xr, ir_, rr, sr, orr = maps
        dev = xl.device
        S2 = int(vl.numel())
        valid = [vl.contiguous().view(torch.uint8), vr.contiguous().view(torch.uint8)]
        xyz, img = [_f32(xl.detach()), _f32(xr.detach())], [_f32(il.detach()), _f32(ir_.detach())]
        rot, scale = [_f32(rl.detach()), _f32(rr.detach())], [_f32(sl.detach()), _f32(sr.detach())]
        opac = [_f32(ol.detach()), _f32(orr.detach())]
        if valid[1].numel() != S2:
            raise RuntimeError("pts2render (gpsg): lmain and rmain pts_valid differ in size")
        for t, n in ((xyz, 3), (img, 3), (rot, 4), (scale, 3), (opac, 1)):
            if any(u.numel() != n * S2 for u in t):
                raise RuntimeError("pts2render (gpsg): map shapes do not match pts_valid")
        if any(u.device != dev for t in (valid, xyz, img, rot, scale, opac) for u in t):
            raise RuntimeError("pts2render (gpsg): all source-view maps must live on one CUDA device")
        H, W = int(settings.image_height), int(settings.image_width)
        color = torch.empty((3, H, W), dtype=torch.float32, device=dev)
        radii = torch.empty((2 * S2,), dtype=torch.int32, device=dev)
        n = C.c_int32(0)
        idx = dev.index if dev.index is not None else torch.cuda.current_device()
        _lib.begin_alloc(dev)
        try:
            with torch.cuda.device(dev):
                rc = _lib.lib.gpsg_rasterize_forward_maps(
                    C.byref(settings), idx, C.c_void_p(torch.cuda.current_stream(dev).cuda_stream), S2, _ptrs(valid),
                    _ptrs(xyz), _ptrs(img), _ptrs(rot), _ptrs(scale), _ptrs(opac), C.c_void_p(color.data_ptr()),
                    C.c_void_p(radii.data_ptr()), _lib.ALLOC_CB, C.c_void_p(1), _lib.ALLOC_CB, C.c_void_p(2), _lib.ALLOC_CB,
                    C.c_void_p(3), C.byref(n))
        finally:
            bufs = _lib.end_alloc()
        _lib.check(rc, "gpsg_rasterize_forward_maps")
        ctx.settings, ctx.S2, ctx.n, ctx.idx = settings, S2, int(n.value), idx
        ctx.bufs = (bufs.get(1), bufs.get(2), bufs.get(3))
        ctx.shapes = [tuple(m.shape) for m in maps]
        ctx.save_for_backward(*(valid + xyz + img + rot + scale + opac + [radii]))
        return color

    @staticmethod
    def backward(ctx, grad_color):
        sv = ctx.saved_tensors
        valid, xyz, img, rot, scale, opac, radii = sv[0:2], sv[2:4], sv[4:6], sv[6:8], sv[8:10], sv[10:12], sv[12]
        dev, S2 = radii.device, ctx.S2
        new = lambda ref: [torch.empty_like(ref[0]), torch.empty_like(ref[1])]
        dxyz, dimg, drot, dscale, dopac = new(xyz), new(img), new(rot), new(scale), new(opac)
        ws = torch.empty(int(_lib.lib.gpsg_rasterize_backward_maps_workspace_bytes(S2)), dtype=torch.uint8, device=dev)
        g = _f32(grad_color.detach())
        geom, binning, image = ctx.bufs
        with torch.cuda.device(dev):
            rc = _lib.lib.gpsg_rasterize_backward_maps(
                C.byref(ctx.settings), ctx.idx, C.c_void_p(torch.cuda.current_stream(dev).cuda_stream), S2, ctx.n,
                _ptrs(valid), _ptrs(xyz), _ptrs(img), _ptrs(rot), _ptrs(scale), _ptrs(opac), C.c_void_p(radii.data_ptr()),
                C.c_void_p(geom.data_ptr()), C.c_void_p(binning.data_ptr()), C.c_void_p(image.data_ptr()),
                C.c_void_p(g.data_ptr()), _ptrs(dxyz), _ptrs(dimg), _ptrs(drot), _ptrs(dscale), _ptrs(dopac),
                C.c_void_p(ws.data_ptr()))
        _lib.check(rc, "gpsg_rasterize_backward_maps")
        sh = ctx.shapes
        out = [None, None, dxyz[0].view(sh[1]), dimg[0].view(sh[2]), drot[0].view(sh[3]), dscale[0].view(sh[4]),
               dopac[0].view(sh[5]), None, dxyz[1].view(sh[7]), dimg[1].view(sh[8]), drot[1].view(sh[9]),
               dscale[1].view(sh[10]), dopac[1].view(sh[11])]
        return tuple(out)


class _RasterizeMapsBatch(torch.autograd.Function):
    """(settings_list, *12 maps per sample) -> images [B,3,H,W] with ONE host synchronisation for the whole batch: every
    sample's projection / tile counting is enqueued first (`gpsg_rasterize_forward_maps_begin`), the stream is synchronised
    once, then every sample is binned, sorted and composited (`..._finish`).  The reference loops over the samples with one
    synchronisation each (lib/GaussianRender.py:8; upstream reads num_rendered per call).  Per-sample results, saved buffers
    and the backward are exactly those of `_RasterizeMaps`."""

    @staticmethod
    def forward(ctx, settings_list, *maps):
        B = len(settings_list)
        assert len(maps) == 12 * B
        dev = maps[1].device
        idx = dev.index if dev.index is not None else torch.cuda.current_device()
        stream = torch.cuda.current_stream(dev)
        sptr = C.c_void_p(stream.cuda_stream)
        H, W = int(settings_list[0].image_height), int(settings_list[0].image_width)
        out = torch.empty((B, 3, H, W), dtype=torch.float32, device=dev)
        totals = torch.zeros((B, 8), dtype=torch.int32).pin_memory()
        per = []
        for b in range(B):
            st = settings_list[b]
            if int(st.image_height) != H or int(st.image_width) != W:
                raise RuntimeError("pts2render (gpsg): all samples of a batch must render at one resolution")
            vl, xl, il, rl, sl, ol, vr, xr, ir_, rr, sr, orr = maps[12 * b:12 * b + 12]
            S2 = int(vl.numel())
            valid = [vl.contiguous().view(torch.uint8), vr.contiguous().view(torch.uint8)]
            xyz, img = [_f32(xl.detach()), _f32(xr.detach())], [_f32(il.detach()), _f32(ir_.detach())]
            rot, scale = [_f32(rl.detach()), _f32(rr.detach())], [_f32(sl.detach()), _f32(sr.detach())]
            opac = [_f32(ol.detach()), _f32(orr.detach())]
            if valid[1].numel() != S2:
                raise RuntimeError("pts2render (gpsg): lmain and rmain pts_valid differ in size")
            for t, n in ((xyz, 3), (img, 3), (rot, 4), (scale, 3), (opac, 1)):
                if any(u.numel() != n * S2 for u in t):
                    raise RuntimeError("pts2render (gpsg): map shapes do not match pts_valid")
            if any(u.device != dev for t in (valid, xyz, img, rot, scale, opac) for u in t):
                raise RuntimeError("pts2render (gpsg): all source-view maps must live on one CUDA device")
            radii = torch.empty((2 * S2,), dtype=torch.int32, device=dev)
            ptrs = (_ptrs(valid), _ptrs(xyz), _ptrs(img), _ptrs(rot), _ptrs(scale), _ptrs(opac))
            _lib.begin_alloc(dev)
            try:
                with torch.cuda.device(dev):
                    rc = _lib.lib.gpsg_rasterize_forward_maps_begin(
                        C.byref(st), idx, sptr, S2, *ptrs, C.c_void_p(radii.data_ptr()), _lib.ALLOC_CB, C.c_void_p(1),
                        _lib.ALLOC_CB, C.c_void_p(3), C.c_void_p(totals[b].data_ptr()))
            finally:
                bufs = _lib.end_alloc()
            _lib.check(rc, "gpsg_rasterize_forward_maps_begin")
            per.append(dict(S2=S2, tensors=valid + xyz + img + rot + scale + opac, ptrs=ptrs, radii=radii, geom=bufs.get(1),
                            image=bufs.get(3)))
        stream.synchronize()                                   # the ONE host synchronisation of the batch
        ctx.per = []
        for b in range(B):
            p = per[b]
            n = C.c_int32(0)
            _lib.begin_alloc(dev)
            try:
                with torch.cuda.device(dev):
                    rc = _lib.lib.gpsg_rasterize_forward_maps_finish(
                        C.byref(settings_list[b]), idx, sptr, p["S2"], *p["ptrs"], C.c_void_p(out[b].data_ptr()),
                        C.c_void_p(p["radii"].data_ptr()), C.c_void_p(p["geom"].data_ptr()), C.c_void_p(p["image"].data_ptr()),
                        _lib.ALLOC_CB, C.c_void_p(2), C.c_void_p(totals[b].data_ptr()), C.byref(n))
            finally:
                bufs = _lib.end_alloc()
            _lib.check(rc, "gpsg_rasterize_forward_maps_finish")
            ctx.per.append(dict(S2=p["S2"], n=int(n.value), tensors=p["tensors"], radii=p["radii"],
                                bufs=(p["geom"], bufs.get(2), p["image"])))
        ctx.settings_list, ctx.idx = settings_list, idx
        ctx.shapes = [tuple(m.shape) for m in maps]
        ctx._totals = totals                                   # keep the pinned words alive until the copies have landed
        return out

    @staticmethod
    def backward(ctx, grad_out):
        grads = [None]
        dev = grad_out.device
        for b, p in enumerate(ctx.per):
            t = p["tensors"]
            valid, xyz, img, rot, scale, opac = t[0:2], t[2:4], t[4:6], t[6:8], t[8:10], t[10:12]
            new = lambda ref: [torch.empty_like(ref[0]), torch.empty_like(ref[1])]
            dxyz, dimg, drot, dscale, dopac = new(xyz), new(img), new(rot), new(scale), new(opac)
            ws = torch.empty(int(_lib.lib.gpsg_rasterize_backward_maps_workspace_bytes(p["S2"])), dtype=torch.uint8, device=dev)
            g = _f32(grad_out[b].detach())
            geom, binning, image = p["bufs"]
            with torch.cuda.device(dev):
                rc = _lib.lib.gpsg_rasterize_backward_maps(
                    C.byref(ctx.settings_list[b]), ctx.idx, C.c_void_p(torch.cuda.current_stream(dev).cuda_stream), p["S2"],
                    p["n"], _ptrs(valid), _ptrs(xyz), _ptrs(img), _ptrs(rot), _ptrs(scale), _ptrs(opac),
                    C.c_void_p(p["radii"].data_ptr()), C.c_void_p(geom.data_ptr()), C.c_void_p(binning.data_ptr()),
                    C.c_void_p(image.data_ptr()), C.c_void_p(g.data_ptr()), _ptrs(dxyz), _ptrs(dimg), _ptrs(drot),
                    _ptrs(dscale), _ptrs(dopac), C.c_void_p(ws.data_ptr()))
            _lib.check(rc, "gpsg_rasterize_backward_maps")
            sh = ctx.shapes[12 * b:12 * b + 12]
            grads += [None, dxyz[0].view(sh[1]), dimg[0].view(sh[2]), drot[0].view(sh[3]), dscale[0].view(sh[4]),
                      dopac[0].view(sh[5]), None, dxyz[1].view(sh[7]), dimg[1].view(sh[8]), drot[1].view(sh[9]),
                      dscale[1].view(sh[10]), dopac[1].view(sh[11])]
        return tuple(grads)


def _settings(data, idx, bg_color):
    nv = data['novel_view']
    s = _lib.RasterSettings()
    s.image_height, s.image_width = int(nv['height'][idx]), int(nv['width'][idx])
    s.tanfovx = math.tan(float(nv['FovX'][idx]) * 0.5)
    s.tanfovy = math.tan(float(nv['FovY'][idx]) * 0.5)
    s.bg[:] = [float(v) for v in bg_color]
    s.scale_modifier = 1.0
    # at most one device->host transfer for the 35 camera floats (CUDA in the test scripts, host in training)
    cam = torch.cat([nv['world_view_transform'][idx].detach().reshape(-1).float(), nv['full_proj_transform'][idx].detach().reshape(-1).float(),
                     nv['camera_center'][idx].detach().reshape(-1).float()]).cpu().tolist()
    s.viewmatrix[:] = cam[0:16]
    s.projmatrix[:] = cam[16:32]
    s.sh_degree = 3
    s.campos[:] = cam[32:35]
    s.prefiltered, s.debug = 0, 0
    return s


def pts2render(data, bg_color):
    """Whole batch with one host synchronisation (`_RasterizeMapsBatch`); a batch of one takes the single-sample path."""
    bs = data['lmain']['img'].shape[0]
    maps, settings = [], []
    for i in range(bs):
        for view in _VIEWS:
            d = data[view]
            maps += [d['pts_valid'][i], d['xyz'][i], d['img'][i], d['rot_maps'][i], d['scale_maps'][i], d['opacity_maps'][i]]
        settings.append(_settings(data, i, bg_color))
    if bs == 1:
        data['novel_view']['img_pred'] = _RasterizeMaps.apply(settings[0], *maps).unsqueeze(0)
    else:
        data['novel_view']['img_pred'] = _RasterizeMapsBatch.apply(settings, *maps)
    return data


def pts2render_gather(data, bg_color):
    """The reference's data flow verbatim in behaviour: boolean-mask gather of both views, concat, rgb*0.5+0.5, render."""
    bs = data['lmain']['img'].shape[0]
    out = []
    for i in range(bs):
        parts = {k: [] for k in ('xyz', 'rgb', 'rot', 'scale', 'opacity')}
        for view in _VIEWS:
            d = data[view]
            valid = d['pts_valid'][i, :]
            parts['xyz'].append(d['xyz'][i][valid].view(-1, 3))
            parts['rgb'].append(d['img'][i].permute(1, 2, 0).reshape(-1, 3)[valid].view(-1, 3))
            parts['rot'].append(d['rot_maps'][i].permute(1, 2, 0).reshape(-1, 4)[valid].view(-1, 4))
            parts['scale'].append(d['scale_maps'][i].permute(1, 2, 0).reshape(-1, 3)[valid].view(-1, 3))
            parts['opacity'].append(d['opacity_maps'][i].permute(1, 2, 0).reshape(-1, 1)[valid].view(-1, 1))
        xyz = torch.cat(parts['xyz'], 0)
        rgb = torch.cat(parts['rgb'], 0) * 0.5 + 0.5
        img = render(data, i, xyz, rgb, torch.cat(parts['rot'], 0), torch.cat(parts['scale'], 0),
                     torch.cat(parts['opacity'], 0), bg_color=bg_color)
        out.append(img.unsqueeze(0))
    data['novel_view']['img_pred'] = torch.cat(out, 0)
    return data
