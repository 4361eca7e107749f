"""Mirror of reference lib/GaussianRender.py:5-39 -- `pts2render(data, bg_color)`: per sample, render the novel view
from the valid pixel-aligned Gaussians of both source views into data['novel_view']['img_pred'] [B,3,H,W].

The reference boolean-mask-gathers ten maps per sample (each gather is a `nonzero` + index_select, i.e. a host sync),
concatenates the two views, rescales the colours and only then calls `render`.  Here the sm_90a rasterizer reads the
maps in place (`gpsg_rasterize_forward_maps_begin` / `_finish`): invalid pixels are culled inside the projection
kernel, colours are img*0.5+0.5 on the fly, and the backward writes gradients directly in map layout.  Same signature,
same result (Gaussian order = lmain pixels then rmain pixels, exactly the order of the reference's gather + concat).
`pts2render_gather` keeps the reference's op-by-op data flow (gather -> `render`) for comparison.
`pts2render_ex(data, bg_color, aux=..., antialiasing=...)` is the one implementation behind `pts2render` and
`pts2render_aux`; antialiasing=True renders with the opacity-compensated screen-space filter (GPSG_FWD_ANTIALIAS).
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


def _sample_maps(maps, dev):
    """The 12 maps of one sample (lmain then rmain: valid, xyz, img, rot, scale, opacity), checked, as the pairs the C
    entry points take: (valid, xyz, img, rot, scale, opacity), each [lmain, rmain]."""
    vl, xl, il, rl, sl, ol, vr, xr, ir_, rr, sr, orr = maps
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
    return S2, (valid, xyz, img, rot, scale, opac)


def _maps_forward(ctx, settings_list, flags, maps, aux):
    """Forward of `_RasterizeMaps` (aux: `_RasterizeMapsAux`, which also writes depth and alpha [B,1,H,W]); `flags`: the
    GPSG_FWD_* word of the projection (`_begin`), which the backward follows through the saved image buffers."""
    B = len(settings_list)
    assert len(maps) == 12 * B
    dev = maps[1].device
    idx, sptr = _lib.device_stream(dev)
    H, W = int(settings_list[0].image_height), int(settings_list[0].image_width)
    out = torch.empty((B, 3, H, W), dtype=torch.float32, device=dev)
    depth = torch.empty((B, 1, H, W), dtype=torch.float32, device=dev) if aux else None
    alpha = torch.empty((B, 1, H, W), dtype=torch.float32, device=dev) if aux else None
    totals = torch.empty((B, 8), dtype=torch.int32, pin_memory=True)
    per = []
    for b in range(B):
        st = settings_list[b]
        if int(st.image_height) != H or int(st.image_width) != W:
            raise RuntimeError("pts2render (gpsg): all samples of a batch must render at one resolution")
        S2, tensors = _sample_maps(maps[12 * b:12 * b + 12], dev)
        radii = torch.empty((2 * S2,), dtype=torch.int32, device=dev)
        ptrs = [_ptrs(t) for t in tensors]
        _lib.begin_alloc(dev)
        try:
            with torch.cuda.device(dev):
                rc = _lib.lib.gpsg_rasterize_forward_maps_begin(
                    C.byref(st), idx, sptr, S2, *ptrs, C.c_void_p(radii.data_ptr()), _lib.ALLOC_CB, C.c_void_p(1),
                    _lib.ALLOC_CB, C.c_void_p(3), C.c_void_p(totals[b].data_ptr()), int(flags))
        finally:
            bufs = _lib.end_alloc()
        _lib.check(rc, "gpsg_rasterize_forward_maps_begin")
        per.append(dict(S2=S2, tensors=tensors, ptrs=ptrs, radii=radii, geom=bufs.get(1), image=bufs.get(3)))
    torch.cuda.current_stream(dev).synchronize()           # the ONE host synchronisation of the batch
    ctx.per = []
    for b in range(B):
        p = per[b]
        n = C.c_int32(0)
        extra = [C.c_void_p(depth[b].data_ptr()), C.c_void_p(alpha[b].data_ptr())] if aux else [None, None]
        _lib.begin_alloc(dev)
        try:
            with torch.cuda.device(dev):
                rc = _lib.lib.gpsg_rasterize_forward_maps_finish(
                    C.byref(settings_list[b]), idx, sptr, p["S2"], *p["ptrs"], C.c_void_p(out[b].data_ptr()), *extra,
                    C.c_void_p(p["radii"].data_ptr()), C.c_void_p(p["geom"].data_ptr()),
                    C.c_void_p(p["image"].data_ptr()), _lib.ALLOC_CB, C.c_void_p(2),
                    C.c_void_p(totals[b].data_ptr()), C.byref(n))
        finally:
            bufs = _lib.end_alloc()
        _lib.check(rc, "gpsg_rasterize_forward_maps_finish")
        ctx.per.append(dict(S2=p["S2"], n=int(n.value), tensors=p["tensors"], radii=p["radii"],
                            bufs=(p["geom"], bufs.get(2), p["image"])))
    ctx.settings_list = settings_list
    ctx.shapes = [tuple(m.shape) for m in maps]
    ctx._totals = totals                                   # keep the pinned words alive until the copies have landed
    return (out, depth, alpha) if aux else out


def _maps_backward(ctx, grad_out, grad_depth=None, grad_alpha=None):
    """Backward of both map Functions: gradients in map layout; with grad_depth / grad_alpha [B,1,H,W] also the aux
    gradients, on the aux forward's own buffers."""
    aux = grad_depth is not None
    grads = [None, None]                                   # settings_list, flags
    flags = _lib.backward_flags()
    dev = grad_out.device
    idx, sptr = _lib.device_stream(dev)
    for b, p in enumerate(ctx.per):
        new = lambda ref: [torch.empty_like(ref[0]), torch.empty_like(ref[1])]
        dxyz, dimg, drot, dscale, dopac = (new(t) for t in p["tensors"][1:])
        ws = torch.empty(int(_lib.lib.gpsg_rasterize_backward_maps_workspace_bytes(p["S2"], p["n"], flags, int(aux))),
                         dtype=torch.uint8, device=dev)
        g = _f32(grad_out[b].detach())
        gaux = [_f32(grad_depth[b].detach()), _f32(grad_alpha[b].detach())] if aux else [None, None]
        geom, binning, image = p["bufs"]
        with torch.cuda.device(dev):
            rc = _lib.lib.gpsg_rasterize_backward_maps(
                C.byref(ctx.settings_list[b]), idx, sptr, p["S2"], p["n"], *(_ptrs(t) for t in p["tensors"]),
                C.c_void_p(p["radii"].data_ptr()), C.c_void_p(geom.data_ptr()), C.c_void_p(binning.data_ptr()),
                C.c_void_p(image.data_ptr()), C.c_void_p(g.data_ptr()), *map(_lib._ptr, gaux), _ptrs(dxyz), _ptrs(dimg),
                _ptrs(drot), _ptrs(dscale), _ptrs(dopac), C.c_void_p(ws.data_ptr()), flags)
        _lib.check(rc, "gpsg_rasterize_backward_maps")
        sh = ctx.shapes[12 * b:12 * b + 12]
        grads += [None, dxyz[0].view(sh[1]), dimg[0].view(sh[2]), drot[0].view(sh[3]), dscale[0].view(sh[4]),
                  dopac[0].view(sh[5]), None, dxyz[1].view(sh[7]), dimg[1].view(sh[8]), drot[1].view(sh[9]),
                  dscale[1].view(sh[10]), dopac[1].view(sh[11])]
    return tuple(grads)


class _RasterizeMaps(torch.autograd.Function):
    """(settings_list, forward flags, *12 maps per sample) -> images [B,3,H,W] with ONE host synchronisation for the whole batch: every
    sample's projection / tile counting is enqueued first (`gpsg_rasterize_forward_maps_begin`), the stream is synchronised
    once, then every sample is binned, sorted and composited (`..._finish`).  The reference loops over the samples with one
    synchronisation each (lib/GaussianRender.py:8; upstream reads num_rendered per call)."""

    @staticmethod
    def forward(ctx, settings_list, flags, *maps):
        return _maps_forward(ctx, settings_list, flags, maps, aux=False)

    @staticmethod
    def backward(ctx, grad_out):
        return _maps_backward(ctx, grad_out)


class _RasterizeMapsAux(torch.autograd.Function):
    """`_RasterizeMaps` in aux mode: (images [B,3,H,W], depth [B,1,H,W], alpha [B,1,H,W]), same single synchronisation;
    the images are bit-identical to `_RasterizeMaps`'."""

    @staticmethod
    def forward(ctx, settings_list, flags, *maps):
        return _maps_forward(ctx, settings_list, flags, maps, aux=True)

    @staticmethod
    def backward(ctx, grad_out, grad_depth, grad_alpha):
        return _maps_backward(ctx, grad_out, grad_depth, grad_alpha)


def novel_settings(height, width, fovx, fovy, bg_color, cam):
    """RasterSettings of a novel camera from host values, filled as the reference's render() fills them
    (gaussian_renderer/__init__.py:36-49).  `cam`: 35 floats, world_view_transform (16), full_proj_transform (16) and
    camera_center (3)."""
    s = _lib.RasterSettings()
    s.image_height, s.image_width = int(height), int(width)
    s.tanfovx = math.tan(float(fovx) * 0.5)
    s.tanfovy = math.tan(float(fovy) * 0.5)
    s.bg[:] = [float(v) for v in bg_color]
    s.scale_modifier = 1.0
    s.viewmatrix[:] = cam[0:16]
    s.projmatrix[:] = cam[16:32]
    s.sh_degree = 3
    s.campos[:] = cam[32:35]
    s.prefiltered, s.debug = 0, 0
    return s


def pts2render(data, bg_color):
    """Whole batch with one host synchronisation (`_RasterizeMaps`)."""
    return pts2render_ex(data, bg_color)


def pts2render_aux(data, bg_color):
    """`pts2render` that also sets data['novel_view']['depth_pred'] (expected view-space depth, 0 where nothing is drawn)
    and ['alpha_pred'] (accumulated opacity: the foreground matte of the novel view), both [B,1,H,W] and differentiable,
    from the same forward and the same single host synchronisation (`_RasterizeMapsAux`).  img_pred is bit-identical to
    `pts2render`'s.  (A separate name keeps `pts2render`'s signature the reference's.)"""
    return pts2render_ex(data, bg_color, aux=True)


def pts2render_ex(data, bg_color, *, aux=False, antialiasing=False):
    """`pts2render` (aux=False) or `pts2render_aux` (aux=True); antialiasing=True renders every sample with the
    opacity-compensated screen-space filter (upstream's `antialiasing` setting: each splat's opacity is scaled so its
    integrated alpha does not grow with the fixed 0.3 px^2 dilation; conics, radii and tile lists are unchanged) and the
    backward differentiates that filter.  Same single host synchronisation per batch."""
    nv = data['novel_view']
    bs = data['lmain']['img'].shape[0]
    maps, settings = [], []
    for i in range(bs):
        for view in _VIEWS:
            d = data[view]
            maps += [d['pts_valid'][i], d['xyz'][i], d['img'][i], d['rot_maps'][i], d['scale_maps'][i], d['opacity_maps'][i]]
        # at most one device->host transfer for the 35 camera floats (CUDA in the test scripts, host in training)
        cam = torch.cat([nv[k][i].detach().reshape(-1).float()
                         for k in ('world_view_transform', 'full_proj_transform', 'camera_center')]).cpu().tolist()
        settings.append(novel_settings(nv['height'][i], nv['width'][i], nv['FovX'][i], nv['FovY'][i], bg_color, cam))
    flags = _lib.forward_flags(antialiasing)
    if aux:
        nv['img_pred'], nv['depth_pred'], nv['alpha_pred'] = _RasterizeMapsAux.apply(settings, flags, *maps)
    else:
        nv['img_pred'] = _RasterizeMaps.apply(settings, flags, *maps)
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
