"""Stereo rectification of the real-data loader on the GPU (gpsg_rectify_remap / gpsg_rectify_flow, csrc/rectify.cu).

The reference rectifies every frame on the CPU (lib/human_loader.py:245-366): cv2.stereoRectify, then per view
cv2.initUndistortRectifyMap and two cv2.remap calls, then, with depth, the ground-truth flow and the eroded valid mask,
and finally stereo_to_dict_tensor's elementwise pass.  Here cv2.stereoRectify (3x3 maths) and the reference's own
pts2depth stay on the host; the maps, every remap, the flow, the erode and the tensor contract run in two launches per
pair, bit-identical to the CPU path (DESIGN.md §2, "Rectification").

  rectify_stereo(main_view_data, ref_view_data, src_res, pts2depth=None)
      -> the dict of StereoHumanDataset.get_rectified_stereo_data (numpy: uint8 images / masks, fp64 flow, uint8 valid)
  stereo_item_cuda(main_view_data, ref_view_data, src_res, subject_name, pts2depth=None)
      -> the dict of stereo_to_dict_tensor, with lmain/rmain 'img' and 'mask' as CUDA tensors (same values, dtype,
         shape and strides); everything else as the CPU path makes it.

view data: (img [H,W,C] uint8, mask [H,W,Cm] uint8, intr [3,3], extr [3,4] or [4,4], pts or None), as load_single_view
returns it.  Inputs are uploaded from pageable memory; work runs on the current stream of `device` (default: the current
CUDA device).
"""
import ctypes as C

import numpy as np
import torch

from . import _lib


def stereo_rectify(main_view_data, ref_view_data, src_res):
    """cv2.stereoRectify of the pair, as get_rectified_stereo_data calls it (zero distortion, flags 0, (W, H) =
    (src_res, src_res)).  Returns (camera dict, ((K0, R0, P0), (K1, R1, P1))), the camera dict with the same fp64
    arrays: intr0/1 = P0/1[:3,:3], extr0/1 = R0/1 @ extr0/1, Tf_x = 0-d array of P1[0,3]."""
    import cv2
    intr0, extr0 = main_view_data[2], main_view_data[3]
    intr1, extr1 = ref_view_data[2], ref_view_data[3]
    r0, t0 = extr0[:3, :3], extr0[:3, 3:]
    r1, t1 = extr1[:3, :3], extr1[:3, 3:]
    world0 = np.eye(4)                       # inverse of view 0's extrinsic
    world0[:3, :3], world0[:3, 3:] = r0.T, -r0.T @ t0
    cam1 = np.eye(4)
    cam1[:3, :3], cam1[:3, 3:] = r1, t1
    rel = cam1 @ world0
    dist = np.zeros(4)
    R0, R1, P0, P1, _, _, _ = cv2.stereoRectify(intr0, dist, intr1, dist, (src_res, src_res), rel[:3, :3], rel[:3, 3],
                                                flags=0)
    camera = {'intr0': P0[:3, :3], 'intr1': P1[:3, :3], 'extr0': R0 @ extr0, 'extr1': R1 @ extr1,
              'Tf_x': np.array(P1[0, 3])}
    return camera, ((intr0, R0, P0), (intr1, R1, P1))


def _camera(K, R, P):
    c = _lib.RectifyCamera()
    for name, m in (("K", K), ("R", R), ("P", np.asarray(P)[:3, :3])):
        getattr(c, name)[:] = [float(x) for x in np.asarray(m, dtype=np.float64).reshape(9)]
    return c


def _hwc(a, what):
    a = a.contiguous() if torch.is_tensor(a) else np.ascontiguousarray(a)
    if a.dtype not in (np.uint8, torch.uint8) or a.ndim not in (2, 3) or (a.ndim == 3 and a.shape[2] not in (1, 3, 4)):
        raise ValueError(f"rectify: {what} must be uint8 [H, W] or [H, W, C] with C in (1, 3, 4), got "
                         f"{a.dtype} {a.shape}")
    return a


def _depths(views, camera, pts2depth):
    """The reference's own pts2depth of both views on the CPU (stereo_pts2flow, human_loader.py:67-70)."""
    if pts2depth is None:
        raise ValueError("rectify: pts given without the pts2depth function that turns them into depth")
    out = []
    for k, v in enumerate(views):
        d = pts2depth(torch.FloatTensor(v[4]), torch.FloatTensor(camera[f'extr{k}']), torch.FloatTensor(camera[f'intr{k}']))
        out.append(np.ascontiguousarray(d.detach().numpy(), dtype=np.float32))
    return out


def _empty(shape, dtype, device):
    return torch.empty(shape, dtype=dtype, device=device)


def rectify_device(views, cams, src_res, depths=None, Tf_x=None, numpy_out=True, tensor_out=False, device=None):
    """The two kernels on one pair.  views: ((img0, mask0), (img1, mask1)) uint8 numpy (or tensors, used in place
    when already on the device); cams: ((K, R, P), (K, R, P)) of
    stereo_rectify; depths: None or two float32 [Hin, Win] (then Tf_x is needed).  Returns per view k a dict of device
    tensors: numpy contract 'img', 'mask' (shapes as cv2.remap returns them), with depth also 'depth', 'flow' (fp64),
    'valid' (uint8); tensor contract 'img_t', 'mask_t' ([C,H,W] views of HWC storage)."""
    device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
    imgs = [_hwc(v[0], "img") for v in views]
    masks = [_hwc(v[1], "mask") for v in views]
    if imgs[0].shape != imgs[1].shape or masks[0].shape != masks[1].shape or imgs[0].shape[:2] != masks[0].shape[:2]:
        raise ValueError(f"rectify: both views need one image and mask size, got {[a.shape for a in imgs + masks]}")
    Hin, Win = imgs[0].shape[:2]
    Ci = imgs[0].shape[2] if imgs[0].ndim == 3 else 1
    Cm = masks[0].shape[2] if masks[0].ndim == 3 else 1
    if tensor_out and not (imgs[0].ndim == 3 and masks[0].ndim == 3 and Cm in (1, Ci)):
        raise ValueError("rectify: the tensor contract needs [H, W, C] images and masks with Cm == 1 or Cm == C")
    H = W = int(src_res)
    with_depth = depths is not None
    up = lambda a: a.to(device) if torch.is_tensor(a) else torch.from_numpy(a).to(device)
    new = lambda shape, dt: _empty(shape, dt, device)
    out, srcs, planes, cams_c = [], [], (_lib.RectifyPlanes * 2)(), (_lib.RectifyCamera * 2)()
    for k in range(2):
        o = {}
        src = dict(img=up(imgs[k]), mask=up(masks[k]))
        srcs.append(src)                                         # alive until launched: no output may reuse their blocks
        if numpy_out or with_depth:                              # the flow kernel reads the rectified mask
            o['img'] = new((H, W, Ci) if Ci > 1 else (H, W), torch.uint8)
            o['mask'] = new((H, W, Cm) if Cm > 1 else (H, W), torch.uint8)
        if with_depth:
            src['depth'] = up(depths[k].contiguous() if torch.is_tensor(depths[k]) else
                              np.ascontiguousarray(depths[k], dtype=np.float32))
            if src['depth'].shape != (Hin, Win):
                raise ValueError(f"rectify: depth must be [{Hin}, {Win}], got {tuple(src['depth'].shape)}")
            o['depth'] = new((H, W), torch.float32)
        if tensor_out:
            o['img_t'] = new((H, W, Ci), torch.float32).permute(2, 0, 1)
            o['mask_t'] = new((H, W, Cm), torch.float32).permute(2, 0, 1)
        p = lambda t: t.data_ptr() if t is not None else None
        planes[k] = _lib.RectifyPlanes(p(src['img']), p(src['mask']), p(src.get('depth')), p(o.get('img')),
                                       p(o.get('mask')), p(o.get('depth')), p(o.get('img_t')), p(o.get('mask_t')))
        cams_c[k] = _camera(*cams[k])
        out.append(o)
    idx, stream = _lib.device_stream(device)
    with torch.cuda.device(device):
        rc = _lib.lib.gpsg_rectify_remap(idx, stream, cams_c, Hin, Win, Ci, Cm, H, W, planes)
        _lib.check(rc, "gpsg_rectify_remap")
        if with_depth:
            for o in out:
                o['flow'] = new((H, W), torch.float64)
                o['valid'] = new((H, W), torch.uint8)
            arr = lambda key: (C.c_void_p * 2)(*[o[key].data_ptr() for o in out])
            rc = _lib.lib.gpsg_rectify_flow(idx, stream, H, W, Cm, float(Tf_x), float(np.asarray(cams[0][2])[0, 2]),
                                            float(np.asarray(cams[1][2])[0, 2]), arr('depth'), arr('mask'), arr('flow'),
                                            arr('valid'))
            _lib.check(rc, "gpsg_rectify_flow")
    # the uploaded inputs are freed on return: the caching allocator hands their blocks only to later work on this
    # stream, which runs after the kernels that read them
    del srcs
    return out


def _pair(main_view_data, ref_view_data, src_res, pts2depth, numpy_out, tensor_out, device):
    views = (main_view_data, ref_view_data)
    camera, cams = stereo_rectify(main_view_data, ref_view_data, src_res)
    depths = _depths(views, camera, pts2depth) if main_view_data[4] is not None else None
    out = rectify_device([(v[0], v[1]) for v in views], cams, src_res, depths=depths, Tf_x=camera['Tf_x'],
                         numpy_out=numpy_out, tensor_out=tensor_out, device=device)
    return camera, out


def rectify_stereo(main_view_data, ref_view_data, src_res, pts2depth=None, device=None):
    """StereoHumanDataset.get_rectified_stereo_data on the GPU: the same dict, keys, dtypes, shapes and values.
    pts2depth: the reference's own function (lib.human_loader.pts2depth), needed when the views carry pts."""
    camera, out = _pair(main_view_data, ref_view_data, src_res, pts2depth, True, False, device)
    host = [{k: t.cpu().numpy() for k, t in o.items()} for o in out]
    data = {'img0': host[0]['img'], 'mask0': host[0]['mask'], 'img1': host[1]['img'], 'mask1': host[1]['mask'],
            'camera': camera}
    if 'flow' in host[0]:
        data.update({'flow0': host[0]['flow'], 'valid0': host[0]['valid'], 'flow1': host[1]['flow'],
                     'valid1': host[1]['valid']})
    return data


def stereo_item_cuda(main_view_data, ref_view_data, src_res, subject_name, pts2depth=None, device=None):
    """get_rectified_stereo_data followed by stereo_to_dict_tensor, without the numpy round trip: lmain/rmain 'img'
    ([C,H,W] fp32) and 'mask' ([Cm,H,W] fp32) are CUDA tensors with the CPU path's values and strides; intr, ref_intr,
    extr and Tf_x (and flow / valid when the views carry pts) are the CPU tensors that function makes."""
    with_pts = main_view_data[4] is not None
    camera, out = _pair(main_view_data, ref_view_data, src_res, pts2depth, False, True, device)
    views = []
    for k in range(2):
        v = {'img': out[k]['img_t'], 'mask': out[k]['mask_t'],
             'intr': torch.FloatTensor(camera[f'intr{k}']), 'ref_intr': torch.FloatTensor(camera[f'intr{1 - k}']),
             'extr': torch.FloatTensor(camera[f'extr{k}']),
             'Tf_x': torch.FloatTensor(camera['Tf_x']) if k == 0 else -torch.FloatTensor(camera['Tf_x'])}
        if with_pts:
            v['flow'] = torch.unsqueeze(out[k]['flow'].cpu(), dim=0)
            v['valid'] = torch.unsqueeze(out[k]['valid'].cpu(), dim=0) / 255.0
        views.append(v)
    return {'name': subject_name, 'lmain': views[0], 'rmain': views[1]}
