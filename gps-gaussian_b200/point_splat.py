"""1-pixel z-buffer point splat on inverse depth (gpsg_point_splat, csrc/point_splat.cu): the stage-1 validation preview of
the reference (lib/TaichiRender.py:13-24, `TaichiRenderBatch.render_respective_color`), race-free and deterministic."""
import ctypes as C

import torch

from . import _lib


def point_splat(pts, mask, depth, color, B=None, N=None, res=None):
    """One call of `render_respective_color` over the loop domain (B, N), in place on `depth` / `color`.

    pts [Bp, Np, 6] = (x_pix, y_pix, inverse depth, r, g, b); mask [Bp, Np] or [Bp, Np, 1] (a point is skipped when
    mask < 0.5); depth [Bp, 1, res, res] and color [Bp, 3, res, res] are read and written.  All contiguous fp32 on one
    CUDA device.  B <= Bp and N <= Np default to Bp and Np; batches b >= B and rows i >= N are not touched.  `res`, when
    given, must match depth's size.  The result is the serial reading of the reference kernel (include/gpsg.h): per pixel
    the nearest point (largest z) wins, the highest index among equal z; calls in sequence compose like the reference's two.
    Launches on the device's current stream without synchronising.  Returns (depth, color)."""
    ts = dict(pts=pts, mask=mask, depth=depth, color=color)
    for name, t in ts.items():
        if not torch.is_tensor(t) or not t.is_cuda or t.dtype != torch.float32:
            raise TypeError(f"point_splat: {name} must be a CUDA float32 tensor")
        if not t.is_contiguous():
            raise TypeError(f"point_splat: {name} must be contiguous")
        if t.device != pts.device:
            raise TypeError(f"point_splat: {name} is on {t.device}, pts on {pts.device}")
    if pts.dim() != 3 or pts.shape[2] != 6:
        raise ValueError(f"point_splat: pts must be [Bp, Np, 6], got {tuple(pts.shape)}")
    Bp, Np = int(pts.shape[0]), int(pts.shape[1])
    if tuple(mask.shape) not in ((Bp, Np), (Bp, Np, 1)):
        raise ValueError(f"point_splat: mask must be [{Bp}, {Np}] or [{Bp}, {Np}, 1], got {tuple(mask.shape)}")
    R = int(depth.shape[-1]) if depth.dim() == 4 else -1
    if tuple(depth.shape) != (Bp, 1, R, R) or tuple(color.shape) != (Bp, 3, R, R) or (res is not None and int(res) != R):
        raise ValueError(f"point_splat: depth / color must be [{Bp}, 1, res, res] / [{Bp}, 3, res, res]"
                         f"{'' if res is None else f' with res = {res}'}, got {tuple(depth.shape)} / {tuple(color.shape)}")
    B = Bp if B is None else int(B)
    N = Np if N is None else int(N)
    if not (0 <= B <= Bp and 0 <= N <= Np):
        raise ValueError(f"point_splat: loop domain ({B}, {N}) exceeds the points' ({Bp}, {Np})")
    dev = pts.device
    ws = torch.empty(int(_lib.lib.gpsg_point_splat_workspace_bytes(B, R)), dtype=torch.uint8, device=dev)
    p = lambda t: C.c_void_p(t.data_ptr()) if t.numel() else None
    with torch.cuda.device(dev):
        rc = _lib.lib.gpsg_point_splat(*_lib.device_stream(dev), B, N, R, Np, p(pts), p(mask), p(depth), p(color), p(ws))
    _lib.check(rc, "gpsg_point_splat")
    return depth, color
