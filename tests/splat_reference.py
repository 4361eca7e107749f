"""Serial reference of the stage-1 preview splat (reference lib/TaichiRender.py:13-24), for tests.

It runs the C oracle's restatement (`oracle_taichi_splat` in oracle/taichi_splat_oracle.c: points in index order,
`if z > old: depth = z`, `if z >= old: colour = rgb`) in two ways `oracle.raster_oracle.taichi_splat` does not:
  - in/out: the caller's depth / colour buffers are updated in place, so the reference's two calls (lmain then rmain on
    the same buffers, TaichiRender.py:56-57) are two calls here;
  - any float input: the oracle casts x, y with C's `(int)`, which is undefined for NaN and |x| >= 2^31.  Here x and y
    are first replaced by their saturating truncation (NaN -> 0), clipped to [-1, res] so that the C cast is defined and
    the oracle's clamp to [0, res-1] gives what cvt.rzi.s32.f32 (CUDA's __float2int_rz) and the clamp give.
"""
import ctypes as C

import numpy as np

from oracle.raster_oracle import RasterOracle, _p


def saturating_pixel(x, res):
    """min(res-1, max(0, trunc_sat(x))) with NaN -> 0, as int64 (the device's pixel index)."""
    t = np.trunc(np.asarray(x, np.float64))
    return np.clip(np.where(np.isnan(t), 0.0, t), 0, res - 1).astype(np.int64)


def splat_serial(pts, mask, depth, color, B=None, N=None):
    """One call of the reference kernel over the loop domain (B, N) (default: all of pts), in place on depth
    [Bp,1,res,res] / color [Bp,3,res,res] (C-contiguous float32 numpy).  pts [Bp,Np,6], mask [Bp,Np] or [Bp,Np,1]."""
    o = RasterOracle("f32")
    pts = np.asarray(pts, np.float32)
    Bp, Np = pts.shape[:2]
    B = Bp if B is None else B
    N = Np if N is None else N
    res = depth.shape[-1]
    assert depth.dtype == np.float32 and color.dtype == np.float32 and depth.flags.c_contiguous and color.flags.c_contiguous
    assert depth.shape == (Bp, 1, res, res) and color.shape == (Bp, 3, res, res)
    p = np.ascontiguousarray(pts[:B, :N])
    for k in (0, 1):
        t = np.trunc(p[..., k].astype(np.float64))
        p[..., k] = np.clip(np.where(np.isnan(t), 0.0, t), -1, res).astype(np.float32)
    m = np.ascontiguousarray(np.asarray(mask, np.float32).reshape(Bp, Np)[:B, :N])
    d, c = depth[:B], color[:B]                      # contiguous views: the oracle writes through them
    o._fn("oracle_taichi_splat")(C.c_int(B), C.c_int(N), C.c_int(res), _p(p), _p(m), _p(d), _p(c))
    return depth, color


def fresh_buffers(Bp, res):
    """The reference's initial buffers (TaichiRender.py:53-55): depth 0, colour -1."""
    return np.zeros((Bp, 1, res, res), np.float32), np.full((Bp, 3, res, res), -1.0, np.float32)
