"""ctypes front-end of the CPU rasterizer oracle (oracle/gpsg_oracle.c).

TEST INFRASTRUCTURE, NOT PRODUCT CODE.  Only tests/, __graft_entry__.smoke() and the
cpu_baseline / `--impl reference` legs of bench.py may import this module.

The oracle restates SURVEY.md Appendix A (the published algorithm of
graphdeco-inria/diff-gaussian-rasterization, pre-antialiasing API, which the reference calls at
gaussian_renderer/__init__.py:36-62 and which is absent from the original project's tree).
PARITY UNPINNED against the real extension -- see the header of gpsg_oracle.c.
"""
import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIBS = {}


def _lib(tag):
    if tag not in _LIBS:
        path = os.path.join(_HERE, "_build", f"liboracle_{tag}.so")
        if not os.path.exists(path):
            import importlib.util
            spec = importlib.util.spec_from_file_location("_oracle_build", os.path.join(_HERE, "build.py"))
            mod = importlib.util.module_from_spec(spec)
            spec.loader.exec_module(mod)
            mod.build()
        _LIBS[tag] = C.CDLL(path)
    return _LIBS[tag]


def _p(a):
    return a.ctypes.data_as(C.c_void_p) if a is not None else None


class RasterOracle:
    """dtype 'f32' (fixed-op-order fp32, for bit-exact integer parity) or 'f64' (gradient truth)."""

    def __init__(self, dtype="f32"):
        assert dtype in ("f32", "f64")
        self.tag = dtype
        self.np = np.float32 if dtype == "f32" else np.float64
        self.creal = C.c_float if dtype == "f32" else C.c_double
        self.lib = _lib(dtype)

    def _fn(self, name):
        return getattr(self.lib, f"{name}_{self.tag}")

    def _a(self, x, shape=None):
        if x is None:
            return None
        x = np.ascontiguousarray(np.asarray(x, dtype=self.np))
        if shape is not None:
            x = x.reshape(shape)
        return x

    def max_threads(self):
        """Host cores available to OpenMP (not OMP_NUM_THREADS, which torchrun forces to 1)."""
        return int(self._fn("oracle_max_threads")())

    def set_threads(self, n):
        self._fn("oracle_set_threads")(C.c_int(int(n)))

    def sh_colors(self, means3D, campos, shs, deg):
        """SH -> RGB (+0.5, clamp at 0).  shs: [P, M, 3].  Returns (colors[P,3], clamped[P,3] bool)."""
        shs = self._a(shs); P, M = shs.shape[0], shs.shape[1]
        m3 = self._a(means3D, (P, 3)); cp = self._a(campos, (3,))
        col = np.zeros((P, 3), self.np); cl = np.zeros((P, 3), np.uint8)
        self._fn("oracle_sh_forward")(C.c_int(P), C.c_int(deg), C.c_int(M), _p(m3), _p(cp), _p(shs), _p(col), _p(cl))
        return col, cl

    def sh_backward(self, means3D, campos, shs, deg, clamped, dL_dcolors, dL_dmeans3D):
        """Returns dL_dsh[P,M,3]; ADDS the view-direction term into dL_dmeans3D (in place)."""
        shs = self._a(shs); P, M = shs.shape[0], shs.shape[1]
        m3 = self._a(means3D, (P, 3)); cp = self._a(campos, (3,)); g = self._a(dL_dcolors, (P, 3))
        cl = np.ascontiguousarray(clamped, np.uint8)
        dsh = np.zeros((P, M, 3), self.np)
        assert dL_dmeans3D.dtype == self.np and dL_dmeans3D.flags.c_contiguous
        self._fn("oracle_sh_backward")(C.c_int(P), C.c_int(deg), C.c_int(M), _p(m3), _p(cp), _p(shs), _p(cl), _p(g), _p(dsh),
                                       _p(dL_dmeans3D))
        return dsh

    def forward(self, means3D, colors, opacity, scales, rots, view, proj, tanfovx, tanfovy, W, H, bg,
                scale_mod=1.0, cov3D_precomp=None, nthreads=1, render=True):
        """view/proj: the 4x4 tensors exactly as the reference passes them (row-vector convention,
        i.e. flat[c*4+r] = maths M(r,c)); flattened row-major here."""
        P = int(np.asarray(means3D).reshape(-1, 3).shape[0])
        r = self.np
        m3 = self._a(means3D, (P, 3)); col = self._a(colors, (P, 3)); op = self._a(opacity, (P,))
        sc = self._a(scales, (P, 3)) if scales is not None else None
        ro = self._a(rots, (P, 4)) if rots is not None else None
        cp = self._a(cov3D_precomp, (P, 6)) if cov3D_precomp is not None else None
        vm = self._a(view, (16,)); pm = self._a(proj, (16,)); bgc = self._a(bg, (3,))
        st = dict(P=P, W=W, H=H)
        st["radii"] = np.zeros(P, np.int32); st["means2D"] = np.zeros((P, 2), r); st["depth"] = np.zeros(P, r)
        st["cov3D"] = np.zeros((P, 6), r); st["conic_opacity"] = np.zeros((P, 4), r)
        st["tiles_touched"] = np.zeros(P, np.uint32); st["rects"] = np.zeros((P, 4), np.int32)
        f = self._fn("oracle_preprocess"); f.restype = C.c_int
        cr = self.creal
        st["n_visible"] = f(C.c_int(P), C.c_int(W), C.c_int(H), _p(m3), _p(sc), _p(ro), _p(op), _p(cp), cr(scale_mod),
                            _p(vm), _p(pm), cr(tanfovx), cr(tanfovy), _p(st["radii"]), _p(st["means2D"]),
                            _p(st["depth"]), _p(st["cov3D"]), _p(st["conic_opacity"]), _p(st["tiles_touched"]),
                            _p(st["rects"]))
        N = int(st["tiles_touched"].astype(np.int64).sum())
        gx, gy = (W + 15) // 16, (H + 15) // 16
        st["keys"] = np.zeros(max(N, 1), np.uint64)[:N]; st["vals"] = np.zeros(max(N, 1), np.uint32)[:N]
        st["ranges"] = np.zeros((gx * gy, 2), np.uint32)
        depth32 = np.ascontiguousarray(st["depth"].astype(np.float32))
        keys = np.zeros(max(N, 1), np.uint64); vals = np.zeros(max(N, 1), np.uint32)
        f = self._fn("oracle_bin"); f.restype = C.c_int64
        n = f(C.c_int(P), C.c_int(W), C.c_int(H), _p(st["radii"]), _p(st["rects"]), _p(depth32), _p(keys), _p(vals),
              _p(st["ranges"]))
        assert n == N, (n, N)
        st["keys"], st["vals"], st["num_rendered"] = keys[:N], vals[:N], N
        st["_vals_full"] = vals
        st["inputs"] = dict(means3D=m3, colors=col, opacity=op, scales=sc, rots=ro, cov3D_precomp=cp, view=vm, proj=pm,
                            tanfovx=tanfovx, tanfovy=tanfovy, bg=bgc, scale_mod=scale_mod)
        if render:
            st["color"] = np.zeros((3, H, W), r); st["final_T"] = np.zeros((H, W), r)
            st["n_contrib"] = np.zeros((H, W), np.uint32)
            self._fn("oracle_render")(C.c_int(W), C.c_int(H), _p(st["ranges"]), _p(vals), _p(st["means2D"]), _p(col),
                                      _p(st["conic_opacity"]), _p(bgc), _p(st["color"]), _p(st["final_T"]),
                                      _p(st["n_contrib"]), C.c_int(nthreads))
        return st

    def render_state(self, st, nthreads=1):
        """A.4 compositing in THIS oracle's precision on the per-Gaussian state (means2D, conic_opacity, colours, tile
        lists) of a forward done in any precision -- isolates the compositing arithmetic from the projection's."""
        W, H = st["W"], st["H"]
        r = self.np
        i = st["inputs"]
        m2 = self._a(st["means2D"]); co = self._a(st["conic_opacity"]); col = self._a(i["colors"]); bg = self._a(i["bg"])
        out = dict(color=np.zeros((3, H, W), r), final_T=np.zeros((H, W), r), n_contrib=np.zeros((H, W), np.uint32))
        self._fn("oracle_render")(C.c_int(W), C.c_int(H), _p(st["ranges"]), _p(st["_vals_full"]), _p(m2), _p(col), _p(co),
                                  _p(bg), _p(out["color"]), _p(out["final_T"]), _p(out["n_contrib"]), C.c_int(nthreads))
        return out

    # rounding-distance thresholds of the three hard decisions of A.4 (see oracle_render_margins in gpsg_oracle.c):
    # relative on alpha vs 1/255 and test_T vs 1e-4, absolute on power vs 0.
    EPS = dict(alpha=2e-5, T=2e-3, power=1e-5)

    def margins(self, st, eps=None, nthreads=1):
        """Per-pixel distance of the closest hard decision to its threshold, the `near` mask (a decision within eps:
        the pixel may legitimately differ between two correct implementations) and the per-Gaussian `taint` flag
        (evaluated by a `near` pixel: its gradient may legitimately differ; `taint_own`: its own alpha/power is the near one)."""
        eps = dict(self.EPS, **(eps or {}))
        W, H, P = st["W"], st["H"], st["P"]
        ma = np.zeros((H, W), np.float64); mt = np.zeros((H, W), np.float64); mp = np.zeros((H, W), np.float64)
        taint = np.zeros(max(P, 1), np.uint8); own = np.zeros(max(P, 1), np.uint8)
        self._fn("oracle_render_margins")(C.c_int(W), C.c_int(H), _p(st["ranges"]), _p(st["_vals_full"]), _p(st["means2D"]),
                                          _p(st["conic_opacity"]), C.c_double(eps["alpha"]), C.c_double(eps["T"]),
                                          C.c_double(eps["power"]), _p(ma), _p(mt), _p(mp), _p(taint), _p(own), C.c_int(nthreads))
        near = (ma < eps["alpha"]) | (mt < eps["T"]) | (mp < eps["power"])
        return dict(alpha=ma, T=mt, power=mp, near=near, taint=taint[:P].astype(bool), taint_own=own[:P].astype(bool), eps=eps)

    def backward(self, st, dL_dpix):
        P, W, H = st["P"], st["W"], st["H"]
        r = self.np
        i = st["inputs"]
        g = self._a(dL_dpix, (3, H, W))
        out = dict(dL_dmean2D=np.zeros((P, 2), r), dL_dconic=np.zeros((P, 3), r), dL_dopacity=np.zeros(P, r),
                   dL_dcolors=np.zeros((P, 3), r), dL_dmeans3D=np.zeros((P, 3), r), dL_dcov3D=np.zeros((P, 6), r),
                   dL_dscales=np.zeros((P, 3), r), dL_drots=np.zeros((P, 4), r))
        self._fn("oracle_render_backward")(C.c_int(P), C.c_int(W), C.c_int(H), _p(st["ranges"]), _p(st["_vals_full"]),
                                           _p(st["means2D"]), _p(i["colors"]), _p(st["conic_opacity"]), _p(i["bg"]),
                                           _p(st["final_T"]), _p(st["n_contrib"]), _p(g), _p(out["dL_dmean2D"]),
                                           _p(out["dL_dconic"]), _p(out["dL_dopacity"]), _p(out["dL_dcolors"]))
        cr = self.creal
        self._fn("oracle_preprocess_backward")(C.c_int(P), C.c_int(W), C.c_int(H), _p(i["means3D"]), _p(st["radii"]),
                                               _p(i["scales"]), _p(i["rots"]), _p(i["cov3D_precomp"]), cr(i["scale_mod"]),
                                               _p(i["view"]), _p(i["proj"]), cr(i["tanfovx"]), cr(i["tanfovy"]),
                                               _p(out["dL_dmean2D"]), _p(out["dL_dconic"]), _p(out["dL_dmeans3D"]),
                                               _p(out["dL_dcov3D"]), _p(out["dL_dscales"]), _p(out["dL_drots"]))
        return out

    def mark_visible(self, means3D, view):
        P = int(np.asarray(means3D).reshape(-1, 3).shape[0])
        m3 = self._a(means3D, (P, 3)); vm = self._a(view, (16,))
        out = np.zeros(P, np.uint8)
        self._fn("oracle_mark_visible")(C.c_int(P), _p(m3), _p(vm), _p(out))
        return out.astype(bool)


def taichi_splat(pts, mask, res, dtype="f32"):
    """Restated reference lib/TaichiRender.py:12-23 (one call = one view's points). Returns (depth, color)."""
    o = RasterOracle(dtype)
    pts = o._a(pts); B, N = pts.shape[0], pts.shape[1]
    mask = o._a(mask, (B, N))
    depth = np.zeros((B, 1, res, res), o.np); color = np.full((B, 3, res, res), -1.0, o.np)
    o._fn("oracle_taichi_splat")(C.c_int(B), C.c_int(N), C.c_int(res), _p(pts), _p(mask), _p(depth), _p(color))
    return depth, color
