"""Sync-free rasterizer front end over `gpsg_rasterize_forward_planned` (include/gpsg.h).

`PlannedRasterizer` owns persistent scratch buffers sized for a pair capacity, so a forward is a fixed sequence of
kernel launches with no host synchronisation and no allocation: the CPU runs ahead of the GPU, and the whole
forward can be captured into a CUDA graph (`capture()` / `replay()`).  The price is a deferred check: after the
caller next synchronises, `ok()` tells whether the pairs fitted; if not, `grow()` and render again (or use the
exact, one-sync entry point behind `diff_gaussian_rasterization.GaussianRasterizer`).

This is the serving path (fixed scene size class, many views): reference test_view_interp.py:39-47 renders
`novel_view_nums` views of one pair in a loop -- with this class that loop contains no sync at all.
"""
import ctypes as C

import torch

from . import _lib
from .introspect import make_settings


def _aux_args(depth, alpha):
    """The (out_depth, out_alpha) pointer arguments of the planned entry points: (NULL, NULL) without aux outputs."""
    if (depth is None) != (alpha is None):
        raise ValueError("depth and alpha must be given together")
    return (None, None) if depth is None else (C.c_void_p(depth.data_ptr()), C.c_void_p(alpha.data_ptr()))


class PlannedRasterizer:
    def __init__(self, P, height, width, capacity_pairs, device="cuda"):
        self.dev = torch.device("cuda", _lib.device_stream(device)[0])
        self.P, self.H, self.W = int(P), int(height), int(width)
        new = lambda n: torch.empty(int(n), dtype=torch.uint8, device=self.dev)
        self.geom = new(_lib.lib.gpsg_raster_geom_bytes(self.P))
        self.image = new(_lib.lib.gpsg_raster_image_bytes(self.W, self.H))
        self.color = torch.empty((3, self.H, self.W), dtype=torch.float32, device=self.dev)
        self.radii = torch.empty((self.P,), dtype=torch.int32, device=self.dev)
        self.status_host = torch.zeros(4, dtype=torch.int32).pin_memory()
        self._alloc_binning(int(capacity_pairs))
        self.graph = None

    def _alloc_binning(self, cap):
        self.capacity = int(cap)
        self.binning = torch.empty(int(_lib.lib.gpsg_raster_binning_bytes(self.capacity)), dtype=torch.uint8, device=self.dev)

    def forward(self, settings, means3D, colors, opacity, scales, rots, cov3D_precomp=None, out=None, status_host=None,
                depth=None, alpha=None, antialiasing=False):
        """Enqueue one forward on the current stream (P = means3D.shape[0] may be smaller than the P the scratch was
        sized for; `out` / `status_host` redirect the image / deferred status words, as in forward_maps).  Inputs: contiguous fp32 CUDA tensors; `settings`: a
        `_lib.RasterSettings` (see introspect.make_settings) or a synth scene dict.  Returns self.color (valid once the
        stream has run AND ok() holds).  depth / alpha ([H,W] fp32, both or neither): aux mode, which also writes the
        expected depth and the alpha matte.  antialiasing: the opacity-compensated screen-space filter
        (GPSG_FWD_ANTIALIAS); the image buffer then carries that mode to the backward."""
        if isinstance(settings, dict):
            settings = make_settings(settings)
        p = lambda t: C.c_void_p(t.data_ptr()) if t is not None else None
        P = int(means3D.shape[0])
        if P > self.P:
            raise ValueError(f"PlannedRasterizer scratch holds P<={self.P}, got {P}")
        color = self.color if out is None else out
        aux = _aux_args(depth, alpha)
        fn = _lib.lib.gpsg_rasterize_forward_planned
        rc = fn(C.byref(settings), *_lib.device_stream(self.dev), P, p(means3D),
                p(colors), p(opacity), p(scales), p(rots), p(cov3D_precomp), p(color), *aux, p(self.radii), p(self.geom),
                p(self.binning), self.capacity, p(self.image),
                C.c_void_p((self.status_host if status_host is None else status_host).data_ptr()),
                _lib.forward_flags(antialiasing))
        _lib.check(rc, fn.__name__)
        return color

    def forward_maps(self, settings, valid, xyz, img, rot, scale, opacity, out=None, status_host=None, depth=None,
                     alpha=None, antialiasing=False):
        """Same, reading the two source views' pixel-aligned maps in place (`gpsg_rasterize_forward_maps_planned`):
        each argument is a pair (lmain, rmain) of contiguous CUDA tensors -- valid uint8/bool [S2], xyz [S2,3], img
        [3,S2] in [-1,1], rot [4,S2], scale [3,S2], opacity [1,S2]; self.P must be 2*S2.  `out` optionally redirects
        the image to another [3,H,W] tensor (e.g. a slice of a batch); `status_host` optionally redirects the deferred
        status words to another pinned int32[>=3] tensor (one per in-flight job).  depth / alpha, antialiasing: as in
        forward."""
        S2 = int(valid[0].numel())
        if 2 * S2 != self.P:
            raise ValueError(f"PlannedRasterizer built for P={self.P}, maps hold 2*{S2} candidates")
        pp = lambda ts: (C.c_void_p * 2)(*[t.data_ptr() for t in ts])
        color = self.color if out is None else out
        aux = _aux_args(depth, alpha)
        fn = _lib.lib.gpsg_rasterize_forward_maps_planned
        rc = fn(C.byref(settings), *_lib.device_stream(self.dev), S2, pp(valid), pp(xyz),
                pp(img), pp(rot), pp(scale), pp(opacity), C.c_void_p(color.data_ptr()), *aux,
                C.c_void_p(self.radii.data_ptr()), C.c_void_p(self.geom.data_ptr()), C.c_void_p(self.binning.data_ptr()),
                self.capacity, C.c_void_p(self.image.data_ptr()),
                C.c_void_p((self.status_host if status_host is None else status_host).data_ptr()),
                _lib.forward_flags(antialiasing))
        _lib.check(rc, fn.__name__)
        return color

    # ---- deferred status (call after a synchronisation that covers the forward) ----
    def status(self):
        n, mx, ov, _ = (int(v) for v in self.status_host.tolist())
        return dict(num_rendered=n, max_tile=mx, overflow=bool(ov))

    def ok(self):
        return not self.status()["overflow"]

    def grow(self, factor=1.5, needed_pairs=None):
        """Re-allocate the binning buffer.  `needed_pairs`: the pair count a failed job reported (its status words may
        live in a caller-provided slot rather than self.status_host): the new capacity is sized from it directly."""
        need = int(needed_pairs) if needed_pairs is not None else self.status()["num_rendered"]
        self._alloc_binning(max(int(need * 1.05) + 1024, int(self.capacity * factor)) if need > self.capacity
                            else int(self.capacity * factor))
        self.graph = None

    # ---- CUDA graph ----
    def capture(self, settings, means3D, colors, opacity, scales, rots, cov3D_precomp=None, antialiasing=False):
        """Capture one forward (fixed input pointers / camera / mode) into a CUDA graph; replay() re-runs it."""
        if isinstance(settings, dict):
            settings = make_settings(settings)
        self._keep = (settings, means3D, colors, opacity, scales, rots, cov3D_precomp)
        s = torch.cuda.Stream(self.dev)
        s.wait_stream(torch.cuda.current_stream(self.dev))
        with torch.cuda.stream(s):
            self.forward(*self._keep, antialiasing=antialiasing)   # warm-up outside capture (lazy module loads etc.)
        torch.cuda.current_stream(self.dev).wait_stream(s)
        torch.cuda.synchronize(self.dev)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            self.forward(*self._keep, antialiasing=antialiasing)
        self.graph = g
        return g

    def replay(self):
        self.graph.replay()
        return self.color
