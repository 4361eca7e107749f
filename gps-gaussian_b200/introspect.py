"""Direct C-ABI driver that also exposes the saved rasterizer state (depths, means2D, conics,
tiles_touched, sorted keys / point list, tile ranges, final_T, n_contrib) as torch tensors.
Used by the parity tests ("tile indices bit-exact") and by bench.py; not on the training path."""
import ctypes as C

import numpy as np
import torch

from . import _lib


def _sub(buf, ptr, nbytes, dtype):
    off = int(ptr) - buf.data_ptr()
    assert 0 <= off and off + nbytes <= buf.numel(), (off, nbytes, buf.numel())
    return buf[off:off + nbytes].view(dtype)


def make_settings(sc, debug=False):
    s = _lib.RasterSettings()
    s.image_height, s.image_width = int(sc["H"]), int(sc["W"])
    s.tanfovx, s.tanfovy = float(sc["tanfovx"]), float(sc["tanfovy"])
    s.bg[:] = [float(v) for v in np.asarray(sc["bg"]).reshape(3)]
    s.scale_modifier = float(sc.get("scale_modifier", 1.0))
    s.viewmatrix[:] = [float(v) for v in np.asarray(sc["view"], np.float32).reshape(16)]
    s.projmatrix[:] = [float(v) for v in np.asarray(sc["proj"], np.float32).reshape(16)]
    s.sh_degree = 3
    s.campos[:] = [float(v) for v in np.asarray(sc["campos"], np.float32).reshape(3)]
    s.prefiltered, s.debug = 0, int(debug)
    return s


def to_device(sc, device="cuda"):
    """numpy scene dict (synth.py) -> dict of contiguous fp32 CUDA tensors for the five per-Gaussian inputs."""
    t = lambda k: torch.from_numpy(np.ascontiguousarray(sc[k], np.float32)).to(device) if sc.get(k) is not None else None
    return dict(means3D=t("means3D"), colors=t("colors"), opacity=t("opacity"), scales=t("scales"), rots=t("rots"),
                cov3D_precomp=t("cov3D_precomp"))


class RasterCall:
    """One forward (and optionally backward) through gpsg_rasterize_* with raw tensors."""

    def __init__(self, sc, dev_inputs=None, device="cuda", antialiasing=False):
        self.sc = sc
        self.antialiasing = bool(antialiasing)      # forward mode; the backward follows the saved state
        self.device = torch.device(device)
        self.inp = dev_inputs if dev_inputs is not None else to_device(sc, device)
        self.settings = make_settings(sc)
        self.P = int(self.inp["means3D"].shape[0])
        self.H, self.W = int(sc["H"]), int(sc["W"])
        self.color = torch.empty((3, self.H, self.W), dtype=torch.float32, device=self.device)
        self.radii = torch.empty((self.P,), dtype=torch.int32, device=self.device)
        self.num_rendered = 0
        self.bufs = None

    def _inputs(self):
        i = self.inp
        return dict(means3D=i["means3D"], opacities=i["opacity"], colors_precomp=i["colors"], scales=i["scales"],
                    rotations=i["rots"], cov3D_precomp=i.get("cov3D_precomp"))

    def forward(self, out_depth=None, out_alpha=None):
        """out_depth / out_alpha ([H,W], both or neither): aux mode, which also writes depth and alpha."""
        self.num_rendered, self.bufs = _lib.rasterize_forward(self.settings, self.color, self.radii, out_depth=out_depth,
                                                              out_alpha=out_alpha, antialiasing=self.antialiasing,
                                                              **self._inputs())
        return self.color

    def backward(self, grad_color, want_cov3D=False, deterministic=None, grad_depth=None, grad_alpha=None):
        """deterministic: None follows torch.use_deterministic_algorithms, True / False force it (_lib.backward_flags).
        grad_depth / grad_alpha: the aux backward (after an aux forward)."""
        return _lib.rasterize_backward(self.settings, self.num_rendered, self.bufs, self.radii, grad_color,
                                       want_cov3D=want_cov3D, deterministic=deterministic, grad_depth=grad_depth,
                                       grad_alpha=grad_alpha, **self._inputs())

    def state(self):
        """Saved buffers as torch tensors (views into the scratch buffers)."""
        geom, binning, image = self.bufs
        P, N, H, W = self.P, self.num_rendered, self.H, self.W
        tiles = ((W + 15) // 16) * ((H + 15) // 16)
        st = dict(radii=self.radii, num_rendered=N)
        gv, bv, iv = _lib.GeomView(), _lib.BinningView(), _lib.ImageView()
        _lib.check(_lib.lib.gpsg_geom_view(C.c_void_p(geom.data_ptr()), P, C.byref(gv)), "gpsg_geom_view")
        _lib.check(_lib.lib.gpsg_image_view(C.c_void_p(image.data_ptr()), W, H, C.byref(iv)), "gpsg_image_view")
        if P > 0:
            st["depths"] = _sub(geom, gv.depths, 4 * P, torch.float32)
            st["means2D"] = _sub(geom, gv.means2D, 8 * P, torch.float32).view(P, 2)
            st["conic_opacity"] = _sub(geom, gv.conic_opacity, 16 * P, torch.float32).view(P, 4)
            st["tiles_touched"] = _sub(geom, gv.tiles_touched, 4 * P, torch.int32)
            st["point_offsets"] = _sub(geom, gv.point_offsets, 4 * P, torch.int32)
        if N > 0:
            _lib.check(_lib.lib.gpsg_binning_view(C.c_void_p(binning.data_ptr()), N, C.byref(bv)), "gpsg_binning_view")
            st["keys"] = _sub(binning, bv.point_list_keys, 8 * N, torch.int64)
            st["point_list"] = _sub(binning, bv.point_list, 4 * N, torch.int32)
            st["slabA"] = _sub(binning, bv.slabA, 16 * N, torch.float32).view(N, 4)
            st["block_lists"] = _sub(binning, bv.block_lists, 32 * N, torch.int32)
        st["final_T"] = _sub(image, iv.final_T, 4 * H * W, torch.float32).view(H, W)
        st["n_contrib"] = _sub(image, iv.n_contrib, 4 * H * W, torch.int32).view(H, W)
        st["ranges"] = _sub(image, iv.ranges, 8 * tiles, torch.int32).view(tiles, 2)
        st["block_counts"] = _sub(image, iv.block_counts, 32 * tiles, torch.int32).view(tiles, 8)
        return st
