"""CPU: host-side logic and the C-ABI boundary (no compute calls -- there is no GPU here)."""
import ctypes as C
import os
import re

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_library_exports_every_declared_symbol(built_lib):
    hdr = open(os.path.join(ROOT, "include", "gpsg.h")).read()
    declared = set(re.findall(r"GPSG_API\s+[\w\s\*]+?\b(gpsg_\w+)\s*\(", hdr))
    assert len(declared) >= 11
    lib = C.CDLL(built_lib)
    for name in declared:
        assert hasattr(lib, name), name
    from gps_gaussian_b200 import _lib
    assert set(_lib.EXPORTED) == declared
    assert _lib.lib.gpsg_version() == 90


def test_settings_struct_layout_matches_header(built_lib):
    from gps_gaussian_b200 import _lib
    # 2 ints + 2 floats + 3 + 1 + 16 + 16 floats + int + 3 floats + 2 ints = 46 4-byte fields
    assert C.sizeof(_lib.RasterSettings) == 46 * 4
    assert _lib.RasterSettings.viewmatrix.offset == 8 * 4 and _lib.RasterSettings.campos.offset == 41 * 4


def test_argument_validation_without_gpu(built_lib):
    """Error paths return codes + messages and never touch the device."""
    from gps_gaussian_b200 import _lib
    s = _lib.RasterSettings()
    s.image_height, s.image_width = 0, 16
    n = C.c_int32(0)
    rc = _lib.lib.gpsg_rasterize_forward(C.byref(s), 0, None, 0, 0, None, None, None, None, None, None, None, None, None,
                                         _lib.ALLOC_CB, None, _lib.ALLOC_CB, None, _lib.ALLOC_CB, None, C.byref(n))
    assert rc == -1 and b"image size" in _lib.lib.gpsg_last_error()
    with pytest.raises(_lib.GpsgError):
        _lib.check(rc, "x")
    assert _lib.lib.gpsg_corr_sampler_forward(0, None, 7, 1, 1, 1, 1, None, 0, 0, 0, None, 0, 4, None) == -1
    assert _lib.lib.gpsg_corr_sampler_forward(0, None, 0, 0, 4, 4, 4, None, 0, 0, 0, None, 0, 4, None) == 0   # empty batch: no-op
    assert _lib.lib.gpsg_rasterize_backward_workspace_bytes(1000) >= 16000
    # the newer rows: shape / pointer validation happens before any CUDA call
    assert _lib.lib.gpsg_l1_ssim_forward(0, None, 0, 8, 8, None, None, 0.8, 0.2, None, None, None) == -1
    assert b"empty image" in _lib.lib.gpsg_last_error()
    assert _lib.lib.gpsg_l1_ssim_workspace_bytes(3, 1024, 1024) >= 2 * 8 * 3 * 32 * 32
    assert _lib.lib.gpsg_corr_build_backward(0, None, 5, 1, 16, 1, 8, 16, None, None, None, None, None) == -1
    assert _lib.lib.gpsg_corr_build_backward(0, None, 1, 0, 16, 1, 8, 16, None, None, None, None, None) == 0   # empty batch
    assert _lib.lib.gpsg_unproject_forward(0, None, 0, 16, None, None, 0, None, None, 3, None, None, None, None, None) == 0
    s.image_height = 16
    pp = (C.c_void_p * 2)()
    rc = _lib.lib.gpsg_rasterize_forward_maps_planned(C.byref(s), 0, None, 0, pp, pp, pp, pp, pp, pp, None, None, None, None,
                                                      1, None, None)
    assert rc == -1 and b"pixels per view" in _lib.lib.gpsg_last_error()


def test_dropin_api_surface(built_lib):
    import diff_gaussian_rasterization as dgr
    import corr_sampler
    assert dgr.GaussianRasterizationSettings._fields == (
        "image_height", "image_width", "tanfovx", "tanfovy", "bg", "scale_modifier", "viewmatrix", "projmatrix",
        "sh_degree", "campos", "prefiltered", "debug")                      # reference gaussian_renderer/__init__.py:36-49
    rs = dgr.GaussianRasterizationSettings(image_height=16, image_width=16, tanfovx=1.0, tanfovy=1.0,
                                           bg=torch.zeros(3), scale_modifier=1.0, viewmatrix=torch.eye(4),
                                           projmatrix=torch.eye(4), sh_degree=3, campos=torch.zeros(3),
                                           prefiltered=False, debug=False)
    r = dgr.GaussianRasterizer(raster_settings=rs)
    x = torch.zeros(4, 3)
    with pytest.raises(Exception, match="SHs or precomputed colors"):
        r(means3D=x, means2D=x, opacities=x[:, :1], shs=None, colors_precomp=None, scales=x, rotations=torch.zeros(4, 4))
    with pytest.raises(Exception, match="scale/rotation pair or precomputed 3D covariance"):
        r(means3D=x, means2D=x, opacities=x[:, :1], colors_precomp=x, scales=x, rotations=None, cov3D_precomp=None)
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        r(means3D=x, means2D=x, opacities=x[:, :1], colors_precomp=x, scales=x, rotations=torch.zeros(4, 4))
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        corr_sampler.forward(torch.zeros(1, 2, 3, 4), torch.zeros(1, 1, 2, 3), 4)
    s = dgr._pack_settings(rs._replace(viewmatrix=torch.arange(16.).reshape(4, 4), campos=torch.tensor([1., 2., 3.])))
    assert list(s.viewmatrix) == list(range(16)) and list(s.campos) == [1, 2, 3] and s.sh_degree == 3


def test_mirrored_interface_names():
    from gps_gaussian_b200 import GaussianRender, corr, gaussian_renderer
    import inspect
    assert list(inspect.signature(gaussian_renderer.render).parameters) == [
        "data", "idx", "pts_xyz", "pts_rgb", "rotations", "scales", "opacity", "bg_color"]   # gaussian_renderer/__init__.py:17
    assert list(inspect.signature(GaussianRender.pts2render).parameters) == ["data", "bg_color"]  # lib/GaussianRender.py:5
    sig = inspect.signature(corr.CorrBlockFast1D.__init__).parameters
    assert list(sig) == ["self", "fmap1", "fmap2", "num_levels", "radius"] and sig["radius"].default == 4
    assert hasattr(corr, "CorrSampler")
    from gps_gaussian_b200 import loss, novel_calib, shard, unproject
    assert list(inspect.signature(novel_calib.get_novel_calib).parameters) == ["data", "opt", "ratio", "intr_key", "extr_key"]  # lib/utils.py:8
    assert list(inspect.signature(loss.ssim).parameters) == ["img1", "img2", "window_size", "size_average"]   # lib/loss.py:52
    assert list(inspect.signature(loss.l1_loss).parameters) == ["network_output", "gt"]                          # lib/loss.py:35
    assert hasattr(unproject, "flow2xyz")
    info = shard.bind_host_to_gpu(0)            # no NVML here: must degrade to a no-op description, never raise
    assert isinstance(info, dict) and "bound" in info
    shard.unbind_host()


def test_synth_matches_reference_conventions():
    """Shapes / ranges of the synthetic C2 unit (reference lib/gs_parm_network.py:72-78, lib/utils.py:36-41)."""
    from gps_gaussian_b200 import synth
    sc = synth.stereo_pair_scene(256)
    P = sc["means3D"].shape[0]
    assert 0.15 * 2 * 256 * 256 < P < 0.30 * 2 * 256 * 256
    assert np.allclose(np.linalg.norm(sc["rots"], axis=1), 1, atol=1e-5)
    assert sc["scales"].max() <= 0.01 + 1e-9 and sc["opacity"].min() >= 0.2 and 0 <= sc["colors"].min()
    v = sc["view"]                                                  # W2V^T: last COLUMN is (0,0,0,1)
    assert np.allclose(v[:, 3], [0, 0, 0, 1], atol=1e-6)
    hom = np.concatenate([sc["means3D"][:100], np.ones((100, 1), np.float32)], 1)
    assert np.allclose((hom @ sc["proj"])[:, 3], (hom @ v)[:, 2], atol=1e-5)   # clip-space w == view-space depth (P[3,2] = 1)
    assert ((hom @ v)[:, 2] > 1.0).all()                            # the body is in front of the novel camera


def test_render_mirror_passes_what_the_rasterizer_module_would(built_lib, monkeypatch):
    """`render()` enters the autograd function directly; the arguments must equal what
    GaussianRasterizer(raster_settings)(means3D=..., means2D=..., shs=None, colors_precomp=..., ...) hands over
    (reference gaussian_renderer/__init__.py:36-62)."""
    import math
    from gps_gaussian_b200 import gaussian_renderer as gr
    import diff_gaussian_rasterization as dgr
    seen = []
    monkeypatch.setattr(dgr, "rasterize_gaussians", lambda *a: (seen.append(a), (torch.zeros(3, 4, 4), None))[1])
    P = 5
    xyz, rgb = torch.randn(P, 3, requires_grad=True), torch.rand(P, 3)
    rot, sc, op = torch.randn(P, 4), torch.rand(P, 3), torch.rand(P, 1)
    nv = {"FovX": torch.tensor([0.9, 1.1], dtype=torch.float64), "FovY": torch.tensor([0.8, 1.0], dtype=torch.float64),
          "height": torch.tensor([32, 48]), "width": torch.tensor([40, 56]),
          "world_view_transform": torch.randn(2, 4, 4), "full_proj_transform": torch.randn(2, 4, 4),
          "camera_center": torch.randn(2, 3)}
    out = gr.render({"novel_view": nv}, 1, xyz, rgb, rot, sc, op, [0.1, 0.2, 0.3])
    assert out.shape == (3, 4, 4)
    direct = seen.pop()
    rs = dgr.GaussianRasterizationSettings(image_height=48, image_width=56, tanfovx=math.tan(0.55), tanfovy=math.tan(0.5),
                                           bg=torch.tensor([0.1, 0.2, 0.3]), scale_modifier=1.0,
                                           viewmatrix=nv["world_view_transform"][1], projmatrix=nv["full_proj_transform"][1],
                                           sh_degree=3, campos=nv["camera_center"][1], prefiltered=False, debug=False)
    sink = torch.zeros_like(xyz)
    dgr.GaussianRasterizer(raster_settings=rs)(means3D=xyz, means2D=sink, shs=None, colors_precomp=rgb, opacities=op,
                                               scales=sc, rotations=rot, cov3D_precomp=None)
    via_module = seen.pop()
    assert len(direct) == len(via_module) == 9
    for k, (a, b) in enumerate(zip(direct[:8], via_module[:8])):
        assert a.shape == b.shape and a.dtype == b.dtype and torch.equal(a.detach(), b.detach()), k
    assert direct[1].requires_grad and direct[1].grad_fn is not None          # the means2D gradient sink is live
    sa, sb = dgr._pack_settings(direct[8]), dgr._pack_settings(via_module[8])
    assert bytes(sa) == bytes(sb)                                              # identical by-value camera struct
    with torch.no_grad():
        gr.render({"novel_view": nv}, 0, xyz, rgb, rot, sc, op, [0, 0, 0])
    assert not seen.pop()[1].requires_grad
