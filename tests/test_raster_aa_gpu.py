"""GPU: anti-aliasing (GPSG_FWD_ANTIALIAS) -- the device against the fp32 / fp64 oracles fed with o * rho
(tests/aa_reference.py), the discrete state against the forward without it, the mode carried by the saved state, and
every entry point and Python layer against each other."""
import numpy as np
import pytest
import torch

import helpers
import aa_reference as aar
from gps_gaussian_b200 import _lib, synth
from gps_gaussian_b200.introspect import RasterCall, make_settings
from helpers import _threads, assert_grad_parity, assert_image_parity

pytestmark = pytest.mark.gpu

SCENES = {
    "C1": lambda: synth.random_cube_scene(10_000, 256),
    "sweep-square": lambda: synth.random_cube_scene(4000, 96, seed=41, scale_mul=0.3),
    "sweep-aniso": lambda: synth.random_cube_scene(3000, 64, seed=42, width=160, height=90, focal=(150.0, 95.0),
                                                   principal=(70.0, 40.0), scale_mul=2.0),
    "scale_modifier": lambda: synth.random_cube_scene(3000, 96, seed=43, scale_modifier=0.5),
    "C2": lambda: synth.stereo_pair_scene(1024),
    "2048": lambda: synth.random_cube_scene(60_000, 2048, seed=3, scale_mul=2.0),
}


def _np(t):
    return t.detach().cpu().numpy()


def _pair(sc):
    off = RasterCall(sc)
    off.forward()
    aa = RasterCall(sc, dev_inputs=off.inp, antialiasing=True)
    aa.forward()
    torch.cuda.synchronize()
    return off, aa


def _check_forward(tag, sc):
    off, aa = _pair(sc)
    so, sa = off.state(), aa.state()
    assert torch.equal(off.radii, aa.radii) and so["num_rendered"] == sa["num_rendered"], tag
    for k in ("depths", "means2D", "tiles_touched", "keys", "point_list", "ranges"):
        if k in so:
            assert torch.equal(so[k], sa[k]), (tag, k)
    assert torch.equal(so["conic_opacity"][:, :3], sa["conic_opacity"][:, :3]), tag
    o, ref, _ = aar.aa_forward(sc, "f32", nthreads=_threads())
    vis = ref["radii"] > 0
    assert np.array_equal(_np(sa["conic_opacity"][:, 3])[vis], ref["conic_opacity"][vis, 3]), tag   # o * rho, bit for bit
    assert (_np(sa["conic_opacity"][:, 3])[vis] <= _np(so["conic_opacity"][:, 3])[vis]).all()
    assert_image_parity(tag + ":aa", _np(aa.color), _np(sa["final_T"]), _np(sa["n_contrib"]).view(np.uint32), o, ref)
    return off, aa, ref


@pytest.mark.parametrize("name", list(SCENES))
def test_aa_forward_state_and_image(name):
    _check_forward(name, SCENES[name]())


def test_aa_forward_cov3d_precomp():
    sc = synth.random_cube_scene(3000, 128, seed=5)
    _, ref = helpers.oracle_forward(sc, "f32")
    _check_forward("cov3D_precomp", dict(sc, cov3D_precomp=ref["cov3D"].copy(), scales=None, rots=None))


def _grad_check(tag, sc, aa, g, monkeypatch):
    got = aa.backward(torch.from_numpy(g).cuda(), want_cov3D=True, deterministic=False)
    got = {k: (_np(v) if v is not None else None) for k, v in got.items()}
    st = aa.state()
    base = aar.aa_forward(sc, "f32", render=False)[1]
    monkeypatch.setattr(helpers, "forced_backward", aar.aa_forced_backward)
    return assert_grad_parity(tag, sc, got, base, _np(st["final_T"]), _np(st["n_contrib"]).view(np.uint32), g)


@pytest.mark.parametrize("name", ["C1", "sweep-aniso", "scale_modifier"])
def test_aa_gradients_vs_oracle(name, monkeypatch):
    """Gradients of the device's AA backward on its own forward state against the oracle backward on o' plus the
    anti-aliasing chain, fp32 and fp64, under the clean / shared / own classes (tests/helpers.py)."""
    sc = SCENES[name]()
    aa = RasterCall(sc, antialiasing=True)
    aa.forward()
    g = np.random.default_rng(3).standard_normal((3, aa.H, aa.W)).astype(np.float32)
    _grad_check(name, sc, aa, g, monkeypatch)


def test_aa_gradients_cov3d_precomp(monkeypatch):
    sc = synth.random_cube_scene(3000, 128, seed=5)
    _, ref = helpers.oracle_forward(sc, "f32")
    sc = dict(sc, cov3D_precomp=ref["cov3D"].copy(), scales=None, rots=None)
    aa = RasterCall(sc, antialiasing=True)
    aa.forward()
    g = np.random.default_rng(4).standard_normal((3, aa.H, aa.W)).astype(np.float32)
    _grad_check("cov3D_precomp", sc, aa, g, monkeypatch)


def test_aa_deterministic_and_aux_backward():
    """DET with AA: bit-identical reruns; its gradients agree with the atomic backward; the aux backward with zero depth
    and alpha gradients equals the plain AA backward in DET mode, bit for bit; the AA gradients differ from AA-off."""
    sc = SCENES["C1"]()
    off, aa = _pair(sc)
    g = torch.from_numpy(np.random.default_rng(5).standard_normal((3, aa.H, aa.W)).astype(np.float32)).cuda()
    d1 = {k: v.clone() for k, v in aa.backward(g, deterministic=True).items() if v is not None}
    d2 = {k: v.clone() for k, v in aa.backward(g, deterministic=True).items() if v is not None}
    at = {k: v.clone() for k, v in aa.backward(g, deterministic=False).items() if v is not None}
    do = {k: v.clone() for k, v in off.backward(g, deterministic=True).items() if v is not None}
    for k in d1:
        assert torch.equal(d1[k], d2[k]), k
        assert float((d1[k] - at[k]).abs().max()) <= 1e-4 * float(d1[k].abs().max()) + 1e-12, k
    assert float((d1["dL_dopacity"] - do["dL_dopacity"]).abs().max()) > 1e-3 * float(do["dL_dopacity"].abs().max())
    # aux forward with AA, aux backward with zero depth / alpha gradients
    depth = torch.empty((aa.H, aa.W), device="cuda")
    alpha = torch.empty_like(depth)
    n, bufs = _lib.rasterize_forward(aa.settings, torch.empty_like(aa.color), torch.empty_like(aa.radii), out_depth=depth,
                                     out_alpha=alpha, antialiasing=True, **aa._inputs())
    z = torch.zeros_like(depth)
    ga = _lib.rasterize_backward(aa.settings, n, bufs, aa.radii, g, deterministic=True, grad_depth=z, grad_alpha=z,
                                 **aa._inputs())
    for k in d1:
        assert torch.equal(ga[k], d1[k]), k


def test_aa_mode_follows_state():
    """A planned AA forward and then an AA-off forward into the same buffers give AA-off gradients, and the reverse."""
    from gps_gaussian_b200.planned import PlannedRasterizer
    sc = SCENES["C1"]()
    rc = RasterCall(sc)
    i = rc._inputs()
    pr = PlannedRasterizer(rc.P, rc.H, rc.W, 1 << 20)
    g = torch.from_numpy(np.random.default_rng(6).standard_normal((3, rc.H, rc.W)).astype(np.float32)).cuda()

    def run(modes):
        for m in modes:
            pr.forward(rc.settings, i["means3D"], i["colors_precomp"], i["opacities"], i["scales"], i["rotations"],
                       antialiasing=m)
        torch.cuda.synchronize()
        assert pr.ok()
        img = pr.color.clone()
        out = _lib.rasterize_backward(rc.settings, pr.capacity, (pr.geom, pr.binning, pr.image), pr.radii, g,
                                      deterministic=False, **i)
        return img, {k: v.clone() for k, v in out.items() if v is not None}

    img_off, g_off = run([False])
    img_aa, g_aa = run([True])
    img_aa_off, g_aa_off = run([True, False])
    img_off_aa, g_off_aa = run([False, True])
    assert torch.equal(img_aa_off, img_off) and torch.equal(img_off_aa, img_aa)
    for k in g_off:
        tol = 1e-4 * float(g_off[k].abs().max()) + 1e-12
        assert float((g_aa_off[k] - g_off[k]).abs().max()) <= tol, k
        assert float((g_off_aa[k] - g_aa[k]).abs().max()) <= 1e-4 * float(g_aa[k].abs().max()) + 1e-12, k
    assert float((g_aa["dL_dopacity"] - g_off["dL_dopacity"]).abs().max()) > 1e-3 * float(g_off["dL_dopacity"].abs().max())


def test_aa_paths_bit_identical():
    """With AA: exact, planned, graph replay and the drop-in GaussianRasterizer give the same image bit for bit."""
    import diff_gaussian_rasterization as dgr
    from gps_gaussian_b200.planned import PlannedRasterizer
    sc = SCENES["C1"]()
    rc = RasterCall(sc, antialiasing=True)
    ref = rc.forward().clone()
    i = rc._inputs()
    pr = PlannedRasterizer(rc.P, rc.H, rc.W, 1 << 20)
    pr.forward(rc.settings, i["means3D"], i["colors_precomp"], i["opacities"], i["scales"], i["rotations"], antialiasing=True)
    torch.cuda.synchronize()
    assert pr.ok() and torch.equal(pr.color, ref)
    pr.color.zero_()
    pr.capture(rc.settings, i["means3D"], i["colors_precomp"], i["opacities"], i["scales"], i["rotations"], antialiasing=True)
    pr.color.zero_()
    pr.replay()
    torch.cuda.synchronize()
    assert torch.equal(pr.color, ref)
    T = lambda a: torch.tensor(np.asarray(a, np.float32), device="cuda", requires_grad=True)
    m, c, op, s, r = T(sc["means3D"]), T(sc["colors"]), T(sc["opacity"]), T(sc["scales"]), T(sc["rots"])
    rs = dgr.GaussianRasterizationSettings(
        image_height=rc.H, image_width=rc.W, tanfovx=sc["tanfovx"], tanfovy=sc["tanfovy"], bg=torch.tensor(sc["bg"]),
        scale_modifier=1.0, viewmatrix=torch.tensor(sc["view"]), projmatrix=torch.tensor(sc["proj"]), sh_degree=3,
        campos=torch.tensor(sc["campos"]), prefiltered=False, debug=False, antialiasing=True)
    img, radii = dgr.GaussianRasterizer(rs)(m, torch.zeros_like(m, requires_grad=True), op, colors_precomp=c, scales=s,
                                            rotations=r)
    assert torch.equal(img, ref) and torch.equal(radii, rc.radii)
    g = torch.from_numpy(np.random.default_rng(8).standard_normal((3, rc.H, rc.W)).astype(np.float32)).cuda()
    with torch.backends.cudnn.flags(deterministic=True):
        torch.use_deterministic_algorithms(True)
        try:
            (img * g).sum().backward()
        finally:
            torch.use_deterministic_algorithms(False)
    want = rc.backward(g, deterministic=True)
    for leaf, k in ((m, "dL_dmeans3D"), (op, "dL_dopacity"), (s, "dL_dscales"), (r, "dL_drots"), (c, "dL_dcolors")):
        assert torch.equal(leaf.grad.reshape(want[k].shape), want[k]), k
    img_aux, depth, alpha, _ = dgr.rasterize_gaussians_aux(m, torch.zeros_like(m), torch.Tensor([]), c, op, s, r,
                                                           torch.Tensor([]), rs)
    assert torch.equal(img_aux, ref) and float(alpha.max()) > 0.5


def test_aa_pts2render_and_novel_views():
    """pts2render_ex(antialiasing=True) == gather + the drop-in AA render; NovelViewRenderer(antialiasing=True) ==
    pts2render_ex per ratio in both modes (autograd through pts2render_ex: test_aa_pts2render_autograd_matches_gather_and_oracle)."""
    import diff_gaussian_rasterization as dgr
    from gps_gaussian_b200 import novel_calib
    from gps_gaussian_b200 import gaussian_renderer
    from gps_gaussian_b200.GaussianRender import pts2render, pts2render_ex, pts2render_gather
    from gps_gaussian_b200.novel_views import NovelViewRenderer, render_novel_views
    from test_novel_views import OPTS, _pair_data
    res, ratios = 128, [0.2, 0.5, 0.8]
    data = _pair_data(res, (21, 22))
    opt, bg = OPTS["plain"], [0.05, 0.1, 0.2]
    d1 = novel_calib.get_novel_calib(data, opt, ratio=0.5)
    aa_img = pts2render_ex(d1, bg, antialiasing=True)["novel_view"]["img_pred"].clone()
    off_img = pts2render(d1, bg)["novel_view"]["img_pred"].clone()
    assert not torch.equal(aa_img, off_img)
    # the gather path with the drop-in's AA settings
    orig = dgr.GaussianRasterizationSettings

    class _AA(orig):
        def __new__(cls, *a, **k):
            return orig.__new__(cls, *a, **dict(k, antialiasing=True))
    gaussian_renderer._dgr.GaussianRasterizationSettings = _AA
    try:
        g_img = pts2render_gather(d1, bg)["novel_view"]["img_pred"].clone()
    finally:
        gaussian_renderer._dgr.GaussianRasterizationSettings = orig
    assert torch.equal(g_img, aa_img)
    for mode in ("compact", "maps"):
        nvr = NovelViewRenderer(data, opt, bg, streams=2, mode=mode, antialiasing=True)
        imgs, depth, alpha = nvr.render(ratios, aux=True)
        sweep = render_novel_views(data, opt, ratios, bg, streams=2, mode=mode, antialiasing=True)["novel_view"]
        assert torch.equal(sweep["img_pred_sweep"], imgs)
        for k, ratio in enumerate(ratios):
            nv = pts2render_ex(novel_calib.get_novel_calib(data, opt, ratio=ratio), bg, aux=True,
                               antialiasing=True)["novel_view"]
            assert torch.equal(imgs[:, k], nv["img_pred"]), (mode, ratio)
            assert torch.equal(depth[:, k], nv["depth_pred"]) and torch.equal(alpha[:, k], nv["alpha_pred"]), (mode, ratio)


def test_aa_empty_scene_as_plain():
    """P = 0 through gpsg_rasterize_forward with GPSG_FWD_ANTIALIAS: the background, exactly as with flags = 0."""
    sc = synth.random_cube_scene(10, 64, seed=1, bg=(0.2, 0.4, 0.6))
    sc = dict(sc, **{k: sc[k][:0] for k in ("means3D", "colors", "opacity", "scales", "rots")})
    off, aa = _pair(sc)
    assert aa.num_rendered == 0 and torch.equal(aa.color, off.color)
    assert torch.equal(aa.color, torch.tensor(sc["bg"], device="cuda").view(3, 1, 1).expand_as(aa.color))
    g = aa.backward(torch.ones_like(aa.color), deterministic=False)
    assert g["dL_dmeans3D"].numel() == 0


def _aa_gather_settings():
    """The drop-in settings class with antialiasing=True forced, for the reference's gather -> render data flow."""
    import diff_gaussian_rasterization as dgr
    orig = dgr.GaussianRasterizationSettings

    class _AA(orig):
        def __new__(cls, *a, **k):
            return orig.__new__(cls, *a, **dict(k, antialiasing=True))
    return orig, _AA


@pytest.mark.parametrize("cam", [{}, dict(width=72, height=120, focal=(80.0, 100.0), principal=(35.0, 62.0))],
                         ids=["square", "72x120"])
def test_aa_pts2render_autograd_matches_gather_and_oracle(cam, monkeypatch):
    """Autograd through pts2render_ex(antialiasing=True) (map ingest, gradients in map layout) == autograd through the
    reference's gather -> drop-in AA render, and the map gradients gathered to the valid pixels match the oracle backward
    plus the anti-aliasing chain under the clean / shared / own classes."""
    from gps_gaussian_b200 import gaussian_renderer
    from gps_gaussian_b200.GaussianRender import pts2render_ex, pts2render_gather
    from test_raster_gpu import _stereo_data
    res = 96
    H, W = cam.get("height", res), cam.get("width", res)
    g = torch.randn(1, 3, H, W, device="cuda", generator=torch.Generator("cuda").manual_seed(3))
    keys = ("xyz", "img", "rot_maps", "scale_maps", "opacity_maps")
    orig, aa_cls = _aa_gather_settings()
    grads, outs = [], []
    for path in ("maps", "gather"):
        sc, data = _stereo_data(res, requires_grad=True, seed=4242, **cam)
        if path == "maps":
            out = pts2render_ex(data, [0.1, 0.2, 0.3], antialiasing=True)["novel_view"]["img_pred"]
        else:
            monkeypatch.setattr(gaussian_renderer._dgr, "GaussianRasterizationSettings", aa_cls)
            out = pts2render_gather(data, [0.1, 0.2, 0.3])["novel_view"]["img_pred"]
            monkeypatch.setattr(gaussian_renderer._dgr, "GaussianRasterizationSettings", orig)
        (out * g).sum().backward()
        outs.append(out.detach())
        grads.append({(v, k): data[v][k].grad for v in ("lmain", "rmain") for k in keys})
    assert torch.equal(outs[0], outs[1])
    for key in grads[0]:
        a, b = grads[0][key], grads[1][key]
        assert a is not None and b is not None and a.shape == b.shape, key
        scale = max(float(b.abs().max()), 1e-20)
        per = (a - b).abs().flatten(1).max(0).values / scale if a.dim() > 1 else (a - b).abs() / scale
        assert int((per > helpers.GRAD_TOL).sum()) <= 4 and float(per.max()) < 5e-2, (key, float(per.max()))
    # map gradients gathered into the flat Gaussian order (lmain valid pixels, then rmain) against the oracle
    sc, data = _stereo_data(res, seed=4242, **cam)
    got = {k: [] for k in ("dL_dmeans3D", "dL_dcolors", "dL_drots", "dL_dscales", "dL_dopacity")}
    for v in ("lmain", "rmain"):
        valid = data[v]["pts_valid"][0].reshape(-1).bool()
        gd = {k: grads[0][(v, k)][0] for k in keys}
        got["dL_dmeans3D"].append(gd["xyz"].reshape(-1, 3)[valid])
        got["dL_dcolors"].append(2.0 * gd["img"].reshape(3, -1).t()[valid])          # colours are img * 0.5 + 0.5
        got["dL_drots"].append(gd["rot_maps"].reshape(4, -1).t()[valid])
        got["dL_dscales"].append(gd["scale_maps"].reshape(3, -1).t()[valid])
        got["dL_dopacity"].append(gd["opacity_maps"].reshape(1, -1).t()[valid])
    got = {k: _np(torch.cat(t, 0)) for k, t in got.items()}
    sc = dict(sc, bg=np.array([0.1, 0.2, 0.3], np.float32))
    rc = RasterCall(sc, antialiasing=True)                 # the same forward: its decisions (final_T, n_contrib)
    rc.forward()
    assert torch.equal(rc.color, outs[0][0])
    st = rc.state()
    base = aar.aa_forward(sc, "f32", render=False)[1]
    monkeypatch.setattr(helpers, "forced_backward", aar.aa_forced_backward)
    assert_grad_parity("maps", sc, got, base, _np(st["final_T"]), _np(st["n_contrib"]).view(np.uint32),
                       _np(g[0]), keys=tuple((k, k) for k in got))


def test_aa_aux_backward_with_depth_and_alpha_gradients(monkeypatch):
    """The aux backward with AA and non-zero depth / alpha gradients against the fp64 aux reference of
    tests/test_raster_aux_gpu.py, whose oracle backwards are swapped for the anti-aliased ones (it is linear in them)."""
    import test_raster_aux_gpu as tax
    sc = SCENES["C1"]()
    rc = RasterCall(sc, antialiasing=True)
    depth = torch.empty((rc.H, rc.W), device="cuda")
    alpha = torch.empty_like(depth)
    rc.num_rendered, rc.bufs = _lib.rasterize_forward(rc.settings, rc.color, rc.radii, out_depth=depth, out_alpha=alpha,
                                                      antialiasing=True, **rc._inputs())
    st = rc.state()
    rng = np.random.default_rng(9)
    g_rgb = rng.standard_normal((3, rc.H, rc.W)).astype(np.float32)
    g_D = rng.standard_normal((rc.H, rc.W)).astype(np.float32)
    g_A = rng.standard_normal((rc.H, rc.W)).astype(np.float32)
    monkeypatch.setattr(tax, "forced_backward", aar.aa_forced_backward)
    base = aar.aa_forward(sc, "f32", render=False)[1]
    want, m = tax._fp64_aux_backward(sc, base, _np(st["final_T"]), _np(st["n_contrib"]).view(np.uint32), g_rgb, g_D, g_A)
    own, shared, clean = m["taint_own"], m["taint"] & ~m["taint_own"], ~m["taint"]
    cu = lambda a: torch.from_numpy(a).cuda()
    for det in (False, True):
        got = _lib.rasterize_backward(rc.settings, rc.num_rendered, rc.bufs, rc.radii, cu(g_rgb), want_cov3D=True,
                                      deterministic=det, grad_depth=cu(g_D), grad_alpha=cu(g_A), **rc._inputs())
        for kg, kr in tax.KEYS:
            a = _np(got[kg])
            if kg == "dL_dmeans2D":
                a = a[:, :2]
            per = helpers.grad_err(a, want[kr])
            mx = lambda msk: float(per[msk].max()) if msk.any() else 0.0
            assert mx(clean) <= helpers.GRAD_TOL and mx(shared) <= helpers.SHARED_TOL and mx(own) <= helpers.TAINT_CAP, \
                (det, kg, mx(clean), mx(shared), mx(own))


_RADIX_SCRIPT = r"""
import os, sys
sys.path[:0] = [{root!r}, os.path.join({root!r}, "gps-gaussian_b200", "dropin")]
import numpy as np, torch
from gps_gaussian_b200 import synth
from gps_gaussian_b200.introspect import RasterCall
for name, sc in (("c1", synth.random_cube_scene(10_000, 256)),
                 ("long-tiles", synth.random_cube_scene(30000, 48, spread=0.25, scale_mul=1.0, seed=13))):
    rc = RasterCall(sc, antialiasing=True); rc.forward()
    np.save(os.path.join({out!r}, f"{{name}}_color.npy"), rc.color.cpu().numpy())
    g = torch.from_numpy(np.random.default_rng(7).standard_normal((3, sc["H"], sc["W"])).astype(np.float32)).cuda()
    for k, v in rc.backward(g, want_cov3D=True, deterministic=True).items():
        if v is not None:
            np.save(os.path.join({out!r}, f"{{name}}_{{k}}.npy"), v.cpu().numpy())
"""


def test_aa_radix_binning_path_bit_identical(tmp_path):
    """With AA, the global radix binning (GPSG_BINNING=radix, read once per process: a subprocess each) gives the same
    image and bit-identical deterministic gradients as the tile-bucket path; the bucket path is held to the oracle above."""
    import os
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    outs = {}
    for mode in ("bucket", "radix"):
        d = tmp_path / mode
        d.mkdir()
        env = dict(os.environ)
        env.pop("GPSG_BINNING", None)
        if mode == "radix":
            env["GPSG_BINNING"] = "radix"
        r = subprocess.run([sys.executable, "-c", _RADIX_SCRIPT.format(root=root, out=str(d))], env=env, cwd=root,
                           capture_output=True, text=True, timeout=600)
        assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-3000:]
        outs[mode] = {f.name: np.load(f) for f in sorted(d.iterdir())}
    assert len(outs["bucket"]) >= 14 and outs["bucket"].keys() == outs["radix"].keys()
    for name in outs["bucket"]:
        assert np.array_equal(outs["bucket"][name].view(np.uint32), outs["radix"][name].view(np.uint32)), name
