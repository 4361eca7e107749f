"""CPU: anti-aliasing (GPSG_FWD_ANTIALIAS) -- the C ABI's argument checks, closed forms of the filter, the reference the
GPU tests hold the device to (tests/aa_reference.py) against fp64 autograd, and the Python switches.  No call here
reaches the device."""
import ctypes as C
import math
import os
import re
import sys
import types

import numpy as np
import pytest
import torch

from gps_gaussian_b200 import synth
from helpers import oracle_forward, record
import aa_reference as aar

AA = 1
FWD_FLAGS = ("gpsg_rasterize_forward", "gpsg_rasterize_forward_maps_begin", "gpsg_rasterize_forward_planned",
             "gpsg_rasterize_forward_maps_planned")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_aa_symbols_exported(built_lib):
    from gps_gaussian_b200 import _lib
    hdr = open(os.path.join(ROOT, "include", "gpsg.h")).read()
    assert "#define GPSG_FWD_ANTIALIAS 1" in hdr and _lib.FWD_ANTIALIAS == 1
    for name in FWD_FLAGS:
        assert name in _lib.EXPORTED and hasattr(_lib.lib, name)
        assert re.search(r"GPSG_API int %s\(" % name, hdr)
    assert _lib.lib.gpsg_version() == 90
    assert _lib.forward_flags(True) == 1 and _lib.forward_flags(False) == 0


def _calls(L, s, p, pp, flags):
    alloc = _lib_alloc()
    return {
        "gpsg_rasterize_forward": lambda: L.gpsg_rasterize_forward(s, 0, None, 4, 0, p, p, None, p, p, p, None, p, None,
                                                                   None, p, alloc, None, alloc, None, alloc, None, None,
                                                                   flags),
        "gpsg_rasterize_forward_maps_begin": lambda: L.gpsg_rasterize_forward_maps_begin(
            s, 0, None, 4, *([pp] * 6), p, alloc, None, alloc, None, p, flags),
        "gpsg_rasterize_forward_planned": lambda: L.gpsg_rasterize_forward_planned(
            s, 0, None, 4, p, p, p, p, p, None, p, None, None, p, p, p, 16, p, None, flags),
        "gpsg_rasterize_forward_maps_planned": lambda: L.gpsg_rasterize_forward_maps_planned(
            s, 0, None, 4, *([pp] * 6), p, None, None, p, p, p, 16, p, None, flags),
    }


def _lib_alloc():
    from gps_gaussian_b200 import _lib
    return _lib.ALLOC_CB


def test_aa_unknown_forward_flags_refused_first(built_lib):
    """Every forward that takes flags refuses unknown bits before checking anything else (NULL settings included)."""
    from gps_gaussian_b200 import _lib
    L = _lib.lib
    buf = (C.c_float * 1024)()
    p = C.cast(buf, C.c_void_p)
    pp = (C.c_void_p * 2)(p, p)
    for flags in (2, 4, 1 | 8, -1):
        for name, call in _calls(L, None, p, pp, flags).items():
            assert call() == -1, name
            assert b"flag" in L.gpsg_last_error(), (name, L.gpsg_last_error())


def test_aa_null_and_empty_as_plain(built_lib):
    """With GPSG_FWD_ANTIALIAS the argument checks are those of flags = 0 (same codes, same messages)."""
    from gps_gaussian_b200 import _lib
    L = _lib.lib
    buf = (C.c_float * 1024)()
    p = C.cast(buf, C.c_void_p)
    pp = (C.c_void_p * 2)(p, p)
    s = _lib.RasterSettings()
    s.image_height, s.image_width = 16, 16
    for name, call in _calls(L, None, p, pp, AA).items():      # NULL settings
        assert call() == -1, name
        assert b"settings is NULL" in L.gpsg_last_error(), name
    alloc = _lib.ALLOC_CB
    for flags in (0, AA):
        # planned forwards need P > 0; the maps forwards need pixels_per_view > 0; aux outputs both or neither
        assert L.gpsg_rasterize_forward_planned(C.byref(s), 0, None, 0, p, p, p, p, p, None, p, None, None, p, p, p, 16,
                                                p, None, flags) == -1
        assert b"P > 0" in L.gpsg_last_error()
        assert L.gpsg_rasterize_forward_maps_planned(C.byref(s), 0, None, 0, *([pp] * 6), p, None, None, p, p, p, 16, p,
                                                     None, flags) == -1
        assert b"pixels per view" in L.gpsg_last_error()
        assert L.gpsg_rasterize_forward_maps_begin(C.byref(s), 0, None, 0, *([pp] * 6), p, alloc, None, alloc, None, p,
                                                   flags) == -1
        assert b"pixels per view" in L.gpsg_last_error()
        assert L.gpsg_rasterize_forward(C.byref(s), 0, None, 4, 0, p, p, None, p, p, p, None, p, p, None, p, alloc, None,
                                        alloc, None, alloc, None, None, flags) == -1
        assert b"out_depth and out_alpha" in L.gpsg_last_error()
        assert L.gpsg_rasterize_forward(C.byref(s), 0, None, -1, 0, *([None] * 7), p, None, None, None, alloc, None,
                                        alloc, None, alloc, None, None, flags) == -1
        assert b"P < 0" in L.gpsg_last_error()


# ---- closed forms on the fp64 oracle fed with o * rho -------------------------------------------------------------
def _single(res, sigma_px, opacity, z=2.0, aniso=None):
    """One Gaussian on the optical axis of a square res x res camera, world scale chosen so that its screen standard
    deviation is sigma_px (isotropic) -- or scales `aniso` (3 world-space values) with a tilted rotation."""
    sc = synth.random_cube_scene(1, res, seed=3)
    view = np.asarray(sc["view"], np.float64).reshape(4, 4)
    pw = np.array([0.0, 0.0, z, 1.0]) @ np.linalg.inv(view)
    fx = res / (2.0 * sc["tanfovx"])
    if aniso is None:
        scales = np.full((1, 3), sigma_px * z / fx)
        rots = np.array([[1.0, 0.0, 0.0, 0.0]])
    else:
        scales = np.asarray(aniso, np.float64).reshape(1, 3)
        q = np.array([0.9, 0.3, -0.2, 0.25])
        rots = (q / np.linalg.norm(q)).reshape(1, 4)
    return dict(sc, means3D=pw[None, :3].astype(np.float32), scales=scales.astype(np.float32),
                rots=rots.astype(np.float32), opacity=np.full((1, 1), opacity, np.float32),
                colors=np.ones((1, 3), np.float32), bg=np.zeros(3, np.float32)), fx


def _screen_cov64(sc):
    """The pre-dilation screen covariance [2,2] of Gaussian 0, written as J W Sigma W^T J^T in fp64 matrix form."""
    view = np.asarray(sc["view"], np.float64).reshape(4, 4)
    t = np.append(np.asarray(sc["means3D"], np.float64)[0], 1.0) @ view
    fx = sc["W"] / (2.0 * sc["tanfovx"])
    fy = sc["H"] / (2.0 * sc["tanfovy"])
    J = np.array([[fx / t[2], 0, -fx * t[0] / t[2] ** 2], [0, fy / t[2], -fy * t[1] / t[2] ** 2]])
    q = np.asarray(sc["rots"], np.float64)[0]
    r, x, y, z = q
    R = np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - r * z), 2 * (x * z + r * y)],
                  [2 * (x * y + r * z), 1 - 2 * (x * x + z * z), 2 * (y * z - r * x)],
                  [2 * (x * z - r * y), 2 * (y * z + r * x), 1 - 2 * (x * x + y * y)]])
    Sg = R @ np.diag(np.asarray(sc["scales"], np.float64)[0] ** 2) @ R.T
    Wr = view[:3, :3].T
    return J @ Wr @ Sg @ Wr.T @ J.T


@pytest.mark.parametrize("sigma", [0.15, 0.5, 1.0, 2.5])
def test_aa_isotropic_closed_form(sigma):
    """On-axis isotropic splat: alpha = min(0.99, o s^2 / (s^2 + 0.3)) exp(-r^2 / (2 (s^2 + 0.3))) -- the profile is the
    dilated one, only the amplitude changes."""
    res = 65                                          # odd: the projected centre is pixel 32
    sc, fx = _single(res, sigma, 0.8)
    o, st, r = aar.aa_forward(sc, "f64")
    S = _screen_cov64(sc)
    s2 = float(S[0, 0])
    assert abs(s2 - sigma ** 2) < 1e-5 * sigma ** 2 and abs(S[1, 1] - s2) < 1e-6 * s2 and abs(S[0, 1]) < 1e-6 * s2
    k03 = float(np.float32(0.3))                     # the dilation as the kernel writes it (0.3f)
    assert r[0] == pytest.approx(s2 / (s2 + k03), rel=1e-5)
    m = np.asarray(st["means2D"])[0]
    yy, xx = np.mgrid[0:res, 0:res]
    d2 = (xx - m[0]) ** 2 + (yy - m[1]) ** 2
    want = np.minimum(0.99, float(np.float32(0.8)) * s2 / (s2 + k03) * np.exp(-d2 / (2 * (s2 + k03))))
    got = st["color"][0]
    on = want >= 1.0 / 255 * 1.0001
    assert np.abs(got[on] - want[on]).max() < 1e-5 * want.max()
    assert (got[want < 1.0 / 255 * 0.9999] == 0).all()
    # without the filter the same splat has amplitude o
    _, st0 = oracle_forward(sc, "f64")
    centre = st0["color"][0][int(round(m[1])), int(round(m[0]))]
    assert centre == pytest.approx(min(0.99, float(np.float32(0.8)) * math.exp(-d2.min() / (2 * (s2 + k03)))), rel=1e-6)


def test_aa_anisotropic_rho():
    """Anisotropic tilted splat: rho = sqrt(det S / det(S + 0.3 I)) of its screen covariance S, in fp64 and fp32."""
    sc, _ = _single(64, None, 0.7, aniso=(0.004, 0.0007, 0.002))
    S = _screen_cov64(sc)
    want = math.sqrt(np.linalg.det(S) / np.linalg.det(S + float(np.float32(0.3)) * np.eye(2)))
    _, st, r = aar.aa_forward(sc, "f64")
    assert 0.005 < want < 0.9
    assert r[0] == pytest.approx(want, rel=1e-6)
    assert st["conic_opacity"][0, 3] == pytest.approx(float(np.float32(0.7)) * want, rel=1e-6)
    _, st32, r32 = aar.aa_forward(sc, "f32")
    assert r32[0] == pytest.approx(want, rel=1e-4)
    assert st32["conic_opacity"][0, 3] == np.float32(np.float32(0.7) * r32[0])


@pytest.mark.parametrize("sigma", [0.2, 0.35, 0.7, 1.5, 4.0])
def test_aa_integrated_alpha(sigma):
    """Integrated alpha of an isolated faint splat: o 2 pi sqrt(det S) with the filter, o 2 pi sqrt(det(S + 0.3 I))
    without.  Two departures are bounded separately.  Sampling: the pixel sum of the whole Gaussian of variance
    s'^2 = s^2 + 0.3 differs from its integral by at most 4 exp(-2 pi^2 s'^2) relatively (Poisson summation).  The 1/255
    cut: the rendered sum is the pixel sum minus exactly the pixels whose alpha is below 1/255; in the continuum that mass
    is 1/255 of 2 pi s'^2 (a 2-D Gaussian has a fraction t of its mass below t times its peak), and on the grid it is
    held to twice that (pixels outside the splat's tile rectangle, 3 sigma', count as cut too)."""
    res = 129
    o_in = float(np.float32(0.9))
    sc, _ = _single(res, sigma, o_in)
    s2 = float(_screen_cov64(sc)[0, 0])
    sd2 = s2 + float(np.float32(0.3))
    for aa in (True, False):
        if aa:
            _, st, _ = aar.aa_forward(sc, "f64")
            want = o_in * 2 * math.pi * s2
        else:
            _, st = oracle_forward(sc, "f64")
            want = o_in * 2 * math.pi * sd2
        peak = want / (2 * math.pi * sd2)
        assert 1 / 255 < peak < 0.99
        m = np.asarray(st["means2D"])[0]
        yy, xx = np.mgrid[0:res, 0:res]
        prof = peak * np.exp(-((xx - m[0]) ** 2 + (yy - m[1]) ** 2) / (2 * sd2))
        full = float(prof.sum())
        x0, y0, x1, y1 = (int(v) * 16 for v in st["rects"][0])          # the tiles it is binned into
        inside = (xx >= x0) & (xx < x1) & (yy >= y0) & (yy < y1)
        cut = float(prof[(prof < 1 / 255) | ~inside].sum())
        samp = 4 * math.exp(-2 * math.pi ** 2 * sd2) * want
        got = float(st["color"][0].sum())
        record("aa:integrated_alpha", sigma=sigma, aa=aa, got=got, want=want, cut=cut, sampling_bound=samp)
        assert abs(full - want) <= samp + 1e-12 * want, (sigma, aa, full, want)
        assert cut <= 2 * 2 * math.pi * sd2 / 255, (sigma, aa, cut)
        assert abs(got - (full - cut)) <= 1e-6 * want, (sigma, aa, got, full, cut)


# ---- the reference the GPU tests use, against fp64 autograd -----------------------------------------------------------
def _scenes():
    base = synth.random_cube_scene(300, 48, seed=11, scale_mul=3.0)
    thin = dict(base)
    sc = np.array(base["scales"], np.float32)
    sc[:40] = 1e-6                                   # rho on its floor (sigma ~ 1e-3 px)
    sc[40:80, 0] = 2e-5                              # needles: det S small, off the floor
    op = np.array(base["opacity"], np.float32)
    op[:40] = 0.97                                   # o * 0.005 > 1/255: drawn at their centre pixel
    thin.update(scales=sc, opacity=op)
    mod = synth.random_cube_scene(300, 48, seed=12, scale_modifier=1.7)
    pre = synth.random_cube_scene(300, 48, seed=13, scale_mul=2.0)
    from oracle.raster_torch64 import cov3d
    pre["cov3D_precomp"] = cov3d(torch.tensor(pre["scales"], dtype=torch.float64),
                                 torch.tensor(pre["rots"], dtype=torch.float64)).numpy().astype(np.float32)
    return dict(thin=thin, scale_modifier=mod, cov3D_precomp=pre)


@pytest.mark.parametrize("name", ["thin", "scale_modifier", "cov3D_precomp"])
def test_aa_reference_backward_vs_autograd(name):
    """The oracle backward on o' plus the anti-aliasing chain (aa_reference.aa_backward) equals fp64 autograd of the
    anti-aliased forward (with the hand-written backward's 1/(det^2 + 1e-7) regulariser, DESIGN.md section 2) to 1e-6
    of each tensor's largest entry, including splats on the rho floor, where the extra term vanishes."""
    sc = _scenes()[name]
    o, st, r = aar.aa_forward(sc, "f64")
    vis = st["radii"] > 0
    if name == "thin":
        assert np.allclose(r[:40][vis[:40]], math.sqrt(aar.RHO_FLOOR), rtol=1e-12) and vis[:40].sum() > 10
        assert (st["n_contrib"] > 0).sum() > 100
    g = np.random.default_rng(1).standard_normal((3, sc["H"], sc["W"]))
    grads = aar.aa_backward(sc, st, o.backward(st, g))
    img, th = aar.render_autograd_aa(sc, st, denom_eps=1e-7)
    assert np.abs(img.detach().numpy() - st["color"]).max() < 1e-12
    (img * torch.tensor(g)).sum().backward()
    pairs = [("dL_dmeans3D", th["means3D"]), ("dL_dopacity", th["opacity"]), ("dL_dcolors", th["colors"])]
    pairs += [("dL_dcov3D", th["cov3D"])] if th["cov3D"] is not None else [("dL_dscales", th["scales"]), ("dL_drots", th["rots"])]
    for k, leaf in pairs:
        want = leaf.grad.numpy().reshape(len(vis), -1)
        got = np.asarray(grads[k], np.float64).reshape(len(vis), -1)
        err = np.abs(got - want).max() / np.abs(want).max()
        assert err <= 1e-6, (name, k, err)
    if name == "thin":   # on the floor the opacity gradient is 0.005 dL/do' and the geometry gets no rho term
        base = o.backward(st, g)
        fl = np.flatnonzero(vis[:40])
        np.testing.assert_allclose(grads["dL_dopacity"][fl], math.sqrt(aar.RHO_FLOOR) * base["dL_dopacity"][fl], rtol=1e-9)
        np.testing.assert_array_equal(grads["dL_dscales"][fl], base["dL_dscales"][fl])


def test_aa_fp32_rho_matches_conic_bits():
    """The fp32 restatement reproduces the oracle's fp32 conic bit for bit on C1-style, non-square / anisotropic-focal,
    scale_modifier and cov3D_precomp scenes (aa_reference.rho asserts it), and o' stays in [0.005 o, o)."""
    scenes = [synth.random_cube_scene(5000, 128, seed=21),
              synth.random_cube_scene(3000, 96, seed=22, width=160, height=90, focal=(150.0, 95.0)),
              synth.random_cube_scene(3000, 96, seed=23, scale_modifier=0.6)] + [_scenes()["cov3D_precomp"]]
    for sc in scenes:
        op, r = aar.aa_opacity(sc, "f32")
        _, st = oracle_forward(sc, "f32", render=False)
        vis = st["radii"] > 0
        assert vis.sum() > 100
        assert (r[vis] >= np.float32(0.005)).all() and (r[vis] < 1).all()


# ---- Python switches ---------------------------------------------------------------------------------------------
def test_dropin_settings_antialiasing(built_lib):
    import diff_gaussian_rasterization as dgr
    kw = dict(image_height=16, image_width=24, tanfovx=1.0, tanfovy=0.8, bg=torch.zeros(3), scale_modifier=1.0,
              viewmatrix=torch.eye(4), projmatrix=torch.eye(4), sh_degree=3, campos=torch.zeros(3), prefiltered=False,
              debug=False)
    rs = dgr.GaussianRasterizationSettings(**kw)
    assert len(rs._fields) == 12 and len(rs) == 12 and rs.antialiasing is False
    ra = dgr.GaussianRasterizationSettings(**kw, antialiasing=True)
    assert ra.antialiasing is True and tuple(ra) == tuple(rs)
    assert ra._replace(image_height=32).antialiasing is True and ra._replace(image_height=32).image_height == 32
    assert rs._replace(antialiasing=True).antialiasing is True and ra._replace(antialiasing=False).antialiasing is False
    assert dgr.GaussianRasterizationSettings(*tuple(rs), antialiasing=True).antialiasing is True
    import pickle
    assert pickle.loads(pickle.dumps(ra)).antialiasing is True
    a, b = dgr._pack_settings(rs), dgr._pack_settings(ra)      # the 12 packed fields do not carry the mode
    assert bytes(a) == bytes(b)
    assert dgr._antialiasing(ra) and not dgr._antialiasing(rs) and not dgr._antialiasing(tuple(rs))


def test_patch_reads_antialias_switch(built_lib, monkeypatch):
    from gps_gaussian_b200 import patch
    from gps_gaussian_b200 import GaussianRender as ours
    fake = types.ModuleType("lib.GaussianRender")
    fake.pts2render = lambda data, bg_color: None
    monkeypatch.setitem(sys.modules, "lib.GaussianRender", fake)
    try:
        for env, want in (("1", patch._pts2render_antialiased), ("0", ours.pts2render), (None, ours.pts2render)):
            if env is None:
                monkeypatch.delenv("GPSG_ANTIALIAS", raising=False)
            else:
                monkeypatch.setenv("GPSG_ANTIALIAS", env)
            patch.install()
            assert fake.pts2render is want, env
            assert patch.antialiasing() == (env == "1")
            monkeypatch.setenv("GPSG_ANTIALIAS", "0" if env == "1" else "1")     # read once, at install()
            assert patch.antialiasing() == (env == "1")
            patch.uninstall()
    finally:
        patch.uninstall()


def _box4(img):
    c, h, w = img.shape
    return img.reshape(c, h // 4, 4, w // 4, 4).mean((2, 4))


def test_aa_resolution_consistency_report():
    """Reported, not asserted: a C1-style scene rendered at 1024^2 and at 256^2; the error of the 4x4 box-downsampled
    1024^2 image against the 256^2 render, with and without the filter (the filter is expected to lower it)."""
    out = {}
    for aa in (False, True):
        imgs = {}
        for res in (1024, 256):
            sc = synth.random_cube_scene(10_000, res, seed=31)
            if aa:
                _, st, _ = aar.aa_forward(sc, "f32", nthreads=min(os.cpu_count() or 8, 64))
            else:
                _, st = oracle_forward(sc, "f32", nthreads=min(os.cpu_count() or 8, 64))
            imgs[res] = np.asarray(st["color"], np.float64)
        d = _box4(imgs[1024]) - imgs[256]
        out[aa] = dict(mean_abs=float(np.abs(d).mean()), rmse=float(np.sqrt((d ** 2).mean())),
                       mean_256=float(imgs[256].mean()), mean_1024=float(imgs[1024].mean()))
    record("aa:resolution_consistency", off=out[False], aa=out[True])
    print("\nresolution consistency (box4(1024^2) vs 256^2):", "off", out[False], "aa", out[True])


# ---- the anti-aliased C-oracle forward against the independent numpy restatement -----------------------------------
from test_oracle_cpu import ANISO  # noqa: E402

SEVEN = [(3000, 128, dict(seed=3)), (4000, 250, dict(spread=0.6, scale_mul=4.0, bg=(0.3, 0.6, 0.9), seed=11)),
         (2000, 130, dict(spread=3.0, seed=11)), (10_000, 256, dict()),
         (2500, 64, dict(spread=0.6, scale_mul=2.0, seed=3, **ANISO["wide"])),
         (2500, 64, dict(spread=0.6, scale_mul=2.0, seed=3, **ANISO["tall"])),
         (3000, 64, dict(spread=3.0, scale_mul=8.0, seed=19, width=120, height=48, focal=(70.0, 52.0),
                         principal=(66.0, 20.0), scale_modifier=1.3))]


def _agree(a, b, rho_c, tol):
    assert np.array_equal(a["radii"], b["radii"]) and np.array_equal(a["tiles_touched"], b["tiles_touched"])
    assert a["num_rendered"] == b["num_rendered"] > 0
    assert np.array_equal(a["keys"], b["keys"]) and np.array_equal(a["vals"], b["point_list"])
    assert np.array_equal(a["ranges"], b["ranges"]) and np.array_equal(a["n_contrib"], b["n_contrib"])
    vis = a["radii"] > 0
    assert np.abs(rho_c[vis] - b["rho"][vis]).max() < 1e-9 and (b["rho"][vis] < 1).all()
    assert np.abs(a["color"] - b["color"]).max() < tol and np.abs(a["final_T"] - b["final_T"]).max() < tol


@pytest.mark.parametrize("P,res,kw", SEVEN)
def test_aa_c_oracle_agrees_with_independent_restatement(P, res, kw):
    """The anti-aliased forward two ways that share no code: the C oracle (fp64) on o * rho with rho from the scalar
    restatement of the projection (aa_reference.rho), and oracle/raster_independent.py on o * rho with rho from its own
    matrix-form conic (rho^2 = det(I - 0.3 C)).  Integer state identical, image and final_T to 1e-12."""
    sc = synth.random_cube_scene(P, res, **kw)
    _, a, r = aar.aa_forward(sc, "f64")
    _agree(a, aar.independent_aa_forward(sc), r, 1e-12)


def test_aa_independent_restatement_randomised_sweep():
    """The seeded square and anisotropic sweep of tests/test_oracle_cpu.py (sizes, spreads, splat sizes, fx != fy,
    off-centre principal points, scale_modifier != 1), anti-aliased, both restatements to 1e-11."""
    rng = np.random.default_rng(77)
    cam_rng = np.random.default_rng(78)
    sizes = [(12, 180), (230, 9)] + [tuple(int(v) for v in cam_rng.integers(8, 300, 2)) for _ in range(8)]
    for k in range(10):
        res = int(rng.integers(24, 220))
        P = int(rng.integers(1, 2500))
        kw = dict(spread=float(rng.uniform(0.2, 2.5)), scale_mul=float(rng.uniform(0.5, 8.0)), bg=tuple(rng.uniform(0, 1, 3)),
                  seed=int(rng.integers(1 << 30)))
        W, H = sizes[k]
        fx = 0.8 * math.sqrt(W * H) * cam_rng.uniform(0.7, 1.4)
        aniso = dict(width=W, height=H, focal=(fx, fx * cam_rng.uniform(0.6, 1.6)),
                     principal=(W * cam_rng.uniform(0.3, 0.7), H * cam_rng.uniform(0.3, 0.7)),
                     scale_modifier=cam_rng.uniform(0.5, 2.0))
        for sc in (synth.random_cube_scene(P, res, **kw), synth.random_cube_scene(P, res, **kw, **aniso)):
            _, a, r = aar.aa_forward(sc, "f64")
            if a["num_rendered"] == 0:
                continue
            _agree(a, aar.independent_aa_forward(sc), r, 1e-11)


def test_aa_cov3d_precomp_agrees_with_independent_restatement():
    """cov3D_precomp: the C oracle given Sigma3D = R diag(s^2) R^T (fp64) against the independent restatement on the
    scale / rotation inputs it came from."""
    for sc in (synth.random_cube_scene(3000, 128, seed=5, scale_mul=2.0),
               synth.random_cube_scene(2500, 64, spread=0.6, scale_mul=2.0, seed=3, **ANISO["wide"])):
        q = np.asarray(sc["rots"], np.float64)
        r_, x, y, z = q[:, 0], q[:, 1], q[:, 2], q[:, 3]
        R = np.stack([1 - 2 * (y * y + z * z), 2 * (x * y - r_ * z), 2 * (x * z + r_ * y),
                      2 * (x * y + r_ * z), 1 - 2 * (x * x + z * z), 2 * (y * z - r_ * x),
                      2 * (x * z - r_ * y), 2 * (y * z + r_ * x), 1 - 2 * (x * x + y * y)], 1).reshape(-1, 3, 3)
        s = np.asarray(sc["scales"], np.float64) * sc.get("scale_modifier", 1.0)
        S = np.einsum("pik,pk,pjk->pij", R, s * s, R)
        c6 = S.reshape(-1, 9)[:, [0, 1, 2, 4, 5, 8]]
        pre = dict(sc, cov3D_precomp=c6, scales=None, rots=None)
        _, a, r = aar.aa_forward(pre, "f64")
        _agree(a, aar.independent_aa_forward(sc), r, 1e-11)


# ---- vectors recorded from the real extension's antialiasing=True (tools/dump_reference_vectors.py) ----------------
import glob  # noqa: E402

AA_FILES = sorted(glob.glob(os.path.join(ROOT, "tests", "golden", "raster_aa_reference_*.npz")))


def _aa_case_scene(case):
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    from dump_reference_vectors import RASTER_AA_CASES
    kw = dict(RASTER_AA_CASES[case])
    return synth.random_cube_scene(kw.pop("P"), kw.pop("res"), **kw)


def test_dump_script_records_antialiased_cases():
    """The dump script records its anti-aliased cases exactly when the installed extension takes `antialiasing`, under a
    file name the plain consumer's glob does not match."""
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import dump_reference_vectors as drv
    assert drv.RASTER_AA_CASES and not set(drv.RASTER_AA_CASES) & set(drv.RASTER_CASES)
    assert not glob.fnmatch.fnmatch("raster_aa_reference_c1_antialias.npz", "raster_reference_*.npz")
    import diff_gaussian_rasterization as ours
    assert not drv.upstream_has_antialiasing(ours)                # keyword-only here; `_fields` stays the 12 names
    new_api = types.SimpleNamespace(GaussianRasterizationSettings=types.SimpleNamespace(
        _fields=ours.GaussianRasterizationSettings._fields + ("antialiasing",)))
    assert drv.upstream_has_antialiasing(new_api)
    for case in drv.RASTER_AA_CASES:
        assert _aa_case_scene(case)["means3D"].shape[0] > 0


@pytest.mark.skipif(not AA_FILES, reason="no vectors recorded from the real diff-gaussian-rasterization with "
                    "antialiasing=True yet (tools/dump_reference_vectors.py); the anti-aliasing formula is recalled")
@pytest.mark.parametrize("path", AA_FILES or ["-"])
def test_aa_reference_matches_the_real_extension(path):
    from test_reference_vectors import check_against_vectors
    vec = np.load(path)
    assert bool(vec["antialiasing"])
    sc = _aa_case_scene(str(vec["case"]))
    o, st, _ = aar.aa_forward(sc, "f32")
    gr = aar.aa_backward(sc, st, o.backward(st, vec["grad_out"].astype(np.float32)))
    check_against_vectors(vec, st["color"], st["radii"], gr)


def test_dropin_settings_equality_includes_antialiasing(built_lib):
    import diff_gaussian_rasterization as dgr
    v, p = torch.eye(4), torch.eye(4)
    kw = dict(image_height=16, image_width=24, tanfovx=1.0, tanfovy=0.8, bg=1.0, scale_modifier=1.0, viewmatrix=v,
              projmatrix=p, sh_degree=3, campos=0.0, prefiltered=False, debug=False)
    a, b, c = (dgr.GaussianRasterizationSettings(**kw), dgr.GaussianRasterizationSettings(**kw),
               dgr.GaussianRasterizationSettings(**kw, antialiasing=True))
    assert a == b and not (a != b) and hash(a) == hash(b)
    assert a != c and not (a == c) and hash(a) != hash(c)
    assert c == c._replace() and c != a._replace(antialiasing=False) and a == c._replace(antialiasing=False)
