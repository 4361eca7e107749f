"""CPU: aux mode (depth and alpha beside the colour image) -- the C ABI's argument checks and sizes, and the fp64
reference the GPU tests hold the aux gradients to.  No call here reaches the device.

The reference (tests/test_raster_aux_gpu.py) builds the aux gradients from the oracles' colour entry points: depth is a
fourth colour channel (colour z, background 0) and alpha = 1 + the image of black Gaussians over the background
(-1, 0, 0).  Here that construction is checked against fp64 autograd of depth and alpha written directly, and the
forward identity against closed-form cases."""
import ctypes as C

import numpy as np
import pytest
import torch

from gps_gaussian_b200 import synth
from oracle import raster_torch64 as rt
from helpers import oracle_forward

DET = 1
AUX_SYMBOLS = ("gpsg_rasterize_forward", "gpsg_rasterize_forward_maps_finish", "gpsg_rasterize_forward_planned",
               "gpsg_rasterize_forward_maps_planned", "gpsg_rasterize_backward_workspace_bytes", "gpsg_rasterize_backward",
               "gpsg_rasterize_backward_maps_workspace_bytes", "gpsg_rasterize_backward_maps")
SIZES = [(0, 0), (1, 0), (1, 1), (7, 3), (1000, 5000), (499_400, 1_307_000), (2_000_000, 30_000_000)]


def test_aux_symbols_exported(built_lib):
    from gps_gaussian_b200 import _lib
    for name in AUX_SYMBOLS:
        assert name in _lib.EXPORTED and hasattr(_lib.lib, name)
    assert _lib.lib.gpsg_version() == 90


def test_aux_workspace_sizes(built_lib):
    """Without GPSG_BWD_DETERMINISTIC the aux workspace is the plain one (slot 9 of the accumulator row was spare); with
    it the partial sums are 8 x 10 floats per pair: 321 B per pair plus alignment."""
    from gps_gaussian_b200 import _lib
    L = _lib.lib
    for ws in (L.gpsg_rasterize_backward_workspace_bytes, L.gpsg_rasterize_backward_maps_workspace_bytes):
        for P, N in SIZES:
            assert ws(P, N, 0, 1) == ws(P, N, 0, 0) == ws(P, 0, 0, 0), (ws.__name__, P, N)
            extra = ws(P, N, DET, 1) - ws(P, 0, 0, 0)
            assert 321 * N <= extra <= 352 * N + 512, (ws.__name__, P, N, extra)
        for flags in (2, 4, -1):
            assert ws(10, 5, flags, 1) == 0
        assert ws(10, -1, DET, 1) == 0


def test_aux_argument_validation_without_gpu(built_lib):
    from gps_gaussian_b200 import _lib
    L = _lib.lib
    s = _lib.RasterSettings()
    s.image_height, s.image_width = 16, 16
    buf = (C.c_float * 1024)()
    p = C.cast(buf, C.c_void_p)
    alloc = _lib.ALLOC_CB
    # forward: out_depth / out_alpha both NULL or both set
    for d, a in ((p, None), (None, p)):
        assert L.gpsg_rasterize_forward(C.byref(s), 0, None, 0, 0, *([None] * 7), p, d, a, None, alloc, None, alloc,
                                        None, alloc, None, None, 0) == -1
        assert b"out_depth and out_alpha" in L.gpsg_last_error()
        assert L.gpsg_rasterize_forward_planned(C.byref(s), 0, None, 4, p, p, p, p, p, None, p, d, a, p, p, p, 16,
                                                p, None, 0) == -1
        assert b"out_depth and out_alpha" in L.gpsg_last_error()
        pp = (C.c_void_p * 2)(p, p)
        assert L.gpsg_rasterize_forward_maps_finish(C.byref(s), 0, None, 4, *([pp] * 6), p, d, a, p, p, p, alloc, None,
                                                    p, None) == -1
        assert b"out_depth and out_alpha" in L.gpsg_last_error()
        assert L.gpsg_rasterize_forward_maps_planned(C.byref(s), 0, None, 4, *([pp] * 6), p, d, a, p, p, p, 16, p,
                                                     None, 0) == -1
        assert b"out_depth and out_alpha" in L.gpsg_last_error()
    # backward: dL_dout_depth / dL_dout_alpha both NULL or both set; unknown flags refused first
    for d, a in ((p, None), (None, p)):
        for flags in (0, DET):
            assert L.gpsg_rasterize_backward(C.byref(s), 0, None, 10, 0, 5, *([None] * 12), d, a, *([None] * 9),
                                             flags) == -1
            assert b"dL_dout_depth and dL_dout_alpha" in L.gpsg_last_error()
            assert L.gpsg_rasterize_backward_maps(C.byref(s), 0, None, 8, 5, *([None] * 6), *([None] * 5), d, a,
                                                  *([None] * 5), None, flags) == -1
            assert b"dL_dout_depth and dL_dout_alpha" in L.gpsg_last_error()
    for flags in (2, 4, 1 | 8):
        assert L.gpsg_rasterize_backward(C.byref(s), 0, None, 10, 0, 5, *([None] * 12), p, p, *([None] * 9), flags) == -1
        assert b"flag" in L.gpsg_last_error()
    # P = 0: nothing to do, in both modes; missing inputs otherwise
    for flags in (0, DET):
        assert L.gpsg_rasterize_backward(C.byref(s), 0, None, 0, 0, 0, *([None] * 12), p, p, *([None] * 9), flags) == 0
        assert L.gpsg_rasterize_backward(C.byref(s), 0, None, 10, 0, 5, *([None] * 12), p, p, *([None] * 9), flags) == -1
        assert b"NULL" in L.gpsg_last_error()


def test_python_binding_requires_both_aux_tensors(built_lib):
    from gps_gaussian_b200 import _lib
    t = torch.zeros(4)
    with pytest.raises(ValueError, match="together"):
        _lib.rasterize_forward(None, t, t, t, t, out_depth=t)
    with pytest.raises(ValueError, match="together"):
        _lib.rasterize_backward(None, 0, (None, None, None), t, t, t, t, grad_alpha=t)


# ---- the forward identities on the fp32 oracle ----------------------------------------------------------------------
def _depth_alpha_oracle(o, st):
    """(depth, alpha) of an oracle state through the colour compositing: colours (z, z, z) over black, and 1 - T."""
    z = np.asarray(st["depth"])
    ds = dict(st, inputs=dict(st["inputs"], colors=np.repeat(z[:, None], 3, 1).astype(o.np), bg=np.zeros(3, o.np)))
    d = o.render_state(ds)
    assert np.array_equal(d["final_T"], st["final_T"]) and np.array_equal(d["n_contrib"], st["n_contrib"])
    return d["color"][0], (o.np(1.0) - st["final_T"]).astype(o.np)


def _one_gaussian_scene(res=32):
    sc = synth.random_cube_scene(2, res, seed=0)
    E = sc["cam"]["E"]
    X = lambda zz: ((np.array([0.0, 0.0, zz]) - E[:, 3]) @ E[:, :3])       # on the optical axis at view depth zz
    return sc, X


def test_closed_form_single_and_stacked_gaussians():
    sc, X = _one_gaussian_scene()
    H, W = sc["H"], sc["W"]
    # the principal point pixel of synth scenes: the Gaussian's screen centre
    base = dict(sc, means3D=np.array([X(2.0)], np.float32), colors=np.array([[0.2, 0.4, 0.6]], np.float32),
                opacity=np.array([0.7], np.float32), scales=np.full((1, 3), 0.05, np.float32),
                rots=np.array([[1.0, 0.0, 0.0, 0.0]], np.float32), bg=np.zeros(3, np.float32))
    o, st = oracle_forward(base, "f64")
    depth, alpha = _depth_alpha_oracle(o, st)
    z = float(st["depth"][0])
    px, py = st["means2D"][0]
    iy, ix = int(round(py)), int(round(px))
    G = np.exp(-0.5 * (st["conic_opacity"][0, 0] * (px - ix) ** 2 + st["conic_opacity"][0, 2] * (py - iy) ** 2)
               - st["conic_opacity"][0, 1] * (px - ix) * (py - iy))
    a = min(0.99, st["conic_opacity"][0, 3] * G)
    assert alpha[iy, ix] == pytest.approx(a, rel=1e-12)
    assert depth[iy, ix] == pytest.approx(a * z, rel=1e-12)
    assert np.allclose(depth, alpha * z, rtol=1e-12, atol=0)                  # one Gaussian: depth = alpha z everywhere
    # two stacked Gaussians: D = a1 z1 + a2 z2 (1 - a1)
    two = dict(base, means3D=np.array([X(2.0), X(3.0)], np.float32), colors=np.tile(base["colors"], (2, 1)),
               opacity=np.array([0.6, 0.8], np.float32), scales=np.full((2, 3), 0.05, np.float32),
               rots=np.tile(base["rots"], (2, 1)))
    o, st = oracle_forward(two, "f64")
    depth, alpha = _depth_alpha_oracle(o, st)
    co, m2, zz = st["conic_opacity"], st["means2D"], st["depth"]
    al = []
    for k in range(2):
        dx, dy = m2[k, 0] - ix, m2[k, 1] - iy
        al.append(min(0.99, co[k, 3] * np.exp(-0.5 * (co[k, 0] * dx * dx + co[k, 2] * dy * dy) - co[k, 1] * dx * dy)))
    assert depth[iy, ix] == pytest.approx(al[0] * zz[0] + al[1] * zz[1] * (1 - al[0]), rel=1e-12)
    assert alpha[iy, ix] == pytest.approx(1 - (1 - al[0]) * (1 - al[1]), rel=1e-12)
    # empty scene
    empty = dict(base, **{k: base[k][:0] for k in ("means3D", "colors", "opacity", "scales", "rots")})
    o, st = oracle_forward(empty, "f64")
    depth, alpha = _depth_alpha_oracle(o, st)
    assert not depth.any() and not alpha.any()
    assert (H, W) == depth.shape


# ---- the fp64 aux backward reference against autograd ---------------------------------------------------------------
def _aux_reference(o, st, sc, g_rgb, g_D, g_A):
    """The construction test_raster_aux_gpu.py uses: three colour backwards of the fp64 oracle + the view-row term."""
    P = st["P"]
    z = np.asarray(st["depth"], np.float64)
    out = o.backward(st, g_rgb)
    zero = np.zeros_like(g_D)
    sd = dict(st, inputs=dict(st["inputs"], colors=np.stack([z, np.zeros(P), np.zeros(P)], 1), bg=np.zeros(3)))
    wd = o.backward(sd, np.stack([g_D, zero, zero]))
    sa = dict(st, inputs=dict(st["inputs"], colors=np.zeros((P, 3)), bg=np.array([-1.0, 0.0, 0.0])))
    wa = o.backward(sa, np.stack([g_A, zero, zero]))
    tot = {k: out[k] + wd[k] + wa[k] for k in out if k != "dL_dcolors"}
    tot["dL_dcolors"] = out["dL_dcolors"]
    view = np.asarray(st["inputs"]["view"], np.float64).reshape(16)
    tot["dL_dmeans3D"] = tot["dL_dmeans3D"] + (wd["dL_dcolors"][:, 0] * (st["radii"] > 0))[:, None] * view[[2, 6, 10]]
    return tot


def _autograd(st, sc, g_rgb, g_D, g_A, cov=False):
    """fp64 autograd of <g_rgb, img> + <g_D, depth> + <g_A, alpha>, depth and alpha written directly."""
    dt = torch.float64
    T = lambda a: torch.tensor(np.asarray(a, np.float64), dtype=dt, requires_grad=True)
    i = st["inputs"]
    m3, col, op = T(i["means3D"]), T(i["colors"]), T(i["opacity"])
    sc_, ro = (T(i["scales"]), T(i["rots"])) if not cov else (None, None)
    c6 = T(i["cov3D_precomp"]) if cov else None
    kw = dict(scale_mod=float(i["scale_mod"]), cov3D=c6, denom_eps=1e-7)    # the backward's 1/(denom^2 + 1e-7)
    img = rt.render_autograd(st, m3, col, op, sc_, ro, **kw)
    view = torch.tensor(np.asarray(i["view"], np.float64).reshape(4, 4), dtype=dt)
    z = (torch.cat([m3, torch.ones(m3.shape[0], 1, dtype=dt)], 1) @ view)[:, 2]
    zc = torch.stack([z, torch.zeros_like(z), torch.zeros_like(z)], 1)
    sd = dict(st, inputs=dict(i, bg=np.zeros(3)))
    depth = rt.render_autograd(sd, m3, zc, op, sc_, ro, **kw)[0]
    sa = dict(st, inputs=dict(i, bg=np.array([-1.0, 0.0, 0.0])))
    alpha = 1.0 + rt.render_autograd(sa, m3, torch.zeros_like(col), op, sc_, ro, **kw)[0]
    t = lambda a: torch.tensor(a, dtype=dt)
    loss = (img * t(g_rgb)).sum() + (depth * t(g_D)).sum() + (alpha * t(g_A)).sum()
    loss.backward()
    g = dict(dL_dmeans3D=m3.grad.numpy(), dL_dcolors=col.grad.numpy(), dL_dopacity=op.grad.numpy().reshape(-1))
    if cov:
        g["dL_dcov3D"] = c6.grad.numpy()
    else:
        g["dL_dscales"], g["dL_drots"] = sc_.grad.numpy(), ro.grad.numpy()
    return g


@pytest.mark.parametrize("case", ["square", "mod0.6", "cov3D_precomp", "aniso-wide"])
def test_aux_backward_reference_matches_fp64_autograd(case):
    cam = {"square": {}, "mod0.6": dict(scale_modifier=0.6),
           "cov3D_precomp": {}, "aniso-wide": dict(width=72, height=24, focal=(80.0, 50.0), principal=(34.0, 11.0))}[case]
    sc = synth.random_cube_scene(60, 32, seed=7, scale_mul=3.0, bg=(0.2, 0.5, 0.8), **cam)
    cov = case == "cov3D_precomp"
    if cov:
        _, ref = oracle_forward(sc, "f64")
        sc = dict(sc, cov3D_precomp=ref["cov3D"].copy(), scales=None, rots=None)
    o, st = oracle_forward(sc, "f64")
    rng = np.random.default_rng(3)
    H, W = st["H"], st["W"]
    g_rgb, g_D, g_A = rng.standard_normal((3, H, W)), rng.standard_normal((H, W)), rng.standard_normal((H, W))
    want = _autograd(st, sc, g_rgb, g_D, g_A, cov=cov)
    got = _aux_reference(o, st, sc, g_rgb, g_D, g_A)
    for k, w in want.items():
        a = np.asarray(got[k], np.float64).reshape(w.shape)
        err = np.abs(a - w).max() / max(np.abs(w).max(), 1e-30)
        assert err <= 1e-9, (case, k, err)
    # planted errors the construction must catch: the depth term dropped from dL/dmeans3D, g_A with the wrong sign,
    # g_D scaled by 1 + 1e-3
    bad = [_aux_reference(o, st, sc, g_rgb, g_D, -g_A), _aux_reference(o, st, sc, g_rgb, g_D * (1 + 1e-3), g_A)]
    nodz = dict(got)
    view = np.asarray(st["inputs"]["view"], np.float64).reshape(16)
    zero = np.zeros_like(g_D)
    sd = dict(st, inputs=dict(st["inputs"], colors=np.stack([st["depth"], 0 * st["depth"], 0 * st["depth"]], 1),
                              bg=np.zeros(3)))
    dz = o.backward(sd, np.stack([g_D, zero, zero]))["dL_dcolors"][:, 0] * (st["radii"] > 0)
    nodz["dL_dmeans3D"] = got["dL_dmeans3D"] - dz[:, None] * view[[2, 6, 10]]
    bad.append(nodz)
    for b in bad:
        w = want["dL_dmeans3D"]
        assert np.abs(np.asarray(b["dL_dmeans3D"]) - w).max() / np.abs(w).max() > 1e-6
