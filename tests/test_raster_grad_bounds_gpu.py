"""GPU: every rasterizer gradient element within its own fp32 rounding bound of an fp64 backward on the device's own state.

The fp64 truth is gpsg_oracle.c's backward run on the device's fp32 forward state (means2D / conic_opacity bit-identical
to the fp32 oracle's, tile lists, final_T, n_contrib), so what separates the two is only the backward's rounding and the
device's ex2.approx / rcp.approx.  Each element must satisfy |device - fp64| <= 2^-24 * Mag (oracle/raster_bounds.py: a
running error bound of the compositing pass, chained through the exact per-Gaussian Jacobian of the projection), with the
summation depth of the device's accumulation tree.  Gaussians evaluated by a pixel whose `alpha < 1/255` / `power > 0`
decision lies within fp32 rounding of its threshold are exempt and keep helpers.py's shared / own caps.  The worst
error-to-bound ratio per tensor goes to $GPSG_PARITY_LOG.  The max-normalised checks of test_raster_gpu.py stay as they are.
"""
import contextlib
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from gps_gaussian_b200 import synth
from helpers import EPS_ALPHA_F64, SHARED_TOL, TAINT_CAP, grad_err, oracle_forward, record
from oracle import raster_bounds as rb
from oracle.raster_oracle import RasterOracle

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WIDE = dict(width=250, height=40, focal=(240.0, 190.0), principal=(118.0, 23.0))
TALL = dict(width=40, height=250, focal=(150.0, 260.0), principal=(21.0, 130.0))
# device name -> oracle name
KEYS = (("dL_dmeans2D", "dL_dmean2D"), ("dL_dcolors", "dL_dcolors"), ("dL_dopacity", "dL_dopacity"),
        ("dL_dmeans3D", "dL_dmeans3D"), ("dL_dscales", "dL_dscales"), ("dL_drots", "dL_drots"), ("dL_dcov3D", "dL_dcov3D"))


def _np(t):
    return t.detach().cpu().numpy()


def _threads():
    return min(os.cpu_count() or 8, 64)


@contextlib.contextmanager
def _deterministic():
    was, warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(was, warn_only=warn)


class _Truth:
    """The device forward of `sc`, the fp64 backward on its state for one dL/dpix, the bounds and the exemption set."""

    def __init__(self, sc, seed, colors64=None, col_err=None):
        from gps_gaussian_b200.introspect import RasterCall
        self.sc = sc
        self.rc = RasterCall(sc)
        self.rc.forward()
        torch.cuda.synchronize()
        dst = self.rc.state()
        _, self.ref = oracle_forward(sc, "f32", render=False)
        assert np.array_equal(_np(dst["point_list"]).view(np.uint32), self.ref["vals"])
        vis = self.ref["radii"] > 0
        assert np.array_equal(_np(dst["means2D"])[vis].view(np.uint32), self.ref["means2D"][vis].view(np.uint32))
        assert np.array_equal(_np(dst["conic_opacity"])[vis].view(np.uint32), self.ref["conic_opacity"][vis].view(np.uint32))
        self.st = rb.fp64_state(self.ref, _np(dst["final_T"]), _np(dst["n_contrib"]).view(np.uint32), colors=colors64)
        self.g = np.random.default_rng(seed).standard_normal((3, sc["H"], sc["W"])).astype(np.float32)
        self.want = RasterOracle("f64").backward_mag(self.st, self.g, col_err=col_err)
        self.bounds = rb.grad_bounds(self.st, self.want, rb.device_depth(self.ref, self.want["nterm"]))
        self.shared, self.own, self.m = rb.exempt_sets(self.st, _threads())

    def device_grads(self, deterministic=False):
        got = self.rc.backward(torch.from_numpy(self.g).cuda(), want_cov3D=True, deterministic=deterministic)
        torch.cuda.synchronize()
        return {k: _np(v) for k, v in got.items() if v is not None}

    def check(self, tag, got, keys=KEYS, extra_exempt=None):
        exempt = self.shared | self.own
        if extra_exempt is not None:
            exempt = exempt | extra_exempt
        rec = dict(P=int(self.st["P"]), visible=int((self.st["radii"] > 0).sum()), exempt=int(exempt.sum()))
        for k_got, k_ref in keys:
            if got.get(k_got) is None:
                continue
            a = got[k_got][:, :2] if k_got == "dL_dmeans2D" else got[k_got]
            r = rb.ratios(a, self.want[k_ref], self.bounds[k_ref])
            clean = ~exempt
            worst = int(np.argmax(np.where(clean, r, -1.0))) if clean.any() else 0
            rec[k_got] = float(r[clean].max()) if clean.any() else 0.0
            per = grad_err(a, self.want[k_ref])
            mx = lambda msk: float(per[msk].max()) if msk.any() else 0.0
            assert rec[k_got] <= 1.0, (tag, k_got, rec[k_got], self._where(worst))
            assert mx(self.shared) <= SHARED_TOL and mx(self.own) <= TAINT_CAP, (tag, k_got, mx(self.shared), mx(self.own))
        record(f"{tag}:grad_bound", **rec)
        return rec

    def _where(self, i):
        """Where Gaussian i sits: its list positions / tiles, the transmittance there, which Mag column dominates."""
        ref, st = self.ref, self.st
        pos = np.nonzero(ref["vals"] == i)[0]
        tiles = (ref["keys"][pos] >> np.uint64(32)).astype(np.int64)
        depth_in_tile = pos - ref["ranges"][tiles, 0].astype(np.int64)
        return dict(gaussian=i, tiles=tiles[:8].tolist(), list_pos=depth_in_tile[:8].tolist(),
                    nterm=int(self.want["nterm"][i]), mag=self.want["mag"][i].tolist(),
                    mag_dominant=int(np.argmax(self.want["mag"][i])), absum=self.want["absum"][i].tolist(),
                    conic_opacity=st["conic_opacity"][i].tolist())


def _scene(res, P, spread, mul, bg, cam, seed=13):
    return synth.random_cube_scene(P, res, spread=spread, scale_mul=mul, bg=bg, seed=seed, **cam)


def test_c1_default_and_deterministic_backward_within_the_bound():
    t = _Truth(synth.random_cube_scene(10_000, 256), 0)
    t.check("C1", t.device_grads())
    with _deterministic():
        t.check("C1:det", t.device_grads(deterministic=None))


@pytest.mark.parametrize("res,P,spread,mul,bg,cam", [
    (100, 1500, 0.5, 4.0, (0.3, 0.6, 0.9), {}),
    (64, 300, 0.3, 10.0, (0.0, 0.0, 0.0), {}),
    (64, 300, 0.3, 10.0, (0.3, 0.6, 0.9), {}),   # saturated pixels (T_final < 1e-3) with the background term
    (64, 1500, 0.6, 4.0, (0.3, 0.6, 0.9), dict(WIDE, scale_modifier=0.7)),
    (64, 1500, 0.6, 4.0, (0.0, 0.0, 0.0), dict(TALL, scale_modifier=1.6)),
    (64, 1000, 0.6, 2.0, (0.2, 0.2, 0.2), dict(width=300, height=8, focal=(300.0, 50.0), principal=(150.0, 4.5))),
    (64, 3000, 3.0, 5.0, (0.0, 0.0, 0.0), dict(width=120, height=48, focal=(70.0, 52.0), principal=(66.0, 20.0),
                                               scale_modifier=1.3)),
], ids=["100-1500-0.5-4.0-bg0", "64-300-0.3-10.0-bg1", "64-300-0.3-10.0-bgc", "250x40-mod0.7", "40x250-mod1.6", "300x8",
        "120x48-clamp-mod1.3"])
def test_edge_shapes_within_the_bound(res, P, spread, mul, bg, cam):
    t = _Truth(_scene(res, P, spread, mul, bg, cam), 3)
    t.check(f"edge-{res}-{P}-{'bgc' if any(bg) else 'bg0'}", t.device_grads())


@pytest.mark.parametrize("res,P,spread,mul,lo,hi", [(64, 4500, 0.35, 1.5, 2049, 4096), (48, 30000, 0.25, 1.0, 4097, 1 << 30)],
                         ids=["big-tile-2049-4096", "over-4096-radix"])
def test_long_tile_lists_within_the_bound(res, P, spread, mul, lo, hi):
    """The 2049-4096 in-CTA sort class, and a list over 4096 (global radix fallback); default and deterministic."""
    t = _Truth(_scene(res, P, spread, mul, (0.0, 0.0, 0.0), {}, seed=11), 5)
    r = t.ref["ranges"].astype(np.int64)
    assert lo <= int((r[:, 1] - r[:, 0]).max()) <= hi
    t.check(f"lists-{lo}", t.device_grads())
    t.check(f"lists-{lo}:det", t.device_grads(deterministic=True))


def test_forced_radix_binning_within_the_bound():
    """C1, the big-tile class and the edge shapes again with GPSG_BINNING=radix (every scene through the fallback)."""
    env = dict(os.environ, GPSG_BINNING="radix")
    r = subprocess.run([sys.executable, "-m", "pytest", "-q", "-x", "-m", "gpu", os.path.join(ROOT, "tests", "test_raster_grad_bounds_gpu.py"),
                        "-k", "c1_default or edge_shapes or big-tile"], env=env, cwd=ROOT, capture_output=True, text=True,
                       timeout=1200)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-2000:]


def test_cov3d_precomp_within_the_bound():
    sc = synth.random_cube_scene(3000, 128, seed=5)
    _, ref = oracle_forward(sc, "f32", render=False)
    t = _Truth(dict(sc, cov3D_precomp=ref["cov3D"].copy(), scales=None, rots=None), 1)
    got = t.device_grads()
    t.check("cov3D_precomp", got, keys=tuple(k for k in KEYS if k[0] not in ("dL_dscales", "dL_drots")))


def test_c2_and_2048_within_the_bound_and_a_smaller_exemption():
    """Full size: C2 (default and deterministic backward) and the 2048^2 render.  The exemption set on the device's own
    state must be smaller than the fp64-recomputed one helpers.assert_grad_parity uses (eps_alpha = 1e-3)."""
    sc = synth.stereo_pair_scene(1024)
    t = _Truth(sc, 5)
    rec = t.check("C2", t.device_grads())
    t.check("C2:det", t.device_grads(deterministic=True))
    assert rec["visible"] > 400_000
    o64, st64 = oracle_forward(sc, "f64", render=False)
    st64 = dict(st64, radii=t.ref["radii"], ranges=t.ref["ranges"], _vals_full=t.ref["_vals_full"])
    old = o64.margins(st64, eps=dict(T=0.0, alpha=EPS_ALPHA_F64), nthreads=_threads())["taint"]
    record("C2:exemption", new=rec["exempt"], fp64_recomputed=int(old.sum()), P=rec["P"])
    assert rec["exempt"] < int(old.sum()), (rec["exempt"], int(old.sum()))
    t2 = _Truth(synth.stereo_pair_scene(512, render_res=2048, seed=77), 9)
    t2.check("2048", t2.device_grads())


# SH colours on the device: direction (difference 1, squares and sum 3, rsqrt 2, scaling 1) -> 7u relative; a degree-3
# basis function multiplies up to three direction components and a constant -> 3 * 7 + 4 = 25u, relative to the basis
# polynomial with every term in absolute value (`_abs_basis`: 4zz - xx - yy cancels, 4zz + xx + yy does not); the 16-term
# sum 16, the + 0.5 1.  So |rgb_device - rgb| <= C_SH_RGB * u * (sum_k babs_k |sh_k| + 0.5), and dL_dsh = b_k dL_drgb rounds
# by 25 + 1 relative to babs_k |dL_drgb|.
C_SH_RGB = 48.0
C_SH_GRAD = 26.0


def _abs_basis(means3D, campos):
    """The 16 real SH basis polynomials of degree <= 3 with every coefficient and direction component in absolute value
    and every difference a - b as a + b, [P, 16]."""
    d = np.asarray(means3D, np.float64) - np.asarray(campos, np.float64)
    x, y, z = np.abs(d / np.linalg.norm(d, axis=1, keepdims=True)).T
    C1, C2, C3 = 0.4886025119029199, (1.0925484305920792, 0.31539156525252005, 0.5462742152960396), \
        (0.5900435899266435, 2.890611442640554, 0.4570457994644658, 0.3731763325901154, 1.445305721320277)
    xx, yy, zz = x * x, y * y, z * z
    one = np.ones_like(x)
    return np.stack([0.28209479177387814 * one, C1 * y, C1 * z, C1 * x,
                     C2[0] * x * y, C2[0] * y * z, C2[1] * (2 * zz + xx + yy), C2[0] * x * z, C2[2] * (xx + yy),
                     C3[0] * y * (3 * xx + yy), C3[1] * x * y * z, C3[2] * y * (4 * zz + xx + yy),
                     C3[3] * z * (2 * zz + 3 * xx + 3 * yy), C3[2] * x * (4 * zz + xx + yy), C3[4] * z * (xx + yy),
                     C3[0] * x * (xx + 3 * yy)], 1)


def test_sh_degree3_through_the_dropin_within_the_bound():
    """SH degree 3 through GaussianRasterizer: the device computes the colours itself, so the fp64 backward runs on the
    fp64 SH colours and the colour rounding enters the compositing bound (col_err); dL_dsh is bounded by
    |d rgb / d sh|^T (Mag_rgb) = |b_k| Mag_rgb plus its own rounding.  Channels whose value before the clamp at 0 lies
    within the colour error of 0 may clamp differently and are exempt.  dL_dmeans3D also carries the view-direction term
    of the SH backward, which this bound does not cover; it is checked by test_raster_gpu.py."""
    import diff_gaussian_rasterization as dgr
    P, res, deg, M = 4000, 128, 3, 16
    sc = synth.random_cube_scene(P, res, seed=17, bg=(0.1, 0.2, 0.3), scale_mul=2.0)
    shs = (np.random.default_rng(5).standard_normal((P, M, 3)) * 0.5).astype(np.float32)
    o = RasterOracle("f64")
    col64, cl = o.sh_colors(sc["means3D"], sc["campos"], shs, deg)
    neg, _ = o.sh_colors(sc["means3D"], sc["campos"], -shs, deg)
    v = np.where(cl.astype(bool), 1.0 - neg, col64)                      # the value before the clamp (v(-sh) = 1 - v(sh))
    basis = o.sh_backward(sc["means3D"], sc["campos"], shs, deg, np.zeros((P, 3), np.uint8), np.ones((P, 3)),
                          np.zeros((P, 3)))                              # [P, M, 3]: b_k in every channel
    babs = _abs_basis(sc["means3D"], sc["campos"])[:, :M, None]          # [P, M, 1]
    assert (babs >= np.abs(basis) * (1 - 1e-12)).all()
    col_err = C_SH_RGB * ((babs * np.abs(shs)).sum(1) + 0.5)            # units of u
    near_clamp = (np.abs(v) <= col_err * rb.U).any(1)
    # final_T / n_contrib / the tile lists do not depend on the colours: the C-ABI forward on any colours gives the SH run's
    t = _Truth(dict(sc, colors=col64.astype(np.float32)), 2, colors64=col64, col_err=col_err)
    T = lambda a: torch.tensor(a, device="cuda", requires_grad=True)
    m, sh_t, op, s_, r = T(sc["means3D"]), T(shs), T(sc["opacity"]), T(sc["scales"]), T(sc["rots"])
    rs = dgr.GaussianRasterizationSettings(
        image_height=res, image_width=res, tanfovx=sc["tanfovx"], tanfovy=sc["tanfovy"], bg=torch.tensor(sc["bg"]),
        scale_modifier=1.0, viewmatrix=torch.tensor(sc["view"]), projmatrix=torch.tensor(sc["proj"]), sh_degree=deg,
        campos=torch.tensor(sc["campos"]), prefiltered=False, debug=False)
    img, _ = dgr.GaussianRasterizer(raster_settings=rs)(means3D=m, means2D=torch.zeros_like(m), opacities=op, shs=sh_t,
                                                        colors_precomp=None, scales=s_, rotations=r, cov3D_precomp=None)
    img.backward(torch.from_numpy(t.g).cuda())
    got = dict(dL_dopacity=_np(op.grad).reshape(-1), dL_dscales=_np(s_.grad), dL_drots=_np(r.grad))
    rec = t.check("sh3", got, keys=(("dL_dopacity", "dL_dopacity"), ("dL_dscales", "dL_dscales"), ("dL_drots", "dL_drots")),
                  extra_exempt=near_clamp)
    want_sh = o.sh_backward(sc["means3D"], sc["campos"], shs, deg, cl, t.want["dL_dcolors"], np.zeros((P, 3)))
    g_rgb = np.where(cl.astype(bool), 0.0, np.abs(t.want["dL_dcolors"]))
    b_rgb = np.where(cl.astype(bool), 0.0, t.bounds["dL_dcolors"])
    bound_sh = np.abs(basis) * b_rgb[:, None, :] + C_SH_GRAD * rb.U * babs * g_rgb[:, None, :]
    r_sh = rb.ratios(_np(sh_t.grad), want_sh, bound_sh)
    keep = ~(t.shared | t.own | near_clamp)
    record("sh3:grad_bound_dsh", worst=float(r_sh[keep].max()), near_clamp=int(near_clamp.sum()), **rec)
    assert float(r_sh[keep].max()) <= 1.0, float(r_sh[keep].max())
    assert near_clamp.mean() < 0.01


def _map_data(sc, requires_grad=True):
    cam = sc["cam"]
    data = {"novel_view": {"FovX": torch.tensor([cam["FovX"]], dtype=torch.float64),
                           "FovY": torch.tensor([cam["FovY"]], dtype=torch.float64),
                           "width": torch.tensor([sc["W"]]), "height": torch.tensor([sc["H"]]),
                           "world_view_transform": torch.tensor(cam["world_view_transform"])[None],
                           "full_proj_transform": torch.tensor(cam["full_proj_transform"])[None],
                           "camera_center": torch.tensor(cam["camera_center"])[None]}}
    for name, vw in zip(("lmain", "rmain"), sc["views"]):
        T = lambda a: torch.tensor(a).cuda()[None].requires_grad_(requires_grad)
        data[name] = {"img": T(vw["img"]), "pts_valid": torch.tensor(vw["valid"]).cuda()[None], "xyz": T(vw["xyz"]),
                      "rot_maps": T(vw["rot_maps"]), "scale_maps": T(vw["scale_maps"]), "opacity_maps": T(vw["opacity_maps"])}
    return data


def test_pts2render_map_gradients_within_the_bound():
    """pts2render (the fused map ingest of the training loop), default and deterministic backward, with gradients on the
    maps.  Valid pixels, lmain then rmain in row-major order, are the Gaussians of the gathered scene: each map gradient
    is that Gaussian's gradient (the image one 0.5 * dL_dcolors, since colour = img * 0.5 + 0.5) within its bound;
    invalid pixels get exactly zero."""
    from gps_gaussian_b200.GaussianRender import pts2render
    sc = synth.stereo_pair_scene(128, keep_maps=True, seed=4242, bg=(0.1, 0.2, 0.3))
    t = _Truth(sc, 6)
    g = torch.from_numpy(t.g).cuda()[None]
    for det in (False, True):
        data = _map_data(sc)
        ctx = _deterministic() if det else contextlib.nullcontext()
        with ctx:
            out = pts2render(data, [float(v) for v in sc["bg"]])["novel_view"]["img_pred"]
            (out * g).sum().backward()
        assert torch.equal(out[0], t.rc.color)
        got = {k: [] for k in ("dL_dmeans3D", "dL_dcolors", "dL_dopacity", "dL_dscales", "dL_drots")}
        for name, vw in zip(("lmain", "rmain"), sc["views"]):
            d = data[name]
            valid = np.asarray(vw["valid"]).reshape(-1).astype(bool)
            maps = dict(dL_dmeans3D=_np(d["xyz"].grad[0]).reshape(-1, 3),
                        dL_dcolors=_np(d["img"].grad[0]).reshape(3, -1).T / 0.5,
                        dL_dopacity=_np(d["opacity_maps"].grad[0]).reshape(-1),
                        dL_dscales=_np(d["scale_maps"].grad[0]).reshape(3, -1).T,
                        dL_drots=_np(d["rot_maps"].grad[0]).reshape(4, -1).T)
            for k, a in maps.items():
                assert float(np.abs(a[~valid]).max()) == 0.0, (det, name, k)      # invalid pixels: exactly zero
                got[k].append(a[valid])
        got = {k: np.concatenate(v) for k, v in got.items()}
        assert got["dL_dopacity"].shape[0] == t.st["P"]
        t.check("pts2render:det" if det else "pts2render", got,
                keys=tuple((k, k) for k in ("dL_dmeans3D", "dL_dcolors", "dL_dopacity", "dL_dscales", "dL_drots")))
