"""CPU tests of the oracle itself (no GPU): analytic closed forms, autograd cross-check of the
hand-written backward, binning invariants.  These are what pin the rasterizer oracle, since the
reference ships no golden vectors for this path (SURVEY.md section 4 / 8c)."""
import math

import numpy as np
import pytest
import torch

from gps_gaussian_b200 import synth
from helpers import oracle_forward, rel_err
from oracle.raster_oracle import RasterOracle, taichi_splat


def _single_gaussian_scene(res=64, sigma_px=2.0, opacity=0.8, bg=(0.1, 0.2, 0.3)):
    K0, E0 = synth.ring_camera(0.0, res)
    cam = synth.novel_camera(K0, E0, K0, E0, res, res, 0.5)
    R, t = E0[:, :3], E0[:, 3]
    z = 2.0
    pc = np.array([0.0, 0.0, z])                       # ON the optical axis => J02 = J12 = 0, Sigma2D exactly isotropic
    xyz = (R.T @ (pc - t)).astype(np.float32)[None]
    s = np.float32(sigma_px * z / K0[0, 0])
    return dict(means3D=xyz, colors=np.array([[1.0, 0.5, 0.25]], np.float32), opacity=np.array([[opacity]], np.float32),
                scales=np.full((1, 3), s, np.float32), rots=np.array([[1, 0, 0, 0]], np.float32),
                view=cam["world_view_transform"], proj=cam["full_proj_transform"], campos=cam["camera_center"],
                tanfovx=math.tan(cam["FovX"] * 0.5), tanfovy=math.tan(cam["FovY"] * 0.5), W=res, H=res,
                bg=np.asarray(bg, np.float32)), sigma_px


def test_single_isotropic_gaussian_closed_form():
    """alpha(r) = min(0.99, o*exp(-r^2/(2(sigma^2+0.3)))), C = c*alpha + (1-alpha)*bg  (SURVEY 8c-iv)."""
    sc, sig = _single_gaussian_scene()
    _, st = oracle_forward(sc, "f64")
    assert st["n_visible"] == 1
    cx, cy = st["means2D"][0]
    # principal point (cx, cy) in continuous coords == pixel INDEX (cx-0.5, cy-0.5): ndc2pix folds the -0.5
    assert abs(cx - (32.0 - 0.5)) < 1e-3 and abs(cy - (32.0 + 25.0 * 64 / 1024 - 0.5)) < 1e-3
    var = sig * sig + 0.3
    assert st["radii"][0] == math.ceil(3 * math.sqrt(var))
    ys, xs = np.mgrid[0:64, 0:64]
    r2 = (xs - cx) ** 2 + (ys - cy) ** 2
    alpha = np.minimum(0.99, 0.8 * np.exp(-r2 / (2 * var)))
    alpha[alpha < 1 / 255] = 0
    # only tiles in the splat's rect see it
    rect = st["rects"][0]
    mask = np.zeros((64, 64), bool)
    mask[rect[1] * 16:rect[3] * 16, rect[0] * 16:rect[2] * 16] = True
    alpha = np.where(mask, alpha, 0)
    for ch, c in enumerate((1.0, 0.5, 0.25)):
        want = c * alpha + (1 - alpha) * sc["bg"][ch]
        assert np.abs(st["color"][ch] - want).max() < 2e-4       # det-normalised conic vs exact var: ~1e-5


def test_anisotropic_camera_matches_the_pinhole_model():
    """External truth for a camera with fx != fy, W != H and an off-centre principal point, from its K and E alone (none of
    the three restatements): means2D is the pinhole projection K [R|t] X minus the half pixel of ndc2pix, and inside the
    1.3 tanfov guard band inverse(conic) - 0.3 I = J Sigma3D J^T, with J the central-difference Jacobian of that projection
    and Sigma3D = R diag(scale_modifier * s)^2 R^T.  The guard band clamps t.x and t.y separately, so a Gaussian clamped
    in x only keeps the exact yy entry and one clamped in y only the exact xx entry.  This pins focal_x / focal_y and the
    two clamps without trusting the written-out Jacobian."""
    from scipy.spatial.transform import Rotation
    sc = synth.random_cube_scene(3000, 64, spread=3.0, scale_mul=8.0, width=120, height=48, focal=(70.0, 52.0),
                                 principal=(66.0, 20.0), scale_modifier=1.3, seed=19)
    _, st = oracle_forward(sc, "f64")
    K, E = sc["cam"]["K"], sc["cam"]["E"]

    def pinhole(X):
        pc = X @ E[:, :3].T + E[:, 3]
        return np.stack([K[0, 0] * pc[..., 0] / pc[..., 2] + K[0, 2], K[1, 1] * pc[..., 1] / pc[..., 2] + K[1, 2]], -1)

    X = sc["means3D"].astype(np.float64)
    vis = st["radii"] > 0
    assert np.abs(st["means2D"][vis] - (pinhole(X[vis]) - 0.5)).max() < 1e-4          # fp32 rounding of view / proj
    h = 1e-5
    J = np.stack([(pinhole(X + h * e) - pinhole(X - h * e)) / (2 * h) for e in np.eye(3)], -1)          # [P,2,3]
    q = sc["rots"].astype(np.float64)
    R = Rotation.from_quat(q[:, [1, 2, 3, 0]]).as_matrix()                                             # (r,x,y,z) unit
    s = sc["scales"].astype(np.float64) * sc["scale_modifier"]
    cov2 = J @ (R * (s * s)[:, None, :]) @ np.swapaxes(R, 1, 2) @ np.swapaxes(J, 1, 2)
    co = st["conic_opacity"][:, :3]
    inv = np.linalg.inv(np.stack([co[:, 0], co[:, 1], co[:, 1], co[:, 2]], -1).reshape(-1, 2, 2)[vis]) - 0.3 * np.eye(2)
    cov2 = cov2[vis]
    err = np.abs(inv - cov2) / np.abs(cov2).max((1, 2))[:, None, None]
    pc = X[vis] @ E[:, :3].T + E[:, 3]
    over = [np.abs(pc[:, k] / pc[:, 2]) - np.float32(1.3) * sc[f"tanfov{a}"] for k, a in ((0, "x"), (1, "y"))]
    inside_x, inside_y = over[0] < -1e-6, over[1] < -1e-6
    only_x, only_y = (over[0] > 1e-6) & inside_y, (over[1] > 1e-6) & inside_x
    assert only_x.sum() > 10 and only_y.sum() > 10 and (inside_x & inside_y).sum() > 1000
    assert err[inside_x & inside_y].max() < 1e-5
    assert err[only_x, 1, 1].max() < 1e-5 and err[only_y, 0, 0].max() < 1e-5
    assert err[only_x, 0, 0].max() > 1e-2 and err[only_y, 1, 1].max() > 1e-2        # and the clamp does act


def test_front_to_back_order_and_bg():
    sc, _ = _single_gaussian_scene(opacity=0.99)
    # second, farther Gaussian of another colour exactly behind the first
    far = sc["means3D"][0] + (sc["means3D"][0] - sc["campos"]) * 0.25
    sc["means3D"] = np.stack([far, sc["means3D"][0]]).astype(np.float32)        # far one FIRST in index order
    sc["colors"] = np.array([[0, 1, 0], [1, 0, 0]], np.float32)
    sc["opacity"] = np.array([[0.99], [0.99]], np.float32)
    sc["scales"] = np.repeat(sc["scales"], 2, 0); sc["rots"] = np.repeat(sc["rots"], 2, 0)
    _, st = oracle_forward(sc, "f64")
    tile = (33 // 16) * 4 + 31 // 16
    s, e = st["ranges"][tile]
    assert list(st["vals"][s:e]) == [1, 0]                        # near Gaussian first although it has the larger index
    c = st["color"][:, 33, 31]
    assert c[0] > 0.9 and c[1] < 0.08                            # near (red) dominates


# anisotropic, non-square, off-centre cameras (fx != fy, W != H) and scale_modifier != 1
ANISO = dict(wide=dict(width=96, height=40, focal=(80.0, 60.0), principal=(50.0, 17.0)),
             tall=dict(width=40, height=100, focal=(50.0, 70.0), principal=(18.0, 55.0), scale_modifier=1.7),
             small=dict(width=72, height=56, focal=(64.0, 64.0), principal=(30.0, 30.0), scale_modifier=0.6))


@pytest.mark.parametrize("res,P,spread,mul,kw,precomp", [
    pytest.param(64, 600, 0.45, 3.0, {}, False, id="64-600-0.45-3.0"),
    pytest.param(64, 600, 0.45, 3.0, {}, True, id="64-600-0.45-3.0-precomp"),
    pytest.param(48, 300, 0.3, 6.0, {}, False, id="48-300-0.3-6.0"),
    pytest.param(48, 300, 0.3, 6.0, {}, True, id="48-300-0.3-6.0-precomp"),
    pytest.param(64, 600, 0.6, 2.0, ANISO["wide"], False, id="wide"),
    pytest.param(64, 600, 0.6, 2.0, ANISO["wide"], True, id="wide-precomp"),
    pytest.param(64, 600, 0.6, 2.0, ANISO["tall"], False, id="tall"),
    pytest.param(64, 600, 0.6, 2.0, ANISO["tall"], True, id="tall-precomp"),
    pytest.param(64, 600, 0.6, 2.0, ANISO["small"], False, id="small"),
    pytest.param(64, 600, 0.6, 2.0, ANISO["small"], True, id="small-precomp"),
])
def test_backward_matches_fp64_autograd(res, P, spread, mul, kw, precomp):
    """The hand-written backward against fp64 autograd, incl. dL_dcov3D: on the scale/rotation path (Sigma3D an
    intermediate of the autograd graph) and on the cov3D_precomp path (Sigma3D a leaf, no scale/rotation chain)."""
    from oracle.raster_torch64 import cov3d, render_autograd
    sc = synth.random_cube_scene(P, res, spread=spread, scale_mul=mul, bg=(0.2, 0.5, 0.7), seed=7, **kw)
    mod = sc["scale_modifier"]
    o, st = oracle_forward(sc, "f64")
    cov3D = st["cov3D"].copy()
    if precomp:
        o, pre = oracle_forward(dict(sc, cov3D_precomp=cov3D, scales=None, rots=None), "f64")
        assert np.array_equal(pre["radii"], st["radii"])
        st = pre
    g = np.random.default_rng(0).standard_normal(st["color"].shape)
    gr = o.backward(st, g)
    for denom_eps in (0.0, 1e-7):
        T = lambda a: torch.tensor(np.asarray(a, np.float64), requires_grad=True)
        m, c, op, s, r = T(sc["means3D"]), T(sc["colors"]), T(sc["opacity"]), T(sc["scales"]), T(sc["rots"])
        if precomp:
            cov = T(cov3D)
        else:
            cov = cov3d(s, r, mod)
            cov.retain_grad()
        img = render_autograd(st, m, c, op, s, r, scale_mod=mod, cov3D=cov, denom_eps=denom_eps)
        assert np.abs(img.detach().numpy() - st["color"]).max() < 1e-12
        (img * torch.tensor(g)).sum().backward()
        checks = [("means3D", m.grad, gr["dL_dmeans3D"]), ("colors", c.grad, gr["dL_dcolors"]),
                  ("opacity", op.grad.reshape(-1), gr["dL_dopacity"]), ("cov3D", cov.grad, gr["dL_dcov3D"])]
        if not precomp:
            checks += [("scales", s.grad, gr["dL_dscales"]), ("rots", r.grad, gr["dL_drots"])]
        # The true derivative (denom_eps = 0) differs from the backward's 1/(denom^2 + 1e-7) by a relative 1e-7/denom^2,
        # which grows as splats shrink: 1.7e-6 at scale_modifier 0.6.  With the same regulariser in the autograd graph the
        # two agree to 1e-12 in every case, so the regulariser is the whole difference.
        tol = 1e-12 if denom_eps else (3e-6 if mod < 1 else 1e-6)
        for name, a, b in checks:
            assert rel_err(b, a.numpy()) < tol, (name, denom_eps)


def test_backward_matches_fp64_autograd_with_independent_binning():
    """Same cross-check, but the autograd forward takes its discrete state (tile lists, ranges) from the independent numpy
    restatement instead of gpsg_oracle.c: the truth the hand-written A.6-A.8 backward is held to then shares nothing with the
    C oracle (VERDICT r1 missing #6)."""
    from oracle import raster_independent as ri
    from oracle.raster_torch64 import render_autograd
    sc = synth.random_cube_scene(500, 56, spread=0.45, scale_mul=3.0, bg=(0.2, 0.5, 0.7), seed=9)
    ind = ri.forward_scene(sc)
    st_ind = dict(W=sc["W"], H=sc["H"], ranges=ind["ranges"], vals=ind["point_list"],
                  inputs=dict(view=sc["view"], proj=sc["proj"], tanfovx=sc["tanfovx"], tanfovy=sc["tanfovy"], bg=sc["bg"]))
    T = lambda a: torch.tensor(np.asarray(a, np.float64), requires_grad=True)
    m, c, op, s, r = T(sc["means3D"]), T(sc["colors"]), T(sc["opacity"]), T(sc["scales"]), T(sc["rots"])
    img = render_autograd(st_ind, m, c, op, s, r)
    assert np.abs(img.detach().numpy() - ind["color"]).max() < 1e-12          # torch forward == numpy forward
    g = np.random.default_rng(2).standard_normal(ind["color"].shape)
    (img * torch.tensor(g)).sum().backward()
    o, st = oracle_forward(sc, "f64")
    assert np.array_equal(st["vals"], ind["point_list"]) and np.abs(st["color"] - ind["color"]).max() < 1e-12
    gr = o.backward(st, g)
    for name, a, b in (("means3D", m.grad, gr["dL_dmeans3D"]), ("colors", c.grad, gr["dL_dcolors"]),
                       ("opacity", op.grad.reshape(-1), gr["dL_dopacity"]), ("scales", s.grad, gr["dL_dscales"]),
                       ("rots", r.grad, gr["dL_drots"])):
        assert rel_err(b, a.numpy()) < 1e-6, name


def test_f32_and_f64_oracles_agree():
    sc = synth.random_cube_scene(3000, 128, seed=3)
    _, a = oracle_forward(sc, "f32")
    _, b = oracle_forward(sc, "f64")
    # 1e-4 everywhere except at pixels where a hard threshold (alpha<1/255, T<1e-4, power>0) flips between
    # precisions; such a flip moves a pixel by at most ~1/255 and is inherent to the algorithm
    d = np.abs(a["color"] - b["color"]).max(0)
    assert (d > 1e-4).mean() < 5e-4 and d.max() < 1e-2
    assert (a["radii"] != b["radii"]).mean() < 1e-3


def test_threshold_margins_explain_every_f32_f64_compositing_difference():
    """The flip allowance as a theorem (VERDICT r1 weak #1), exercised on the CPU with the fp64 oracle standing in for the
    device: compositing the SAME per-Gaussian state in fp32 and in fp64, every pixel that is NOT within `RasterOracle.EPS`
    of a hard threshold (alpha vs 1/255, test_T vs 1e-4, power vs 0) agrees to 2e-6 with identical n_contrib, so any pixel
    over 1e-4 must be a near-threshold one; likewise every gradient of a Gaussian no near-threshold pixel evaluates."""
    from helpers import assert_grad_parity, assert_image_parity
    sc = synth.random_cube_scene(40_000, 256, spread=0.5, scale_mul=2.0, seed=21)
    o32, a = oracle_forward(sc, "f32")
    b = RasterOracle("f64").render_state(a, nthreads=8)
    rec = assert_image_parity("cpu_selfcheck", b["color"], b["final_T"], b["n_contrib"], o32, a)
    assert 0 < rec["near"] < 0.02 * rec["pixels"] and rec["max_err_not_near"] <= 2e-6
    # gradients: "device" = the fp32 oracle's own backward; checked against fp32/fp64 backward forced onto its decisions
    g = np.random.default_rng(1).standard_normal((3, 256, 256)).astype(np.float32)
    got = o32.backward(a, g)
    got = {"dL_dmeans3D": got["dL_dmeans3D"], "dL_dcolors": got["dL_dcolors"], "dL_dopacity": got["dL_dopacity"],
           "dL_dscales": got["dL_dscales"], "dL_drots": got["dL_drots"], "dL_dmeans2D": got["dL_dmean2D"]}
    rep = assert_grad_parity("cpu_selfcheck", sc, got, a, a["final_T"], a["n_contrib"], g)
    r32 = rep[("f32", "dL_dmeans3D")]
    assert r32["max_err_clean"] == r32["max_err_shared"] == r32["max_err_own"] == 0.0     # same code, same decisions
    assert rep[("f64", "dL_dmeans3D")]["own"] < 0.1 * 40_000


@pytest.mark.parametrize("P,res,kw", [(3000, 128, dict(seed=3)), (4000, 250, dict(spread=0.6, scale_mul=4.0, bg=(0.3, 0.6, 0.9), seed=11)),
                                      (2000, 130, dict(spread=3.0, seed=11)), (10_000, 256, dict()),
                                      (2500, 64, dict(spread=0.6, scale_mul=2.0, seed=3, **ANISO["wide"])),
                                      (2500, 64, dict(spread=0.6, scale_mul=2.0, seed=3, **ANISO["tall"])),
                                      (3000, 64, dict(spread=3.0, scale_mul=8.0, seed=19, width=120, height=48,
                                                      focal=(70.0, 52.0), principal=(66.0, 20.0), scale_modifier=1.3))])
def test_independent_numpy_restatement_agrees_with_the_c_oracle(P, res, kw):
    """oracle/raster_independent.py takes only the raw call arguments (no state of gpsg_oracle.c): culling, radii, tile
    counts, the sorted 64-bit keys, point list and tile ranges must be IDENTICAL to the C oracle's fp64 build, the image,
    final_T to 1e-12 and n_contrib identical (VERDICT r1 missing #6)."""
    from oracle import raster_independent as ri
    sc = synth.random_cube_scene(P, res, **kw)
    _, a = oracle_forward(sc, "f64")
    b = ri.forward_scene(sc)
    assert np.array_equal(a["radii"], b["radii"]) and np.array_equal(a["tiles_touched"], b["tiles_touched"])
    assert a["num_rendered"] == b["num_rendered"] > 0
    assert np.array_equal(a["keys"], b["keys"]) and np.array_equal(a["vals"], b["point_list"])
    assert np.array_equal(a["ranges"], b["ranges"])
    assert np.abs(a["means2D"] - b["means2D"]).max() < 1e-9 and np.abs(a["conic_opacity"][:, :3] - b["conic"]).max() < 1e-9
    assert np.abs(a["color"] - b["color"]).max() < 1e-12 and np.abs(a["final_T"] - b["final_T"]).max() < 1e-12
    assert np.array_equal(a["n_contrib"], b["n_contrib"])


def test_non_finite_inputs_are_culled_in_both_restatements():
    """NaN / inf scales, rotations, positions: culled (radius 0 is not a splat), so sum(tiles_touched) == number of emitted
    pairs -- the invariant whose violation crashed the tile sort on the device (tests/test_raster_gpu.py has the GPU half)."""
    from oracle import raster_independent as ri
    sc = synth.random_cube_scene(3000, 128, seed=3)
    sc["scales"][::7] = np.nan; sc["rots"][3::11] = np.nan; sc["means3D"][1::13] = np.nan
    sc["means3D"][5::17, 0] = np.inf; sc["scales"][2::23, 1] = np.inf
    for dt in ("f32", "f64"):
        _, a = oracle_forward(sc, dt)
        assert a["num_rendered"] == int(a["tiles_touched"].sum()) == int((a["ranges"][:, 1].astype(np.int64) - a["ranges"][:, 0]).sum())
        assert np.all((a["radii"] > 0) == (a["tiles_touched"] > 0)) and np.isfinite(a["color"]).all()
    with np.errstate(all="ignore"):
        b = ri.forward_scene(sc)
    assert np.array_equal(a["radii"], b["radii"]) and np.array_equal(a["vals"], b["point_list"])
    assert np.abs(a["color"] - b["color"]).max() < 1e-12


def test_independent_restatement_randomised_sweep():
    """Seeded sweep over image size, point count, spread, splat size, background: the two restatements (C, scalar chains;
    numpy, matrix form + global argsort) must agree on every integer output and on the image to 1e-11.  Every scene is
    also rendered through a second camera with width and height drawn independently (one 12 px wide: a single tile
    column; one 9 px tall), fx != fy, an off-centre principal point and a scale_modifier != 1."""
    from oracle import raster_independent as ri
    rng = np.random.default_rng(77)
    cam_rng = np.random.default_rng(78)
    sizes = [(12, 180), (230, 9)] + [tuple(int(v) for v in cam_rng.integers(8, 300, 2)) for _ in range(8)]   # grid_x == 1, H < 16
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
            _, a = oracle_forward(sc, "f64")
            b = ri.forward_scene(sc)
            assert np.array_equal(a["radii"], b["radii"]) and np.array_equal(a["tiles_touched"], b["tiles_touched"]), k
            assert np.array_equal(a["keys"], b["keys"]) and np.array_equal(a["vals"], b["point_list"]), k
            assert np.array_equal(a["ranges"], b["ranges"]) and np.array_equal(a["n_contrib"], b["n_contrib"]), k
            assert np.abs(a["color"] - b["color"]).max() < 1e-11 and np.abs(a["final_T"] - b["final_T"]).max() < 1e-11, k


def test_binning_invariants():
    sc = synth.random_cube_scene(5000, 200, seed=5)               # 200 is not a multiple of 16
    _, st = oracle_forward(sc, "f32")
    keys = st["keys"]
    assert np.all(keys[1:] >= keys[:-1])                          # sortedness
    assert st["num_rendered"] == int(st["tiles_touched"].sum())
    tiles = (keys >> np.uint64(32)).astype(np.int64)
    gx = (200 + 15) // 16
    for t in np.unique(tiles):
        s, e = st["ranges"][t]
        assert np.all(tiles[s:e] == t) and (s == 0 or tiles[s - 1] != t) and (e == len(tiles) or tiles[e] != t)
    # every pair's tile lies inside its Gaussian's rect
    r = st["rects"][st["vals"]]
    assert np.all((tiles % gx >= r[:, 0]) & (tiles % gx < r[:, 2]) & (tiles // gx >= r[:, 1]) & (tiles // gx < r[:, 3]))
    # equal (tile, depth) keys keep Gaussian-index order (stable sort)
    same = keys[1:] == keys[:-1]
    assert np.all(st["vals"][1:][same] > st["vals"][:-1][same])


def test_empty_and_culled():
    sc = synth.random_cube_scene(50, 64, seed=1)
    sc["means3D"] = (sc["means3D"] + (sc["campos"] - np.array([0, 0.85, 0], np.float32)) * 3).astype(np.float32)  # behind cam
    _, st = oracle_forward(sc, "f32")
    assert st["n_visible"] == 0 and st["num_rendered"] == 0
    assert np.allclose(st["color"], sc["bg"][:, None, None]) and np.all(st["final_T"] == 1)
    o = RasterOracle("f32")
    assert not o.mark_visible(sc["means3D"], sc["view"]).any()


def test_mark_visible_at_the_near_plane():
    """mark_visible is the preprocess's z > 0.2 cull: points on both sides of view-space z = 0.2 (further than fp32 rounding
    from it) get the expected mask in both precisions, and no Gaussian it marks absent is rendered."""
    from helpers import near_plane_scene
    sc, z = near_plane_scene(synth.random_cube_scene(2000, 64, seed=5, **ANISO["wide"]))
    far = np.abs(z - 0.2) > 1e-5
    assert (far & (z > 0.2)).sum() > 500 and (far & (z < 0.2)).sum() > 500
    for dt in ("f32", "f64"):
        present = RasterOracle(dt).mark_visible(sc["means3D"], sc["view"])
        assert np.array_equal(present[far], z[far] > 0.2), dt
        _, st = oracle_forward(sc, dt, render=False)
        assert (st["radii"] > 0).sum() > 500 and not (st["radii"] > 0)[~present].any(), dt


def test_taichi_splat_restatement():
    """Sequential semantics of reference lib/TaichiRender.py:12-23 (z-buffer on inverse depth)."""
    pts = np.array([[[3.2, 4.9, 0.5, 1, 0, 0], [3.7, 4.1, 0.8, 0, 1, 0], [3.0, 4.0, 0.6, 0, 0, 1],
                     [-5.0, 99.0, 0.1, 1, 1, 1], [1.0, 1.0, 9.0, 9, 9, 9]]], np.float32)
    mask = np.array([[1, 1, 1, 1, 0]], np.float32)
    depth, color = taichi_splat(pts, mask, 8)
    assert depth[0, 0, 4, 3] == np.float32(0.8) and list(color[0, :, 4, 3]) == [0, 1, 0]      # nearest (largest 1/z) wins
    assert depth[0, 0, 7, 0] == np.float32(0.1) and list(color[0, :, 7, 0]) == [1, 1, 1]      # clamped to the border
    assert color[0, 0, 1, 1] == -1                                                           # masked point ignored
