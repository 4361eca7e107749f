"""GPU parity tests of the sm_90a rasterizer against the CPU oracle (run with -m gpu on an H100).

Bars (BASELINE.md section 2): tile indices (radii, tiles_touched, offsets, sorted keys + point list, ranges) bit-exact;
RGB <= 1e-4 abs (except threshold-flip pixels, see test_oracle_cpu.test_f32_and_f64_oracles_agree);
gradients <= 1e-3 rel against the fp64 oracle.  Everything goes through the C-ABI (ctypes)."""
import math
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from gps_gaussian_b200 import synth
from helpers import (GRAD_TOL, RGB_TOL, assert_grad_parity, assert_image_parity, grad_err as _grad_err, oracle_forward,
                     rel_err)

pytestmark = pytest.mark.gpu


def _run(sc):
    from gps_gaussian_b200.introspect import RasterCall
    rc = RasterCall(sc)
    rc.color.fill_(float("nan"))          # poison: a tile the kernels never visit cannot pass on stale allocator contents
    rc.forward()
    torch.cuda.synchronize()
    return rc


def _np(t):
    return t.detach().cpu().numpy()


def _assert_forward_parity(sc, check_geom_bits=True, tag=None):
    rc = _run(sc)
    st = rc.state()
    o, ref = oracle_forward(sc, "f32")
    P = sc["means3D"].shape[0]
    # ---- integer / index outputs: bit-exact
    assert np.array_equal(_np(st["radii"]), ref["radii"])
    assert rc.num_rendered == ref["num_rendered"]
    if P:
        assert np.array_equal(_np(st["tiles_touched"]).view(np.uint32), ref["tiles_touched"])
        if os.environ.get("GPSG_BINNING", "").startswith("r"):    # the per-Gaussian scan only exists on the radix fallback path
            assert np.array_equal(_np(st["point_offsets"]).view(np.uint32), np.cumsum(ref["tiles_touched"], dtype=np.uint32))
    if ref["num_rendered"]:
        assert np.array_equal(_np(st["keys"]).view(np.uint64), ref["keys"])
        assert np.array_equal(_np(st["point_list"]).view(np.uint32), ref["vals"])
    assert np.array_equal(_np(st["ranges"]).view(np.uint32), ref["ranges"])
    # ---- per-Gaussian fp32 state: same op order, no FMA contraction => identical bits for visible Gaussians
    vis = ref["radii"] > 0
    if check_geom_bits and vis.any():
        assert np.array_equal(_np(st["depths"])[vis].view(np.uint32), ref["depth"][vis].view(np.uint32))
        assert np.array_equal(_np(st["means2D"])[vis].view(np.uint32), ref["means2D"][vis].view(np.uint32))
        assert np.array_equal(_np(st["conic_opacity"])[vis].view(np.uint32), ref["conic_opacity"][vis].view(np.uint32))
    # ---- image: 1e-4 on every pixel that is not within rounding of a hard threshold; every pixel over 1e-4 is (helpers.py)
    assert_image_parity(tag or f"{sc['W']}x{sc['H']}_P{P}", _np(rc.color), _np(st["final_T"]), _np(st["n_contrib"]).view(np.uint32),
                        o, ref)
    return rc, ref


def test_c1_forward_parity():
    """BASELINE config C1: 256x256, 10k random Gaussians."""
    _assert_forward_parity(synth.random_cube_scene(10_000, 256), tag="C1")


@pytest.mark.parametrize("res,P,spread,mul,bg", [
    (250, 4000, 0.6, 4.0, (0.3, 0.6, 0.9)),      # image not a multiple of 16, coloured bg, fat splats
    (64, 300, 0.3, 12.0, (1.0, 1.0, 1.0)),       # splats covering many tiles; saturating pixels (T<1e-4 stop)
    (130, 2000, 3.0, 1.0, (0.0, 0.0, 0.0)),      # wide cloud: many off-screen / frustum-clamped Gaussians
    (64, 4500, 0.35, 1.5, (0.0, 0.0, 0.0)),      # 2-3.4k pairs per tile: the 16-keys-per-thread in-CTA sort variant
    (48, 30000, 0.25, 1.0, (0.0, 0.0, 0.0)),     # > 4096 pairs in a tile: automatic fallback to the global radix path
])
def test_forward_parity_edge_shapes(res, P, spread, mul, bg):
    sc = synth.random_cube_scene(P, res, spread=spread, scale_mul=mul, bg=bg, seed=11)
    _assert_forward_parity(sc)


def test_empty_inputs_and_all_culled():
    sc = synth.random_cube_scene(64, 96, bg=(0.2, 0.4, 0.6))
    empty = dict(sc)
    for k in ("means3D", "colors", "scales"):
        empty[k] = np.zeros((0, 3), np.float32)
    empty["rots"] = np.zeros((0, 4), np.float32); empty["opacity"] = np.zeros((0, 1), np.float32)
    rc = _run(empty)
    assert rc.num_rendered == 0
    assert torch.allclose(rc.color, torch.tensor(sc["bg"], device="cuda")[:, None, None].expand(3, 96, 96))
    behind = dict(sc)
    behind["means3D"] = (sc["means3D"] + (sc["campos"] - np.array([0, 0.85, 0], np.float32)) * 3).astype(np.float32)
    rc, ref = _assert_forward_parity(behind)
    assert rc.num_rendered == 0 and int(rc.radii.abs().sum()) == 0
    g = rc.backward(torch.ones_like(rc.color))
    assert all(float(v.abs().sum()) == 0 for v in g.values() if v is not None)


@pytest.mark.parametrize("P,res,kw", [(10_000, 256, dict()), (4000, 250, dict(spread=0.6, scale_mul=4.0, bg=(0.3, 0.6, 0.9), seed=11))])
def test_device_against_the_independent_numpy_restatement(P, res, kw):
    """The device vs oracle/raster_independent.py (fp64, raw inputs only, no state shared with gpsg_oracle.c).  fp32 vs
    fp64 projection can round a radius / tile rectangle differently, so the comparison is made on the tiles whose lists
    are identical in both (asserted to be > 99 % of the non-empty ones); there, every pixel that is not within rounding of
    a hard threshold (helpers.py) matches to 1e-4."""
    from oracle import raster_independent as ri
    sc = synth.random_cube_scene(P, res, **kw)
    rc = _run(sc)
    st = rc.state()
    ind = ri.forward_scene(sc)
    o32, ref = oracle_forward(sc, "f32")
    near = o32.margins(ref, nthreads=8)["near"]
    assert (_np(rc.radii) != ind["radii"]).mean() < 2e-3
    gx = (sc["W"] + 15) // 16
    plist, rng_d = _np(st["point_list"]).view(np.uint32), _np(st["ranges"]).view(np.uint32).reshape(-1, 2)
    same = np.zeros(rng_d.shape[0], bool)
    for t in range(rng_d.shape[0]):
        a, b = rng_d[t], ind["ranges"][t]
        same[t] = (a[1] - a[0] == b[1] - b[0]) and np.array_equal(plist[a[0]:a[1]], ind["point_list"][b[0]:b[1]])
    nonempty = (rng_d[:, 1] > rng_d[:, 0]) | (ind["ranges"][:, 1] > ind["ranges"][:, 0])
    assert same[nonempty].mean() > 0.99, same[nonempty].mean()
    ty, tx = np.divmod(np.arange(rng_d.shape[0]), gx)
    pix_same = np.zeros((sc["H"], sc["W"]), bool)
    for t in np.nonzero(same)[0]:
        pix_same[ty[t] * 16:ty[t] * 16 + 16, tx[t] * 16:tx[t] * 16 + 16] = True
    d = np.abs(_np(rc.color).astype(np.float64) - ind["color"]).max(0)
    ok = pix_same & ~near
    assert ok.mean() > 0.95
    assert d[ok].max() <= RGB_TOL, d[ok].max()
    assert np.array_equal(_np(st["n_contrib"]).view(np.uint32).reshape(sc["H"], sc["W"])[ok], ind["n_contrib"][ok])


def _poison(sc, seed=0):
    """NaN / inf in the per-Gaussian inputs, as an fp16 overflow inside the AMP network produces them (observed at step 18 of
    the C5-size stage-2 run: every scale / rotation / opacity NaN, half of the positions NaN)."""
    sc = {k: (v.copy() if isinstance(v, np.ndarray) else v) for k, v in sc.items()}
    sc["scales"][::7] = np.nan
    sc["rots"][3::11] = np.nan
    sc["means3D"][1::13] = np.nan
    sc["means3D"][5::17, 0] = np.inf
    sc["means3D"][6::19] = -np.inf
    sc["scales"][2::23, 1] = np.inf
    return sc


def test_non_finite_inputs_are_culled_not_crashed():
    """A NaN covariance converts to radius 0, whose 1-tile rectangle used to be COUNTED into the tile (tiles_touched = 1)
    but skipped by the scatter (radii <= 0): the tile list kept an uninitialised pair -> illegal address in the tile sort
    (found by running the reference's stage-2 loop at C5 size for 18 steps).  Such splats are now culled -- here, in the
    oracle and in the independent restatement alike; everything else about the scene stays bit-exact."""
    sc = _poison(synth.random_cube_scene(8000, 200, spread=0.6, scale_mul=2.0, seed=31, bg=(0.2, 0.3, 0.4)))
    rc, ref = _assert_forward_parity(sc, tag="nonfinite")
    bad = ~(np.isfinite(sc["scales"]).all(1) & np.isfinite(sc["rots"]).all(1) & np.isfinite(sc["means3D"]).all(1))
    assert bad.sum() > 1000 and int((_np(rc.radii)[bad] != 0).sum()) == 0 and int((_np(rc.radii)[~bad] > 0).sum()) > 3000
    assert bool(torch.isfinite(rc.color).all())
    got = rc.backward(torch.randn(3, 200, 200, device="cuda", generator=torch.Generator("cuda").manual_seed(1)))
    for k in ("dL_dmeans3D", "dL_dscales", "dL_drots", "dL_dopacity", "dL_dcolors"):
        g = _np(got[k]).reshape(8000, -1)
        assert np.isfinite(g).all() and float(np.abs(g[bad]).sum()) == 0.0, k          # culled: exactly zero gradient
    # the all-NaN frame of the real failure: nothing visible, background only, backward is a no-op
    allnan = dict(sc)
    allnan["scales"] = np.full_like(sc["scales"], np.nan); allnan["rots"] = np.full_like(sc["rots"], np.nan)
    allnan["opacity"] = np.full_like(sc["opacity"], np.nan)
    rc2 = _run(allnan)
    assert rc2.num_rendered == 0 and int(rc2.radii.abs().sum()) == 0
    assert torch.allclose(rc2.color, torch.tensor(sc["bg"], device="cuda")[:, None, None].expand(3, 200, 200))


def test_cov3d_precomp_path_matches_scale_rot_path():
    sc = synth.random_cube_scene(3000, 128, seed=5)
    _, ref = oracle_forward(sc, "f32")
    pre = dict(sc)
    pre["cov3D_precomp"] = ref["cov3D"].copy()
    # visible Gaussians carry their cov3D; culled ones have zeros there but are culled again anyway
    pre["scales"] = None; pre["rots"] = None
    rc = _run(pre)
    assert np.array_equal(_np(rc.radii), ref["radii"])
    assert np.abs(_np(rc.color) - ref["color"]).max() < 1e-2


def test_idempotent_and_deterministic_forward():
    sc = synth.random_cube_scene(10_000, 256, seed=2)
    a, b = _run(sc), _run(sc)
    assert torch.equal(a.color, b.color) and torch.equal(a.radii, b.radii)
    assert torch.equal(a.state()["point_list"], b.state()["point_list"])


def _assert_backward_parity(sc, seed=0, tag=None, rc=None, ref=None):
    """<= 1e-3 rel (max-normalised) against the fp32 AND the fp64 oracle backward run on the forward decisions the device
    took (its final_T / n_contrib / tile lists -- the inputs A.6 replays), for every Gaussian that no near-threshold pixel
    evaluates; the few that one does are bounded (helpers.assert_grad_parity)."""
    if rc is None:
        rc = _run(sc)
    if ref is None:
        _, ref = oracle_forward(sc, "f32", render=False)
    st = rc.state()
    P = sc["means3D"].shape[0]
    assert np.array_equal(_np(st["point_list"]).view(np.uint32), ref["vals"])     # same tile lists => forced replay is exact
    g = np.random.default_rng(seed).standard_normal((3, sc["H"], sc["W"])).astype(np.float32)
    got = rc.backward(torch.from_numpy(g).cuda(), want_cov3D=False)
    torch.cuda.synchronize()
    assert float(got["dL_dmeans2D"][:, 2].abs().sum()) == 0
    return assert_grad_parity(tag or f"{sc['W']}x{sc['H']}_P{P}", sc, {k: _np(v) for k, v in got.items() if v is not None}, ref,
                              _np(st["final_T"]), _np(st["n_contrib"]).view(np.uint32), g)


def test_c1_backward_parity():
    _assert_backward_parity(synth.random_cube_scene(10_000, 256), tag="C1")


@pytest.mark.parametrize("res,P,spread,mul,bg", [
    (100, 1500, 0.5, 4.0, (0.3, 0.6, 0.9)),      # coloured background term of dL/dalpha, ragged image
    (64, 300, 0.3, 10.0, (0.0, 0.0, 0.0)),       # heavy overlap, saturated pixels
])
def test_backward_parity_edge_shapes(res, P, spread, mul, bg):
    _assert_backward_parity(synth.random_cube_scene(P, res, spread=spread, scale_mul=mul, bg=bg, seed=13), seed=3)


def test_backward_is_linear_in_grad_out():
    """AMP loss scaling relies on it (reference train_stage2.py:83): backward(s*g) == s*backward(g)."""
    sc = synth.random_cube_scene(4000, 128, seed=4)
    rc = _run(sc)
    g = torch.randn(3, 128, 128, device="cuda", generator=torch.Generator("cuda").manual_seed(0))
    a = rc.backward(g)
    a = {k: v.clone() for k, v in a.items() if v is not None}
    b = rc.backward(g * 1024.0)
    for k in a:
        assert rel_err(_np(b[k]) / 1024.0, _np(a[k])) < 1e-4, k


def test_dropin_autograd_module_matches_capi():
    """The reference-facing path: GaussianRasterizer(...) autograd Function == raw C-ABI results."""
    import diff_gaussian_rasterization as dgr
    sc = synth.random_cube_scene(5000, 160, seed=6, bg=(0.1, 0.2, 0.3))
    rc = _run(sc)
    T = lambda a, rg=True: torch.tensor(a, device="cuda", requires_grad=rg)
    m, c, op, s, r = T(sc["means3D"]), T(sc["colors"]), T(sc["opacity"]), T(sc["scales"]), T(sc["rots"])
    m2d = torch.zeros_like(m, requires_grad=True)
    rs = dgr.GaussianRasterizationSettings(
        image_height=160, image_width=160, tanfovx=sc["tanfovx"], tanfovy=sc["tanfovy"],
        bg=torch.tensor(sc["bg"], device="cuda"), scale_modifier=1.0, viewmatrix=torch.tensor(sc["view"]),     # host cam
        projmatrix=torch.tensor(sc["proj"], device="cuda"), sh_degree=3, campos=torch.tensor(sc["campos"]),     # device proj
        prefiltered=False, debug=False)
    img, radii = dgr.GaussianRasterizer(raster_settings=rs)(means3D=m, means2D=m2d, opacities=op, shs=None,
                                                            colors_precomp=c, scales=s, rotations=r, cov3D_precomp=None)
    assert img.shape == (3, 160, 160) and radii.dtype == torch.int32 and torch.equal(radii, rc.radii)
    assert torch.equal(img, rc.color)
    g = torch.randn_like(img)
    img.backward(g)
    want = rc.backward(g)
    assert rel_err(_np(m.grad), _np(want["dL_dmeans3D"])) < 1e-5
    assert rel_err(_np(s.grad), _np(want["dL_dscales"])) < 1e-5 and rel_err(_np(r.grad), _np(want["dL_drots"])) < 1e-5
    assert rel_err(_np(op.grad), _np(want["dL_dopacity"])) < 1e-5 and rel_err(_np(c.grad), _np(want["dL_dcolors"])) < 1e-5
    assert m2d.grad is not None and m2d.grad.shape == (5000, 3)
    vis = dgr.GaussianRasterizer(raster_settings=rs).markVisible(m.detach())
    assert vis.dtype == torch.bool and bool(vis.all())


def _stereo_data(res, requires_grad=False, seed=None):
    sc = synth.stereo_pair_scene(res, keep_maps=True) if seed is None else synth.stereo_pair_scene(res, keep_maps=True, seed=seed)
    cam = sc["cam"]
    data = {"novel_view": {"FovX": torch.tensor([cam["FovX"]], dtype=torch.float64),
                           "FovY": torch.tensor([cam["FovY"]], dtype=torch.float64),
                           "width": torch.tensor([res]), "height": torch.tensor([res]),
                           "world_view_transform": torch.tensor(cam["world_view_transform"])[None],
                           "full_proj_transform": torch.tensor(cam["full_proj_transform"])[None],
                           "camera_center": torch.tensor(cam["camera_center"])[None]}}
    for name, vw in zip(("lmain", "rmain"), sc["views"]):
        T = lambda a: torch.tensor(a).cuda()[None].requires_grad_(requires_grad)
        data[name] = {"img": T(vw["img"]), "pts_valid": torch.tensor(vw["valid"]).cuda()[None], "xyz": T(vw["xyz"]),
                      "rot_maps": T(vw["rot_maps"]), "scale_maps": T(vw["scale_maps"]), "opacity_maps": T(vw["opacity_maps"])}
    return sc, data


def test_mirrored_render_and_pts2render():
    """reference-signature wrappers: pts2render(data, bg_color) (fused map ingest) and the gather -> render(data, idx, ...)
    data flow of the reference give the same image, equal to the oracle on the gathered Gaussians."""
    from gps_gaussian_b200.GaussianRender import pts2render, pts2render_gather
    res = 128
    sc, data = _stereo_data(res)
    out = pts2render(data, [0.0, 0.0, 0.0])["novel_view"]["img_pred"]
    assert out.shape == (1, 3, res, res)
    _, ref = oracle_forward(sc, "f32")
    d = np.abs(_np(out[0]) - ref["color"]).max(0)
    assert (d > RGB_TOL).mean() < 5e-4 and d.max() < 1e-2
    out2 = pts2render_gather(data, [0.0, 0.0, 0.0])["novel_view"]["img_pred"]
    assert torch.equal(out, out2)                 # same Gaussians in the same order -> bit-identical image


def test_fused_ingest_gradients_match_gather_path():
    """d(loss)/d(maps) of the fused ingest == autograd through the reference's gather/concat/render data flow."""
    from gps_gaussian_b200.GaussianRender import pts2render, pts2render_gather
    res = 96
    g = torch.randn(1, 3, res, res, device="cuda", generator=torch.Generator("cuda").manual_seed(3))
    grads = []
    for fn in (pts2render, pts2render_gather):
        _, data = _stereo_data(res, requires_grad=True, seed=4242)
        out = fn(data, [0.1, 0.2, 0.3])["novel_view"]["img_pred"]
        (out * g).sum().backward()
        grads.append({(v, k): data[v][k].grad for v in ("lmain", "rmain") for k in ("xyz", "img", "rot_maps", "scale_maps", "opacity_maps")})
    for key in grads[0]:
        a, b = grads[0][key], grads[1][key]
        assert a is not None and b is not None and a.shape == b.shape, key
        scale = max(float(b.abs().max()), 1e-20)
        per = (a - b).abs().flatten(1).max(0).values / scale if a.dim() > 1 else (a - b).abs() / scale
        assert int((per > GRAD_TOL).sum()) <= 4 and float(per.max()) < 5e-2, (key, float(per.max()))


def test_c2_full_size_parity_and_properties():
    """BASELINE config C2: 1024x1024, ~500k pixel-aligned Gaussians (full size; oracle forward takes ~1 s)."""
    sc = synth.stereo_pair_scene(1024)
    assert 400_000 < sc["means3D"].shape[0] < 600_000
    rc, ref = _assert_forward_parity(sc, tag="C2")
    st = rc.state()
    keys = st["keys"]
    assert bool((keys[1:] >= keys[:-1]).all())                                    # sortedness (size-independent property)
    assert int(st["tiles_touched"].to(torch.int64).sum()) == rc.num_rendered     # checksum of the binning
    # transmittance/colour consistency: C + T*bg with bg=0 => sum over channels bounded by 1 - T (colours in [0,1])
    assert bool((rc.color.sum(0) <= 3 * (1 - st["final_T"]) + 1e-4).all())


def test_c2_full_size_backward_parity():
    """BASELINE config C2 backward: all five gradient tensors of the ~500k Gaussians at 1024^2 against the fp32 and fp64
    oracle (VERDICT r1 weak #2: the largest backward check used to be C1)."""
    sc = synth.stereo_pair_scene(1024)
    rep = _assert_backward_parity(sc, seed=5, tag="C2")
    assert rep[("f64", "dL_dmeans3D")]["P"] > 400_000


def test_radix_fallback_path_is_bit_identical_to_tile_bucket_path():
    """The global-radix-sort fallback (used when a tile list exceeds the in-CTA sort capacity; forced here with
    GPSG_BINNING=radix in a subprocess) must give the same parity results, incl. the per-Gaussian offsets."""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    env = dict(os.environ, GPSG_BINNING="radix")
    r = subprocess.run([sys.executable, "-m", "pytest", "-q", "-x", "-m", "gpu", os.path.join(root, "tests", "test_raster_gpu.py"),
                        "-k", "c1_forward_parity or edge_shapes or c1_backward_parity or idempotent"],
                       env=env, cwd=root, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-2000:]


def test_planned_sync_free_forward_and_cuda_graph():
    """gpsg_rasterize_forward_planned: no host sync, caller buffers, device-side overflow flag, graph capture;
    bit-identical image / radii to the exact entry point."""
    from gps_gaussian_b200.introspect import to_device
    from gps_gaussian_b200.planned import PlannedRasterizer
    sc = synth.random_cube_scene(10_000, 256, seed=8, bg=(0.05, 0.1, 0.2))
    ref = _run(sc)
    d = to_device(sc)
    args = (sc, d["means3D"], d["colors"], d["opacity"], d["scales"], d["rots"])
    pr = PlannedRasterizer(10_000, 256, 256, capacity_pairs=int(ref.num_rendered * 1.25))
    out = pr.forward(*args)
    torch.cuda.synchronize()
    st = pr.status()
    assert not st["overflow"] and st["num_rendered"] == ref.num_rendered
    assert torch.equal(out, ref.color) and torch.equal(pr.radii, ref.radii)
    # overflow: capacity too small -> flagged, nothing written out of bounds, recoverable with grow()
    small = PlannedRasterizer(10_000, 256, 256, capacity_pairs=ref.num_rendered // 2)
    small.forward(*args)
    torch.cuda.synchronize()
    assert small.status()["overflow"] and not small.ok()
    small.grow()
    out2 = small.forward(*args)
    torch.cuda.synchronize()
    assert small.ok() and torch.equal(out2, ref.color)
    # CUDA graph capture + replay
    pr.capture(*args)
    pr.color.zero_()
    pr.replay(); pr.replay()
    torch.cuda.synchronize()
    assert pr.ok() and torch.equal(pr.color, ref.color)


@pytest.mark.parametrize("base_P,rep", [(1500, 3), (120, 40)])
def test_equal_depth_runs_are_ordered_by_gaussian_index(base_P, rep):
    """Exact depth ties (identical positions): the in-CTA sort orders equal-depth runs by Gaussian id with a shared-memory
    fix-up (runs <= 16) or the full radix fallback (longer runs) -- both must reproduce the stable (tile, depth) order."""
    sc = synth.random_cube_scene(base_P, 96, spread=0.5, scale_mul=2.0, seed=21, bg=(0.1, 0.1, 0.1))
    for k in ("means3D", "colors", "opacity", "scales", "rots"):
        sc[k] = np.ascontiguousarray(np.repeat(sc[k], rep, axis=0))
    perm = np.random.default_rng(0).permutation(base_P * rep)       # interleave the duplicates in index space
    for k in ("means3D", "colors", "opacity", "scales", "rots"):
        sc[k] = np.ascontiguousarray(sc[k][perm])
    _assert_forward_parity(sc)


@pytest.mark.parametrize("deg,M", [(3, 16), (1, 4), (0, 16)])
def test_sh_colour_branch_forward_backward(deg, M):
    """`GaussianRasterizer(shs=...)`: SH->RGB (+0.5, clamp) in front of the rasterizer and its backward (dL_dsh and the
    view-direction term of dL_dmeans3D).  Not used by GPS-Gaussian (it passes colors_precomp); API completeness."""
    import diff_gaussian_rasterization as dgr
    P, res = 4000, 128
    sc = synth.random_cube_scene(P, res, seed=17, bg=(0.1, 0.2, 0.3), scale_mul=2.0)
    rng = np.random.default_rng(5)
    shs = (rng.standard_normal((P, M, 3)) * 0.5).astype(np.float32)
    o = RasterOracleF64 = None
    from oracle.raster_oracle import RasterOracle
    o = RasterOracle("f64")
    col, cl = o.sh_colors(sc["means3D"], sc["campos"], shs, deg)
    assert 0.01 < cl.mean() < 0.95 or deg == 0                                   # the clamp is exercised
    sc_o = dict(sc, colors=col)
    _, ref = oracle_forward(sc_o, "f64")
    T = lambda a: torch.tensor(a, device="cuda", requires_grad=True)
    m, sh_t, op, s_, r = T(sc["means3D"]), T(shs), T(sc["opacity"]), T(sc["scales"]), T(sc["rots"])
    rs = dgr.GaussianRasterizationSettings(
        image_height=res, image_width=res, tanfovx=sc["tanfovx"], tanfovy=sc["tanfovy"], bg=torch.tensor(sc["bg"]),
        scale_modifier=1.0, viewmatrix=torch.tensor(sc["view"]), projmatrix=torch.tensor(sc["proj"]), sh_degree=deg,
        campos=torch.tensor(sc["campos"]), prefiltered=False, debug=False)
    img, radii = dgr.GaussianRasterizer(raster_settings=rs)(means3D=m, means2D=torch.zeros_like(m), opacities=op, shs=sh_t,
                                                            colors_precomp=None, scales=s_, rotations=r, cov3D_precomp=None)
    d = np.abs(_np(img) - ref["color"]).max(0)
    assert (d > RGB_TOL).mean() < 1e-3 and d.max() < 1e-2
    g = rng.standard_normal((3, res, res)).astype(np.float32)
    img.backward(torch.from_numpy(g).cuda())
    want = o.backward(ref, g.astype(np.float64))
    dsh = o.sh_backward(sc["means3D"], sc["campos"], shs, deg, cl, want["dL_dcolors"], want["dL_dmeans3D"])   # adds dir term
    for got, exp in ((sh_t.grad, dsh), (m.grad, want["dL_dmeans3D"]), (op.grad, want["dL_dopacity"]), (s_.grad, want["dL_dscales"])):
        per = _grad_err(_np(got), exp)
        assert int((per > GRAD_TOL).sum()) <= max(2, int(1e-3 * P)) and per.max() < 5e-2


def test_2048_render_resolution_forward_and_backward():
    """The real pipeline renders at 2 x src_res = 2048^2 (use_hr_img, reference config/stage2.yaml:15): 16384 tiles
    (tile-scan generic path, larger tile grid for the CTA-local histograms)."""
    sc = synth.stereo_pair_scene(512, render_res=2048, seed=77)
    assert sc["W"] == 2048 and sc["means3D"].shape[0] > 100_000
    rc, ref = _assert_forward_parity(sc, tag="2048")
    _assert_backward_parity(sc, seed=9, tag="2048", rc=rc, ref=ref)


def test_randomised_parity_sweep():
    """Small randomised sweep (image size, point count, spread, splat size, background): every integer output bit-exact."""
    rng = np.random.default_rng(2024)
    for k in range(8):
        res = int(rng.integers(40, 300))
        P = int(rng.integers(1, 6000))
        sc = synth.random_cube_scene(P, res, spread=float(rng.uniform(0.2, 2.5)), scale_mul=float(rng.uniform(0.5, 8.0)),
                                     bg=tuple(rng.uniform(0, 1, 3)), seed=int(rng.integers(1 << 30)))
        _assert_forward_parity(sc)


def test_pts2render_batch_of_two_and_host_pipeline():
    """bs = 2 through the reference-signature pts2render, and the packed host-buffer pipeline == direct render."""
    from gps_gaussian_b200.GaussianRender import pts2render
    from gps_gaussian_b200.pipeline import HostRenderPipeline, pack_host
    res = 96
    sc0, d0 = _stereo_data(res, seed=11)
    sc1, d1 = _stereo_data(res, seed=12)
    data = {"novel_view": {k: torch.cat([d0["novel_view"][k], d1["novel_view"][k]]) for k in d0["novel_view"]}}
    for v in ("lmain", "rmain"):
        data[v] = {k: torch.cat([d0[v][k], d1[v][k]]) for k in d0[v]}
    out = pts2render(data, [0.0, 0.0, 0.0])["novel_view"]["img_pred"]
    assert out.shape == (2, 3, res, res)
    for i, sc in enumerate((sc0, sc1)):
        _, ref = oracle_forward(sc, "f32")
        d = np.abs(_np(out[i]) - ref["color"]).max(0)
        assert (d > RGB_TOL).mean() < 1e-3 and d.max() < 1e-2
    pipe = HostRenderPipeline("cuda", max(sc0["means3D"].shape[0], sc1["means3D"].shape[0]), res, res)
    items = [(pack_host(sc), dd, 0) for sc, dd in ((sc0, d0), (sc1, d1), (sc0, d0))]
    outs = [torch.empty(3, res, res).pin_memory() for _ in items]
    pipe.run(items, outs)
    assert torch.equal(outs[0], outs[2]) and torch.equal(outs[0].cuda(), out[0]) and torch.equal(outs[1].cuda(), out[1])


def test_batched_pts2render_one_sync_matches_per_sample_path():
    """pts2render on a batch of two = `_RasterizeMapsBatch` (begin x2 -> ONE stream synchronise -> finish x2): images and map
    gradients equal the single-sample path (`_RasterizeMaps`, one synchronisation per sample) run on each sample alone."""
    from gps_gaussian_b200.GaussianRender import pts2render
    res = 96
    keys = ("xyz", "img", "rot_maps", "scale_maps", "opacity_maps")
    g = torch.randn(2, 3, res, res, device="cuda", generator=torch.Generator("cuda").manual_seed(5))
    singles = [_stereo_data(res, requires_grad=True, seed=sd)[1] for sd in (11, 12)]
    outs = [pts2render(d, [0.1, 0.2, 0.3])["novel_view"]["img_pred"] for d in singles]
    for i, o in enumerate(outs):
        (o * g[i:i + 1]).sum().backward()
    d0, d1 = (_stereo_data(res, seed=sd)[1] for sd in (11, 12))
    batch = {"novel_view": {k: torch.cat([d0["novel_view"][k], d1["novel_view"][k]]) for k in d0["novel_view"]}}
    for v in ("lmain", "rmain"):
        batch[v] = {k: torch.cat([d0[v][k], d1[v][k]]) for k in d0[v]}
        for k in keys:
            batch[v][k].requires_grad_(True)
    syncs = []
    orig = torch.cuda.Stream.synchronize
    torch.cuda.Stream.synchronize = lambda self: (syncs.append(1), orig(self))[1]
    try:
        out = pts2render(batch, [0.1, 0.2, 0.3])["novel_view"]["img_pred"]
    finally:
        torch.cuda.Stream.synchronize = orig
    assert len(syncs) == 1                                                   # one host synchronisation for the batch
    assert torch.equal(out[0:1], outs[0]) and torch.equal(out[1:2], outs[1])
    (out * g).sum().backward()
    for v in ("lmain", "rmain"):
        for k in keys:
            a = batch[v][k].grad
            b = torch.cat([singles[0][v][k].grad, singles[1][v][k].grad])
            assert a is not None and a.shape == b.shape, (v, k)
            assert float((a - b).abs().max()) <= 1e-5 * max(1e-20, float(b.abs().max())), (v, k)   # atomics order only
