"""GPU: the deterministic rasterizer backward (GPSG_BWD_DETERMINISTIC, selected by torch.use_deterministic_algorithms).

Contract: bit-identical gradients for identical inputs whatever the CTA schedule, concurrent streams or binning path;
each gradient differs from the default (atomic) backward only by fp32 re-association, so it passes the same parity
classes against the fp32 / fp64 oracles (helpers.assert_grad_parity)."""
import contextlib
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from gps_gaussian_b200 import synth
from helpers import assert_grad_parity, oracle_forward, rel_err, record

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WIDE = dict(width=250, height=40, focal=(240.0, 190.0), principal=(118.0, 23.0))
TALL = dict(width=40, height=250, focal=(150.0, 260.0), principal=(21.0, 130.0))


@contextlib.contextmanager
def deterministic_algorithms():
    was, warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(was, warn_only=warn)


def _np(t):
    return t.detach().cpu().numpy()


def _run(sc):
    from gps_gaussian_b200.introspect import RasterCall
    rc = RasterCall(sc)
    rc.forward()
    torch.cuda.synchronize()
    return rc


def _grad(rc, g, det=True, **kw):
    out = rc.backward(g, want_cov3D=True, deterministic=det, **kw)
    return {k: v.clone() for k, v in out.items() if v is not None}


def _assert_bitwise(a, b, what=""):
    assert a.keys() == b.keys(), what
    for k in a:
        assert torch.equal(a[k], b[k]), (what, k, float((a[k] - b[k]).abs().max()))


def _det_parity(sc, seed, tag, rc=None, ref=None):
    """helpers.assert_grad_parity for the DET backward; also: equal to itself run under the torch flag (NaN-filled
    scratch / workspace, `fill_uninitialized_memory`) and <= 1e-5 max-normalised from the default backward."""
    if rc is None:
        rc = _run(sc)
    if ref is None:
        _, ref = oracle_forward(sc, "f32", render=False)
    st = rc.state()
    assert np.array_equal(_np(st["point_list"]).view(np.uint32), ref["vals"])
    g = torch.from_numpy(np.random.default_rng(seed).standard_normal((3, sc["H"], sc["W"])).astype(np.float32)).cuda()
    det = _grad(rc, g, det=True)
    with deterministic_algorithms():
        _assert_bitwise(det, _grad(rc, g, det=None), tag + ": DET under the torch flag")
    dflt = _grad(rc, g, det=False)
    for k in det:
        assert rel_err(_np(det[k]), _np(dflt[k])) <= 1e-5, (tag, k, rel_err(_np(det[k]), _np(dflt[k])))
    assert float(det["dL_dmeans2D"][:, 2].abs().sum()) == 0
    return assert_grad_parity(tag + ":det", sc, {k: _np(v) for k, v in det.items()}, ref, _np(st["final_T"]),
                              _np(st["n_contrib"]).view(np.uint32), _np(g))


# ---- 1. parity against the oracles ----------------------------------------------------------------------------------
def test_det_c1_backward_parity():
    _det_parity(synth.random_cube_scene(10_000, 256), 0, "C1")


@pytest.mark.parametrize("res,P,spread,mul,bg,cam", [
    (100, 1500, 0.5, 4.0, (0.3, 0.6, 0.9), {}),
    (64, 300, 0.3, 10.0, (0.0, 0.0, 0.0), {}),
    (64, 1500, 0.6, 4.0, (0.3, 0.6, 0.9), dict(WIDE, scale_modifier=0.7)),
    (64, 1500, 0.6, 4.0, (0.0, 0.0, 0.0), dict(TALL, scale_modifier=1.6)),
    (64, 1000, 0.6, 2.0, (0.2, 0.2, 0.2), dict(width=300, height=8, focal=(300.0, 50.0), principal=(150.0, 4.5))),
    (64, 3000, 3.0, 5.0, (0.0, 0.0, 0.0), dict(width=120, height=48, focal=(70.0, 52.0), principal=(66.0, 20.0),
                                               scale_modifier=1.3)),
    (48, 30000, 0.25, 1.0, (0.0, 0.0, 0.0), {}),     # > 4096 pairs in a tile: the global radix binning path
], ids=["100-1500-0.5-4.0-bg0", "64-300-0.3-10.0-bg1", "250x40-mod0.7", "40x250-mod1.6", "300x8", "120x48-clamp-mod1.3",
        "48-30000-radix-tile"])
def test_det_backward_parity_edge_shapes(res, P, spread, mul, bg, cam):
    sc = synth.random_cube_scene(P, res, spread=spread, scale_mul=mul, bg=bg, seed=13, **cam)
    rc = _run(sc)
    if P == 30000:
        r = rc.state()["ranges"].to(torch.int64)
        assert int((r[:, 1] - r[:, 0]).max()) > 4096
    _det_parity(sc, 3, f"edge-{res}-{P}", rc=rc)


def test_det_cov3d_precomp_parity():
    sc = synth.random_cube_scene(3000, 128, seed=5)
    _, ref = oracle_forward(sc, "f32")
    pre = dict(sc, cov3D_precomp=ref["cov3D"].copy(), scales=None, rots=None)
    _det_parity(pre, 1, "cov3D_precomp")


def test_det_sh_degree3_through_the_dropin():
    """SH colours (degree 3) through GaussianRasterizer under the torch flag: bounds of the SH test against fp64, two runs
    bitwise equal, and within 1e-5 of the default backward."""
    import diff_gaussian_rasterization as dgr
    from oracle.raster_oracle import RasterOracle
    from helpers import grad_err, GRAD_TOL
    P, res, deg, M = 4000, 128, 3, 16
    sc = synth.random_cube_scene(P, res, seed=17, bg=(0.1, 0.2, 0.3), scale_mul=2.0)
    rng = np.random.default_rng(5)
    shs = (rng.standard_normal((P, M, 3)) * 0.5).astype(np.float32)
    o = RasterOracle("f64")
    col, cl = o.sh_colors(sc["means3D"], sc["campos"], shs, deg)
    _, ref = oracle_forward(dict(sc, colors=col), "f64")
    g = rng.standard_normal((3, res, res)).astype(np.float32)
    rs = dgr.GaussianRasterizationSettings(
        image_height=res, image_width=res, tanfovx=sc["tanfovx"], tanfovy=sc["tanfovy"], bg=torch.tensor(sc["bg"]),
        scale_modifier=1.0, viewmatrix=torch.tensor(sc["view"]), projmatrix=torch.tensor(sc["proj"]), sh_degree=deg,
        campos=torch.tensor(sc["campos"]), prefiltered=False, debug=False)

    def run():
        T = lambda a: torch.tensor(a, device="cuda", requires_grad=True)
        ins = [T(sc["means3D"]), T(shs), T(sc["opacity"]), T(sc["scales"]), T(sc["rots"])]
        img, _ = dgr.GaussianRasterizer(raster_settings=rs)(means3D=ins[0], means2D=torch.zeros_like(ins[0]), opacities=ins[2],
                                                            shs=ins[1], colors_precomp=None, scales=ins[3], rotations=ins[4],
                                                            cov3D_precomp=None)
        img.backward(torch.from_numpy(g).cuda())
        return [t.grad.clone() for t in ins]

    with deterministic_algorithms():
        a, b = run(), run()
    dflt = run()
    for x, y, z in zip(a, b, dflt):
        assert torch.equal(x, y)
        assert rel_err(_np(x), _np(z)) <= 1e-5
    want = o.backward(ref, g.astype(np.float64))
    dsh = o.sh_backward(sc["means3D"], sc["campos"], shs, deg, cl, want["dL_dcolors"], want["dL_dmeans3D"])
    for got, exp in ((a[1], dsh), (a[0], want["dL_dmeans3D"]), (a[2], want["dL_dopacity"]), (a[3], want["dL_dscales"])):
        per = grad_err(_np(got), exp)
        assert int((per > GRAD_TOL).sum()) <= max(2, int(1e-3 * P)) and per.max() < 5e-2


def test_det_c2_and_2048_full_size_parity():
    sc = synth.stereo_pair_scene(1024)
    rep = _det_parity(sc, 5, "C2")
    assert rep[("f64", "dL_dmeans3D")]["P"] > 400_000
    sc = synth.stereo_pair_scene(512, render_res=2048, seed=77)
    assert sc["W"] == 2048
    rc = _run(sc)
    from gps_gaussian_b200 import _lib
    record("2048:det_workspace", P=rc.P, N=rc.num_rendered,
           bytes=int(_lib.lib.gpsg_rasterize_backward_workspace_bytes(rc.P, rc.num_rendered, 1, 0)))
    _det_parity(sc, 9, "2048", rc=rc)


# ---- 2./3. agreement with the default path and reproducibility on C2 -----------------------------------------------------
def test_det_c2_reproducible_across_runs_and_concurrent_load():
    from gps_gaussian_b200 import _lib
    sc = synth.stereo_pair_scene(1024)
    rc = _run(sc)
    g = torch.randn(3, 1024, 1024, device="cuda", generator=torch.Generator("cuda").manual_seed(1))
    first = _grad(rc, g)
    side = torch.cuda.Stream()
    x = torch.randn(4096, 4096, device="cuda")
    for i in range(4):
        if i >= 2:   # two of the runs share the GPU with a matmul loop on a second stream
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side):
                for _ in range(20):
                    x = (x @ x).tanh_()
        _assert_bitwise(first, _grad(rc, g), f"DET run {i + 2}")
        torch.cuda.synchronize()
    dflt = [_grad(rc, g, det=False) for _ in range(5)]
    differ = sum(any(not torch.equal(d[k], dflt[0][k]) for k in d) for d in dflt[1:])
    record("C2:default_backward_reruns_that_differ", differ=int(differ), of=4)
    print(f"default backward: {differ} of 4 reruns differed from the first")
    for k in first:
        assert rel_err(_np(first[k]), _np(dflt[0][k])) <= 1e-5, k
    ws = int(_lib.lib.gpsg_rasterize_backward_workspace_bytes(rc.P, rc.num_rendered, 1, 0))
    record("C2:det_workspace", P=rc.P, N=rc.num_rendered, bytes=ws)
    assert ws <= int(_lib.lib.gpsg_rasterize_backward_workspace_bytes(rc.P, 0, 0, 0)) + 320 * rc.num_rendered + 512


# ---- 4. permutation invariance ----------------------------------------------------------------------------------------
def test_det_gradients_are_permutation_equivariant():
    """With distinct depths the tile lists do not depend on the Gaussian ids, so permuting the inputs must permute the
    DET gradients exactly -- a check that does not depend on how the CTAs happen to be scheduled."""
    sc = synth.random_cube_scene(3000, 160, seed=31, bg=(0.1, 0.2, 0.3), scale_mul=2.0)
    rc = _run(sc)
    st = rc.state()
    vis = _np(rc.radii) > 0
    d = _np(st["depths"])[vis]
    assert np.unique(d).size == d.size, "scene has depth ties"
    perm = np.random.default_rng(2).permutation(3000)
    scp = dict(sc)
    for k in ("means3D", "colors", "opacity", "scales", "rots"):
        scp[k] = np.ascontiguousarray(sc[k][perm])
    rcp = _run(scp)
    assert torch.equal(rc.color, rcp.color) and rc.num_rendered == rcp.num_rendered
    g = torch.randn(3, 160, 160, device="cuda", generator=torch.Generator("cuda").manual_seed(4))
    a, b = _grad(rc, g), _grad(rcp, g)
    pt = torch.from_numpy(perm).cuda()
    for k in a:
        assert torch.equal(a[k][pt], b[k]), k


# ---- 5. binning path ------------------------------------------------------------------------------------------------
_RADIX_SCRIPT = r"""
import os, sys
sys.path[:0] = [{root!r}, os.path.join({root!r}, "gps-gaussian_b200", "dropin")]
import numpy as np, torch
from gps_gaussian_b200 import synth
from gps_gaussian_b200.introspect import RasterCall
for name, sc in ({scenes}):
    rc = RasterCall(sc); rc.forward()
    g = torch.from_numpy(np.random.default_rng(7).standard_normal((3, sc["H"], sc["W"])).astype(np.float32)).cuda()
    for k, v in rc.backward(g, want_cov3D=True, deterministic=True).items():
        if v is not None:
            np.save(os.path.join({out!r}, f"{{name}}_{{k}}.npy"), v.cpu().numpy())
"""
_SCENES = ('("c1", synth.random_cube_scene(10_000, 256)), '
           '("wide", synth.random_cube_scene(1500, 64, spread=0.6, scale_mul=4.0, seed=13, width=250, height=40, '
           'focal=(240.0, 190.0), principal=(118.0, 23.0), scale_modifier=0.7))')


def test_det_radix_binning_path_is_bit_identical(tmp_path):
    outs = {}
    for mode in ("bucket", "radix"):
        d = tmp_path / mode
        d.mkdir()
        env = dict(os.environ)
        env.pop("GPSG_BINNING", None)
        if mode == "radix":
            env["GPSG_BINNING"] = "radix"
        r = subprocess.run([sys.executable, "-c", _RADIX_SCRIPT.format(root=ROOT, scenes=_SCENES, out=str(d))], env=env,
                           cwd=ROOT, capture_output=True, text=True, timeout=600)
        assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-3000:]
        outs[mode] = {f.name: np.load(f) for f in sorted(d.iterdir())}
    assert len(outs["bucket"]) >= 12 and outs["bucket"].keys() == outs["radix"].keys()
    for name in outs["bucket"]:
        assert np.array_equal(outs["bucket"][name].view(np.uint32), outs["radix"][name].view(np.uint32)), name


# ---- 6. map ingest under the flag -------------------------------------------------------------------------------------
def _stereo_data(res, seed, requires_grad=True, batch=1):
    scs = [synth.stereo_pair_scene(res, keep_maps=True, seed=seed + b) for b in range(batch)]
    cam = [s["cam"] for s in scs]
    data = {"novel_view": {"FovX": torch.tensor([c["FovX"] for c in cam], dtype=torch.float64),
                           "FovY": torch.tensor([c["FovY"] for c in cam], dtype=torch.float64),
                           "width": torch.tensor([s["W"] for s in scs]), "height": torch.tensor([s["H"] for s in scs]),
                           "world_view_transform": torch.tensor(np.stack([c["world_view_transform"] for c in cam])),
                           "full_proj_transform": torch.tensor(np.stack([c["full_proj_transform"] for c in cam])),
                           "camera_center": torch.tensor(np.stack([c["camera_center"] for c in cam]))}}
    for v, name in enumerate(("lmain", "rmain")):
        T = lambda key: torch.tensor(np.stack([s["views"][v][key] for s in scs])).cuda().requires_grad_(requires_grad)
        data[name] = {"img": T("img"), "xyz": T("xyz"), "rot_maps": T("rot_maps"), "scale_maps": T("scale_maps"),
                      "opacity_maps": T("opacity_maps"),
                      "pts_valid": torch.tensor(np.stack([s["views"][v]["valid"] for s in scs])).cuda()}
    return data


MAP_KEYS = ("xyz", "img", "rot_maps", "scale_maps", "opacity_maps")


def _map_grads(fn, res, seed, g, batch=1):
    data = _stereo_data(res, seed, batch=batch)
    out = fn(data, [0.1, 0.2, 0.3])["novel_view"]["img_pred"]
    (out * g).sum().backward()
    return out.detach(), {(v, k): data[v][k].grad.clone() for v in ("lmain", "rmain") for k in MAP_KEYS}


def test_det_map_ingest_matches_gather_path_bitwise():
    from gps_gaussian_b200.GaussianRender import pts2render, pts2render_gather
    g = torch.randn(1, 3, 128, 128, device="cuda", generator=torch.Generator("cuda").manual_seed(3))
    with deterministic_algorithms():
        img_m, gm = _map_grads(pts2render, 128, 4242, g)
        img_m2, gm2 = _map_grads(pts2render, 128, 4242, g)
        img_g, gg = _map_grads(pts2render_gather, 128, 4242, g)
    assert torch.equal(img_m, img_g) and torch.equal(img_m, img_m2)
    _assert_bitwise(gm, gm2, "maps rerun")
    _assert_bitwise(gm, gg, "maps vs gather")
    img_off, goff = _map_grads(pts2render, 128, 4242, g)        # default path: same image, gradients within 1e-5
    assert torch.equal(img_off, img_m)
    for k in gm:
        assert rel_err(_np(goff[k]), _np(gm[k])) <= 1e-5, k


def test_det_map_ingest_batch_of_two_is_two_batches_of_one():
    from gps_gaussian_b200.GaussianRender import pts2render
    g = torch.randn(2, 3, 96, 96, device="cuda", generator=torch.Generator("cuda").manual_seed(5))
    with deterministic_algorithms():
        img2, g2 = _map_grads(pts2render, 96, 100, g, batch=2)
        for b in range(2):
            img1, g1 = _map_grads(pts2render, 96, 100 + b, g[b:b + 1])
            assert torch.equal(img2[b:b + 1], img1)
            for k in g1:
                assert torch.equal(g2[k][b:b + 1], g1[k]), (b, k)


# ---- 7. drop-in module under the flag ---------------------------------------------------------------------------------
def test_det_dropin_equals_capi_bitwise():
    import diff_gaussian_rasterization as dgr
    sc = synth.random_cube_scene(5000, 160, seed=6, bg=(0.1, 0.2, 0.3), **dict(WIDE, scale_modifier=0.8))
    H, W = sc["H"], sc["W"]
    rc = _run(sc)
    T = lambda a: torch.tensor(a, device="cuda", requires_grad=True)
    m, c, op, s, r = T(sc["means3D"]), T(sc["colors"]), T(sc["opacity"]), T(sc["scales"]), T(sc["rots"])
    m2d = torch.zeros_like(m, requires_grad=True)
    rs = dgr.GaussianRasterizationSettings(
        image_height=H, image_width=W, tanfovx=sc["tanfovx"], tanfovy=sc["tanfovy"], bg=torch.tensor(sc["bg"], device="cuda"),
        scale_modifier=sc["scale_modifier"], viewmatrix=torch.tensor(sc["view"]), projmatrix=torch.tensor(sc["proj"]),
        sh_degree=3, campos=torch.tensor(sc["campos"]), prefiltered=False, debug=False)
    g = torch.randn(3, H, W, device="cuda", generator=torch.Generator("cuda").manual_seed(8))
    with deterministic_algorithms():
        img, _ = dgr.GaussianRasterizer(raster_settings=rs)(means3D=m, means2D=m2d, opacities=op, shs=None,
                                                            colors_precomp=c, scales=s, rotations=r, cov3D_precomp=None)
        img.backward(g)
    assert torch.equal(img, rc.color)
    want = rc.backward(g, deterministic=True)
    for got, k in ((m.grad, "dL_dmeans3D"), (c.grad, "dL_dcolors"), (op.grad, "dL_dopacity"), (s.grad, "dL_dscales"),
                   (r.grad, "dL_drots"), (m2d.grad, "dL_dmeans2D")):
        assert torch.equal(got, want[k].view_as(got)), k


# ---- 8. the whole stack under the flag ------------------------------------------------------------------------------
def test_whole_stack_runs_under_the_flag_and_is_bit_reproducible():
    from gps_gaussian_b200.corr import CorrBlockFast1D
    from gps_gaussian_b200.loss import fused_l1_ssim
    from gps_gaussian_b200.unproject import unproject_view
    from gps_gaussian_b200.GaussianRender import pts2render
    gen = torch.Generator("cuda").manual_seed(11)
    f1 = torch.randn(2, 64, 32, 64, device="cuda", generator=gen).half()
    f2 = torch.randn(2, 64, 32, 64, device="cuda", generator=gen).half()
    coords = torch.rand(2, 2, 32, 64, device="cuda", generator=gen) * 64
    G = np.load(os.path.join(ROOT, "tests", "golden", "unproject_golden.npz"))
    Tg = lambda k: torch.tensor(G[k], dtype=torch.float32, device="cuda")
    img = torch.rand(2, 3, 64, 64, device="cuda", generator=gen)
    gt = torch.rand(2, 3, 64, 64, device="cuda", generator=gen)
    gmap = torch.randn(1, 3, 96, 96, device="cuda", generator=gen)

    def step():
        outs, grads = {}, {}
        a, b = f1.clone().requires_grad_(True), f2.clone().requires_grad_(True)
        blk = CorrBlockFast1D(a, b, num_levels=4, radius=4)
        looks = [blk(coords + i) for i in range(3)]
        sum((l.float() * (i + 1)).sum() for i, l in enumerate(looks)).backward()
        outs["corr"], grads["fmap1"], grads["fmap2"] = torch.cat(looks, 1).detach(), a.grad, b.grad
        flow = Tg("flow").requires_grad_(True)
        depth, xyz, _ = unproject_view({"flow_pred": flow, "mask": Tg("mask"), "intr": Tg("intr"), "extr": Tg("extr"),
                                        "ref_intr": Tg("ref_intr"), "Tf_x": Tg("tf_x")})
        ((xyz * Tg("g_xyz")).sum() + (depth * Tg("g_depth")).sum()).backward()
        outs["xyz"], grads["flow"] = xyz.detach(), flow.grad
        out, mg = _map_grads(pts2render, 96, 7, gmap)
        outs["render"] = out
        grads.update({f"map:{v}:{k}": t for (v, k), t in mg.items()})
        x = img.clone().requires_grad_(True)
        loss = fused_l1_ssim(x, gt)
        loss.backward()
        outs["loss"], grads["loss_img"] = loss.detach(), x.grad
        return outs, grads

    off_outs, _ = step()
    with deterministic_algorithms():
        o1, g1 = step()
        o2, g2 = step()
    _assert_bitwise(g1, g2, "leaf gradients under the flag")
    _assert_bitwise(o1, o2, "outputs under the flag")
    _assert_bitwise(o1, off_outs, "outputs with and without the flag")


# ---- 9. degenerate inputs -------------------------------------------------------------------------------------------
def test_det_empty_and_all_culled():
    sc = synth.random_cube_scene(64, 96, bg=(0.2, 0.4, 0.6))
    empty = dict(sc)
    for k in ("means3D", "colors", "scales"):
        empty[k] = np.zeros((0, 3), np.float32)
    empty["rots"] = np.zeros((0, 4), np.float32); empty["opacity"] = np.zeros((0, 1), np.float32)
    rc = _run(empty)
    assert rc.num_rendered == 0
    g = rc.backward(torch.ones_like(rc.color), deterministic=True)
    assert all(v.numel() == 0 for v in g.values() if v is not None)
    behind = dict(sc)
    behind["means3D"] = (sc["means3D"] + (sc["campos"] - np.array([0, 0.85, 0], np.float32)) * 3).astype(np.float32)
    rc = _run(behind)
    assert rc.num_rendered == 0
    with deterministic_algorithms():
        g = rc.backward(torch.ones_like(rc.color))
    assert all(float(v.abs().sum()) == 0 for v in g.values() if v is not None)
