"""GPU: aux mode of the rasterizer -- expected depth and alpha beside the colour image (the out_depth / out_alpha outputs
of gpsg_rasterize_forward, the aux gradients of gpsg_rasterize_backward and the Python layers above them).

Depth is a fourth colour channel (colour z, background 0) and alpha = 1 - T_final is 1 + the colour image of a scene with
black Gaussians on the background (-1, 0, 0).  The oracles therefore check aux mode with their existing entry points:
  forward   the fp32 oracle composites colours (z, z, z) on a black background (same op order as the device's depth);
  backward  the aux backward is linear in (g_rgb, g_D, g_A): the fp64 oracle's backward of the colour image, plus its
            backward of the depth image (whose colour gradient is dL/dz, taken to dL/dmeans3D through the view matrix's
            third row), plus its backward of the alpha image, all on the device's own forward decisions."""
import numpy as np
import pytest
import torch

from gps_gaussian_b200 import _lib, synth
from gps_gaussian_b200.introspect import RasterCall
from helpers import (GRAD_TOL, SHARED_TOL, TAINT_CAP, EPS_ALPHA_F64, _threads, assert_image_parity, forced_backward,
                     grad_err, oracle_forward, record)

pytestmark = pytest.mark.gpu

WIDE = dict(width=250, height=40, focal=(240.0, 190.0), principal=(118.0, 23.0))
TALL = dict(width=40, height=250, focal=(150.0, 260.0), principal=(21.0, 130.0))


def _np(t):
    return t.detach().cpu().numpy()


class AuxCall(RasterCall):
    """RasterCall with the aux forward / backward."""

    def forward_aux(self):
        self.depth = torch.empty((self.H, self.W), dtype=torch.float32, device=self.device)
        self.alpha = torch.empty((self.H, self.W), dtype=torch.float32, device=self.device)
        self.num_rendered, self.bufs = _lib.rasterize_forward(self.settings, self.color, self.radii, out_depth=self.depth,
                                                              out_alpha=self.alpha, **self._inputs())
        return self.color, self.depth, self.alpha

    def backward_aux(self, g_rgb, g_D, g_A, deterministic=False):
        out = _lib.rasterize_backward(self.settings, self.num_rendered, self.bufs, self.radii, g_rgb, want_cov3D=True,
                                      deterministic=deterministic, grad_depth=g_D, grad_alpha=g_A, **self._inputs())
        return {k: v.clone() for k, v in out.items() if v is not None}


def _pair(sc):
    """(plain RasterCall after its forward, AuxCall after its aux forward) on the same inputs."""
    plain = RasterCall(sc)
    plain.forward()
    aux = AuxCall(sc, dev_inputs=plain.inp)
    aux.forward_aux()
    torch.cuda.synchronize()
    return plain, aux


def _check_forward(tag, sc):
    plain, aux = _pair(sc)
    ps, st = plain.state(), aux.state()
    assert torch.equal(plain.color, aux.color) and torch.equal(plain.radii, aux.radii), tag
    assert torch.equal(ps["final_T"], st["final_T"]) and torch.equal(ps["n_contrib"], st["n_contrib"]), tag
    assert torch.equal(aux.alpha, 1.0 - st["final_T"]), tag                       # the same T, bit for bit
    o, ref = oracle_forward(sc, "f32", nthreads=_threads())
    vis = ref["radii"] > 0
    assert np.array_equal(_np(st["depths"])[vis], ref["depth"].astype(np.float32)[vis]), tag
    # depth == the fp32 oracle compositing colours (z, z, z) over a black background, under the threshold-margin rules
    z = ref["depth"].astype(np.float32)
    zs = float(max(z.max(), 1e-30))
    dref = dict(ref, inputs=dict(ref["inputs"], colors=np.repeat(z[:, None] / zs, 3, 1).astype(np.float32),
                                 bg=np.zeros(3, np.float32)))
    dimg = o.render_state(dref, nthreads=_threads())
    assert np.array_equal(dimg["final_T"], ref["final_T"])
    dd = _np(aux.depth) / zs
    assert_image_parity(tag + ":depth", np.repeat(dd[None], 3, 0), _np(st["final_T"]), _np(st["n_contrib"]).view(np.uint32),
                        o, dict(ref, color=dimg["color"]))
    return plain, aux, ref


SCENES = {
    "C1": lambda: synth.random_cube_scene(10_000, 256),
    "250x40-mod0.7": lambda: synth.random_cube_scene(1500, 64, spread=0.6, scale_mul=4.0, bg=(0.3, 0.6, 0.9), seed=13,
                                                     **dict(WIDE, scale_modifier=0.7)),
    "40x250-mod1.6": lambda: synth.random_cube_scene(1500, 64, spread=0.6, scale_mul=4.0, seed=13,
                                                     **dict(TALL, scale_modifier=1.6)),
    "120x48-clamp": lambda: synth.random_cube_scene(3000, 64, spread=3.0, scale_mul=5.0, seed=13, width=120, height=48,
                                                    focal=(70.0, 52.0), principal=(66.0, 20.0), scale_modifier=1.3),
    "radix-tile": lambda: synth.random_cube_scene(30000, 48, spread=0.25, scale_mul=1.0, seed=13),
}


@pytest.mark.parametrize("name", list(SCENES))
def test_aux_forward_matches_plain_forward_and_oracle(name):
    sc = SCENES[name]()
    _, aux, _ = _check_forward(name, sc)
    if name == "radix-tile":
        r = aux.state()["ranges"].to(torch.int64)
        assert int((r[:, 1] - r[:, 0]).max()) > 4096                          # the global radix binning path


def test_aux_forward_cov3d_precomp_and_2048():
    sc = synth.random_cube_scene(3000, 128, seed=5)
    _, ref = oracle_forward(sc, "f32")
    _check_forward("cov3D_precomp", dict(sc, cov3D_precomp=ref["cov3D"].copy(), scales=None, rots=None))
    _check_forward("2048", synth.random_cube_scene(60_000, 2048, seed=3, scale_mul=2.0))


def test_aux_forward_empty_scene():
    sc = synth.random_cube_scene(10, 64, seed=1)
    sc = dict(sc, **{k: sc[k][:0] for k in ("means3D", "colors", "opacity", "scales", "rots")})     # P = 0
    plain, aux = _pair(sc)
    assert float(aux.depth.abs().max()) == 0.0 and float(aux.alpha.abs().max()) == 0.0
    assert torch.equal(plain.color, aux.color)


# ---- gradients ------------------------------------------------------------------------------------------------------
def _fp64_aux_backward(sc, base, final_T, n_contrib, g_rgb, g_D, g_A):
    """The aux gradients in fp64 on the device's forward decisions, by linearity (see the module docstring), with the
    threshold-margin classes of the forward state."""
    o, st, want = forced_backward(sc, "f64", base, final_T, n_contrib, g_rgb)
    z = st["depth"].astype(np.float64)
    zero = np.zeros_like(g_D)
    P = z.shape[0]
    scd = dict(sc, colors=np.stack([z, np.zeros(P), np.zeros(P)], 1), bg=np.zeros(3))
    _, _, wd = forced_backward(scd, "f64", base, final_T, n_contrib, np.stack([g_D, zero, zero]))
    sca = dict(sc, colors=np.zeros((P, 3)), bg=np.array([-1.0, 0.0, 0.0]))
    _, _, wa = forced_backward(sca, "f64", base, final_T, n_contrib, np.stack([g_A, zero, zero]))
    view = np.asarray(sc["view"], np.float64).reshape(16)
    tot = {k: want[k] + wd[k] + wa[k] for k in want if k != "dL_dcolors"}
    tot["dL_dcolors"] = want["dL_dcolors"]
    dz = wd["dL_dcolors"][:, 0] * (np.asarray(base["radii"]) > 0)
    tot["dL_dmeans3D"] = tot["dL_dmeans3D"] + dz[:, None] * view[[2, 6, 10]][None]
    m = o.margins(st, eps=dict(T=0.0, alpha=EPS_ALPHA_F64), nthreads=_threads())
    return tot, m


KEYS = (("dL_dmeans3D", "dL_dmeans3D"), ("dL_dcolors", "dL_dcolors"), ("dL_dopacity", "dL_dopacity"),
        ("dL_dscales", "dL_dscales"), ("dL_drots", "dL_drots"), ("dL_dmeans2D", "dL_dmean2D"), ("dL_dcov3D", "dL_dcov3D"))


def _check_grads(tag, sc, seed=0):
    _, aux = _pair(sc)
    st = aux.state()
    _, base = oracle_forward(sc, "f32", render=False)
    rng = np.random.default_rng(seed)
    H, W = sc["H"], sc["W"]
    g_rgb = rng.standard_normal((3, H, W)).astype(np.float32)
    g_D = rng.standard_normal((H, W)).astype(np.float32)
    g_A = rng.standard_normal((H, W)).astype(np.float32)
    cu = lambda a: torch.from_numpy(a).cuda()
    want, m = _fp64_aux_backward(sc, base, _np(st["final_T"]), _np(st["n_contrib"]).view(np.uint32), g_rgb, g_D, g_A)
    own, shared, clean = m["taint_own"], m["taint"] & ~m["taint_own"], ~m["taint"]
    got_all = {}
    for det in (False, True):
        got = aux.backward_aux(cu(g_rgb), cu(g_D), cu(g_A), deterministic=det)
        got_all[det] = got
        for kg, kr in KEYS:
            if kg not in got:
                continue
            a = _np(got[kg])
            if kg == "dL_dmeans2D":
                a = a[:, :2]
            per = grad_err(a, want[kr])
            mx = lambda msk: float(per[msk].max()) if msk.any() else 0.0
            rec = dict(det=det, clean=int(clean.sum()), shared=int(shared.sum()), own=int(own.sum()),
                       max_err_clean=mx(clean), max_err_shared=mx(shared), max_err_own=mx(own))
            record(f"{tag}:aux-grad:{kg}", **rec)
            assert rec["max_err_clean"] <= GRAD_TOL, (tag, kg, rec)
            assert rec["max_err_shared"] <= SHARED_TOL, (tag, kg, rec)
            assert rec["max_err_own"] <= TAINT_CAP, (tag, kg, rec)
    # deterministic: reruns bit-identical; g_D = g_A = 0 gives exactly the non-aux deterministic backward
    again = aux.backward_aux(cu(g_rgb), cu(g_D), cu(g_A), deterministic=True)
    for k in got_all[True]:
        assert torch.equal(again[k], got_all[True][k]), (tag, k)
    zero = torch.zeros((H, W), device="cuda")
    z_aux = aux.backward_aux(cu(g_rgb), zero, zero, deterministic=True)
    plain = aux.backward(cu(g_rgb), want_cov3D=True, deterministic=True)
    for k in z_aux:
        assert torch.equal(z_aux[k], plain[k]), (tag, k)
    return got_all


@pytest.mark.parametrize("name", ["C1", "250x40-mod0.7", "40x250-mod1.6", "120x48-clamp", "radix-tile"])
def test_aux_backward_against_fp64(name):
    _check_grads(name, SCENES[name]())


def test_aux_backward_cov3d_precomp():
    sc = synth.random_cube_scene(3000, 128, seed=5)
    _, ref = oracle_forward(sc, "f32")
    _check_grads("cov3D_precomp", dict(sc, cov3D_precomp=ref["cov3D"].copy(), scales=None, rots=None), seed=2)


def test_aux_sh_degree3_through_the_dropin():
    """SH colours through rasterize_gaussians_aux: image bit-identical to rasterize_gaussians, and a depth + alpha loss
    gives the same gradients as the non-aux path plus the aux-only terms (checked by zero aux gradients: equal)."""
    import diff_gaussian_rasterization as dgr
    P, res, M = 4000, 128, 16
    sc = synth.random_cube_scene(P, res, seed=17, bg=(0.1, 0.2, 0.3), scale_mul=2.0)
    rng = np.random.default_rng(5)
    shs = torch.from_numpy((rng.standard_normal((P, M, 3)) * 0.5).astype(np.float32)).cuda()
    cu = lambda k: torch.from_numpy(np.ascontiguousarray(sc[k], np.float32)).cuda()
    rs = dgr.GaussianRasterizationSettings(sc["H"], sc["W"], sc["tanfovx"], sc["tanfovy"], torch.tensor(sc["bg"]).float(),
                                           1.0, torch.from_numpy(np.asarray(sc["view"], np.float32).reshape(4, 4)),
                                           torch.from_numpy(np.asarray(sc["proj"], np.float32).reshape(4, 4)), 3,
                                           torch.from_numpy(np.asarray(sc["campos"], np.float32)), False, False)
    e = torch.Tensor([])

    def run(aux, gw):
        ins = [cu("means3D").requires_grad_(True), shs.clone().requires_grad_(True), cu("opacity").reshape(-1, 1).requires_grad_(True),
               cu("scales").requires_grad_(True), cu("rots").requires_grad_(True)]
        m2 = torch.zeros_like(ins[0], requires_grad=True)
        if aux:
            img, depth, alpha, radii = dgr.rasterize_gaussians_aux(ins[0], m2, ins[1], e, ins[2], ins[3], ins[4], e, rs)
            maps.append((depth.detach(), alpha.detach()))
            loss = (img * gw[0]).sum() + (depth * gw[1]).sum() + (alpha * gw[2]).sum()
        else:
            img, radii = dgr.rasterize_gaussians(ins[0], m2, ins[1], e, ins[2], ins[3], ins[4], e, rs)
            loss = (img * gw[0]).sum()
        loss.backward()
        return img, [t.grad for t in ins]

    maps = []
    g = torch.randn(3, res, res, device="cuda", generator=torch.Generator("cuda").manual_seed(1))
    zero = torch.zeros(res, res, device="cuda")
    was = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        img0, g0 = run(False, (g,))
        img1, g1 = run(True, (g, zero, zero))
        img2, g2 = run(True, (g, torch.randn_like(zero), torch.randn_like(zero)))
    finally:
        torch.use_deterministic_algorithms(was)
    assert torch.equal(img0, img1) and torch.equal(img0, img2)
    for a, b in zip(g0, g1):
        assert torch.equal(a, b)
    assert any(not torch.equal(a, b) for a, b in zip(g0, g2))
    # depth and alpha do not depend on the colour source: the SH path's equal the colors_precomp aux forward's, which
    # test_aux_forward_matches_plain_forward_and_oracle holds to the oracle
    pre = AuxCall(sc)
    pre.forward_aux()
    for d, a in maps:
        assert torch.equal(d, pre.depth) and torch.equal(a, pre.alpha)


# ---- map ingest ------------------------------------------------------------------------------------------------------
def test_pts2render_aux_equals_render_aux_gather_and_batches():
    """pts2render_aux (fused map ingest) == gather -> render_aux bit for bit in the forward; map-layout gradients of a
    loss on all three outputs agree with the gather path, with invalid pixels exactly 0; a batch of two == two batches
    of one, with one host synchronisation per batch."""
    from test_raster_gpu import _stereo_data
    from gps_gaussian_b200.GaussianRender import pts2render, pts2render_aux, _VIEWS
    from gps_gaussian_b200.gaussian_renderer import render_aux
    res = 96
    keys = ("xyz", "img", "rot_maps", "scale_maps", "opacity_maps")
    sc, data = _stereo_data(res, requires_grad=True, seed=11)
    H, W = sc["H"], sc["W"]
    gen = torch.Generator("cuda").manual_seed(3)
    gw = [torch.randn(1, c, H, W, device="cuda", generator=gen) for c in (3, 1, 1)]
    nv = pts2render_aux(data, [0.1, 0.2, 0.3])["novel_view"]
    img, depth, alpha = nv["img_pred"], nv["depth_pred"], nv["alpha_pred"]
    assert depth.shape == (1, 1, H, W) and alpha.shape == (1, 1, H, W)
    with torch.no_grad():
        assert torch.equal(pts2render(data, [0.1, 0.2, 0.3])["novel_view"]["img_pred"], img)
    ((img * gw[0]).sum() + (depth * gw[1]).sum() + (alpha * gw[2]).sum()).backward()
    fused = {(v, k): data[v][k].grad.clone() for v in _VIEWS for k in keys}
    # gather path on fresh leaves
    _, d2 = _stereo_data(res, requires_grad=True, seed=11)
    parts = {k: [] for k in ('xyz', 'rgb', 'rot', 'scale', 'opacity')}
    for v in _VIEWS:
        d = d2[v]
        valid = d['pts_valid'][0, :]
        parts['xyz'].append(d['xyz'][0][valid].view(-1, 3))
        parts['rgb'].append(d['img'][0].permute(1, 2, 0).reshape(-1, 3)[valid].view(-1, 3))
        parts['rot'].append(d['rot_maps'][0].permute(1, 2, 0).reshape(-1, 4)[valid].view(-1, 4))
        parts['scale'].append(d['scale_maps'][0].permute(1, 2, 0).reshape(-1, 3)[valid].view(-1, 3))
        parts['opacity'].append(d['opacity_maps'][0].permute(1, 2, 0).reshape(-1, 1)[valid].view(-1, 1))
    cat = lambda k: torch.cat(parts[k], 0)
    i2, d2_, a2 = render_aux(d2, 0, cat('xyz'), cat('rgb') * 0.5 + 0.5, cat('rot'), cat('scale'), cat('opacity'),
                             [0.1, 0.2, 0.3])
    assert torch.equal(i2, img[0]) and torch.equal(d2_, depth[0]) and torch.equal(a2, alpha[0])
    ((i2 * gw[0][0]).sum() + (d2_ * gw[1][0]).sum() + (a2 * gw[2][0]).sum()).backward()
    for v in _VIEWS:
        inval = ~d2[v]['pts_valid'][0].reshape(-1)
        for k in keys:
            a, b = fused[(v, k)], d2[v][k].grad
            assert float((a - b).abs().max()) <= 1e-5 * max(1e-20, float(b.abs().max())), (v, k)   # atomics order only
            flat = a[0].reshape(a.shape[1], -1) if k != "xyz" else a[0].reshape(-1, 3).t()
            assert float(flat[:, inval].abs().max()) == 0.0, (v, k)
    # a batch of two == two batches of one; one host synchronisation per batch
    syncs = []
    orig = torch.cuda.Stream.synchronize
    torch.cuda.Stream.synchronize = lambda self: (syncs.append(1), orig(self))[1]
    try:
        singles = [pts2render_aux(_stereo_data(res, seed=sd)[1], [0.1, 0.2, 0.3])["novel_view"] for sd in (11, 12)]
        assert len(syncs) == 2
        syncs.clear()
        b0, b1 = (_stereo_data(res, seed=sd)[1] for sd in (11, 12))
        batch = {"novel_view": {k: torch.cat([b0["novel_view"][k], b1["novel_view"][k]]) for k in b0["novel_view"]}}
        for v in _VIEWS:
            batch[v] = {k: torch.cat([b0[v][k], b1[v][k]]) for k in b0[v]}
        out = pts2render_aux(batch, [0.1, 0.2, 0.3])["novel_view"]
        assert len(syncs) == 1
    finally:
        torch.cuda.Stream.synchronize = orig
    for key in ("img_pred", "depth_pred", "alpha_pred"):
        assert torch.equal(out[key][0:1], singles[0][key]) and torch.equal(out[key][1:2], singles[1][key]), key
