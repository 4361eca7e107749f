"""Reference of the anti-aliased (GPSG_FWD_ANTIALIAS) rasterizer for the tests, built on the unchanged oracles.

Anti-aliasing only replaces each splat's opacity o by o' = o * rho, rho = sqrt(max(2.5e-5, det S / det(S + 0.3 I))), S the
screen covariance before the 0.3 px^2 dilation; conics, radii, tile lists and sort keys do not change.  So:

  forward   the C oracle (oracle/raster_oracle.py) run on the opacities o' is the anti-aliased forward.  `rho` restates
            the projection's (a0, b, c0) in the device's fixed fp32 op order (raster_preprocess.cu, no FMA) from the
            oracle's own Sigma3D, so o' in fp32 is bit-identical to conic_opacity.w of the device; the restatement is
            checked on every call against the oracle's conic, which it must reproduce bit for bit.
  backward  the oracle backward on o' gives dL/do' and the conic / position chain; the anti-aliasing chain
            (dL/do = rho dL/do' and the rho term through cov2D -> Sigma3D -> scale / rotation / means3D) is added by fp64
            autograd of sum_i stopgrad(dL/do'_i o_i) rho_i(theta) (`aa_backward`).
  truth     fp64 autograd of the whole forward (`render_autograd_aa`): raster_torch64.render_autograd fed with
            o * rho(theta), so the derivative of rho is autograd's, not a restatement of the kernel's formula.
"""
import numpy as np
import torch

from helpers import forced_backward, oracle_forward
from oracle import raster_torch64 as rt

RHO_FLOOR = float(np.float32(0.000025))     # rho^2 floor (rho >= 0.005), the kernel's fp32 constant


def _k(dt, v):
    """A constant as the kernel and the oracle (RC) write it: fp32-rounded, then in precision dt."""
    return dt(np.float32(v))


def _cam32(sc, dt):
    v = np.asarray(sc["view"], dt).reshape(16)
    tx, ty = dt(sc["tanfovx"]), dt(sc["tanfovy"])
    fx = dt(sc["W"]) / (_k(dt, 2.0) * tx)
    fy = dt(sc["H"]) / (_k(dt, 2.0) * ty)
    return v, tx, ty, fx, fy


def screen_cov(sc, means3D, c6, dtype=np.float32):
    """(a0, b, c0) [P] each: the screen covariance before the dilation, in the device's op order and precision `dtype`
    (np.float32: the preprocess kernel's rounding; np.float64: fp64)."""
    dt = dtype
    v, tanx, tany, fx, fy = _cam32(sc, dt)
    m = np.asarray(means3D, dt).reshape(-1, 3)
    S = np.asarray(c6, dt).reshape(-1, 6)
    x, y, z = m[:, 0], m[:, 1], m[:, 2]
    with np.errstate(all="ignore"):
        tvx = ((v[0] * x + v[4] * y) + v[8] * z) + v[12]
        tvy = ((v[1] * x + v[5] * y) + v[9] * z) + v[13]
        tvz = ((v[2] * x + v[6] * y) + v[10] * z) + v[14]
        limx, limy = _k(dt, 1.3) * tanx, _k(dt, 1.3) * tany
        txc = np.minimum(limx, np.maximum(-limx, tvx / tvz)) * tvz
        tyc = np.minimum(limy, np.maximum(-limy, tvy / tvz)) * tvz
        J00, J02 = fx / tvz, -(fx * txc) / (tvz * tvz)
        J11, J12 = fy / tvz, -(fy * tyc) / (tvz * tvz)
        A = [v[k * 4 + 0] * J00 + v[k * 4 + 2] * J02 for k in range(3)] + \
            [v[k * 4 + 1] * J11 + v[k * 4 + 2] * J12 for k in range(3)]
        S00, S01, S02, S11, S12, S22 = (S[:, k] for k in range(6))
        B00 = (A[0] * S00 + A[1] * S01) + A[2] * S02
        B01 = (A[0] * S01 + A[1] * S11) + A[2] * S12
        B02 = (A[0] * S02 + A[1] * S12) + A[2] * S22
        B10 = (A[3] * S00 + A[4] * S01) + A[5] * S02
        B11 = (A[3] * S01 + A[4] * S11) + A[5] * S12
        B12 = (A[3] * S02 + A[4] * S12) + A[5] * S22
        a0 = (B00 * A[0] + B01 * A[1]) + B02 * A[2]
        b = (B00 * A[3] + B01 * A[4]) + B02 * A[5]
        c0 = (B10 * A[3] + B11 * A[4]) + B12 * A[5]
    return a0, b, c0


def rho_from_abc(a0, b, c0, dtype=np.float32):
    """rho in the kernel's op order: sqrt(max(2.5e-5, (a0 c0 - b^2) / ((a0 + 0.3)(c0 + 0.3) - b^2)))."""
    dt = dtype
    k03 = _k(dt, 0.3)
    with np.errstate(all="ignore"):
        a, c = a0 + k03, c0 + k03
        det = a * c - b * b
        det0 = a0 * c0 - b * b
        return np.sqrt(np.maximum(_k(dt, RHO_FLOOR), det0 / det)), det


def rho(sc, st, dtype=np.float32):
    """rho [P] of the visible Gaussians of oracle state `st` (0 for culled ones), from the state's own Sigma3D, checked
    against the state's conic bit for bit (fp32) or to rounding (fp64)."""
    dt = dtype
    vis = np.asarray(st["radii"]) > 0
    a0, b, c0 = screen_cov(sc, st["inputs"]["means3D"], st["cov3D"], dt)
    r, det = rho_from_abc(a0, b, c0, dt)
    with np.errstate(all="ignore"):
        det_inv = dt(1.0) / det
        con = np.stack([(c0 + _k(dt, 0.3)) * det_inv, -b * det_inv, (a0 + _k(dt, 0.3)) * det_inv], 1)
    want = np.asarray(st["conic_opacity"])[:, :3]
    if dt is np.float32:
        assert np.array_equal(con[vis].astype(np.float32), want[vis]), "fp32 restatement of the projection drifted"
    else:
        scale = np.abs(want[vis]).max(1, keepdims=True) if vis.any() else 1.0
        assert (np.abs(con[vis] - want[vis]) <= 1e-12 * scale).all(), "fp64 restatement of the projection drifted"
    return np.where(vis, r, dt(0)).astype(dt)


def aa_opacity(sc, dtype="f32"):
    """(o' [P] in the oracle's precision, rho [P]) of scene `sc`."""
    _, st = oracle_forward(sc, dtype, render=False)
    dt = np.float32 if dtype == "f32" else np.float64
    r = rho(sc, st, dt)
    o = np.asarray(sc["opacity"], dt).reshape(-1)
    return (o * r).astype(dt), r


def aa_forward(sc, dtype="f32", nthreads=8, render=True):
    """(oracle, state, rho) of the anti-aliased forward of `sc` in `dtype`: the oracle on o * rho."""
    op, r = aa_opacity(sc, dtype)
    o, st = oracle_forward(dict(sc, opacity=op.reshape(np.asarray(sc["opacity"]).shape)), dtype, nthreads, render)
    return o, st, r


def independent_aa_forward(sc):
    """The anti-aliased forward through oracle/raster_independent.py (numpy, matrix form, shares nothing with
    gpsg_oracle.c or with `rho` above): rho from that restatement's own conic C = (S + 0.3 I)^-1 as
    rho^2 = det S / det(S + 0.3 I) = det(I - 0.3 C), and its compositing run on o * rho."""
    from oracle import raster_independent as ri
    g = ri.project(sc["means3D"], sc["scales"], sc["rots"], sc["opacity"], sc["view"], sc["proj"], sc["tanfovx"],
                   sc["tanfovy"], sc["W"], sc["H"], sc.get("scale_modifier", 1.0))
    k = float(np.float32(0.3))
    cx, cy, cz = g["conic"][:, 0], g["conic"][:, 1], g["conic"][:, 2]
    rho = np.where(g["visible"], np.sqrt(np.maximum(RHO_FLOOR, (1 - k * cx) * (1 - k * cz) - k * k * cy * cy)), 0.0)
    op = np.asarray(sc["opacity"], np.float64).reshape(-1) * rho
    keys, plist, ranges = ri.bin_tiles(g)
    img, final_T, n_contrib = ri.composite(g, plist, ranges, sc["colors"], op, sc["bg"], sc["W"], sc["H"])
    rect = g["rect"]
    return dict(radii=g["radii"], means2D=g["pix"], conic=g["conic"], rho=rho, opacity=op,
                tiles_touched=np.where(g["visible"], (rect[:, 2] - rect[:, 0]) * (rect[:, 3] - rect[:, 1]), 0).astype(np.uint32),
                keys=keys, point_list=plist, ranges=ranges, num_rendered=int(keys.size), color=img, final_T=final_T,
                n_contrib=n_contrib)


def _theta(sc):
    t = lambda k: torch.tensor(np.asarray(sc[k], np.float64), dtype=torch.float64, requires_grad=True) \
        if sc.get(k) is not None else None
    return dict(means3D=t("means3D"), scales=t("scales"), rots=t("rots"), cov3D=t("cov3D_precomp"))


def rho_torch(cam, means3D, c6):
    """fp64 differentiable rho [P] (floor included) of Gaussians (means3D [P,3], Sigma3D [P,6])."""
    _, _, _, abc = rt.project(cam, means3D, c6)
    k03 = float(np.float32(0.3))
    a, b, c = abc[:, 0], abc[:, 1], abc[:, 2]
    a0, c0 = a - k03, c - k03
    r = (a0 * c0 - b * b) / (a * c - b * b)
    return torch.sqrt(torch.clamp(r, min=RHO_FLOOR))


def _c6(sc, th):
    return th["cov3D"] if th["cov3D"] is not None else rt.cov3d(th["scales"], th["rots"], float(sc.get("scale_modifier", 1.0)))


def aa_backward(sc, st, grads):
    """Adds the anti-aliasing chain to an oracle backward `grads` taken on the o' state `st` (in place; returns grads):
    dL/do = rho dL/do' and the rho term through Sigma2D -> Sigma3D / scale / rotation -> means3D, by fp64 autograd of
    sum_i stopgrad(dL/do'_i o_i) rho_i(theta)."""
    th = _theta(sc)
    cam = rt.camera(st)
    c6 = _c6(sc, th)
    r = rho_torch(cam, th["means3D"], c6)
    vis = torch.as_tensor(np.asarray(st["radii"]) > 0)
    o = torch.tensor(np.asarray(sc["opacity"], np.float64).reshape(-1))
    dop = torch.tensor(np.asarray(grads["dL_dopacity"], np.float64).reshape(-1))
    S = torch.where(vis, (dop * o).detach() * r, torch.zeros_like(r)).sum()
    precomp = th["cov3D"] is not None
    leaves = [th["means3D"], c6] + ([] if precomp else [th["scales"], th["rots"]])
    gl = [t.numpy() for t in torch.autograd.grad(S, leaves)]
    npd = grads["dL_dopacity"].dtype
    rv = torch.where(vis, r, torch.zeros_like(r)).detach().numpy()
    grads["dL_dopacity"] = (np.asarray(grads["dL_dopacity"], np.float64).reshape(-1) * rv).astype(npd)
    grads["dL_dmeans3D"] = (grads["dL_dmeans3D"] + gl[0]).astype(npd)
    grads["dL_dcov3D"] = (grads["dL_dcov3D"] + gl[1]).astype(npd)       # dL/dSigma3D, written on both paths
    if not precomp:
        grads["dL_dscales"] = (grads["dL_dscales"] + gl[2]).astype(npd)
        grads["dL_drots"] = (grads["dL_drots"] + gl[3]).astype(npd)
    return grads


def render_autograd_aa(sc, st, denom_eps=0.0):
    """fp64 autograd image [3,H,W] of the anti-aliased forward and its leaves (dict of fp64 tensors with requires_grad):
    raster_torch64.render_autograd with opacities o * rho(theta)."""
    th = _theta(sc)
    th["colors"] = torch.tensor(np.asarray(sc["colors"], np.float64), requires_grad=True)
    th["opacity"] = torch.tensor(np.asarray(sc["opacity"], np.float64).reshape(-1), requires_grad=True)
    r = rho_torch(rt.camera(st), th["means3D"], _c6(sc, th))
    img = rt.render_autograd(st, th["means3D"], th["colors"], th["opacity"] * r, th["scales"], th["rots"],
                             float(sc.get("scale_modifier", 1.0)), cov3D=th["cov3D"], denom_eps=denom_eps)
    return img, th


def aa_forced_backward(sc, dtype, base, final_T, n_contrib, g):
    """`helpers.forced_backward` of the anti-aliased forward: the oracle backward on the o' state with the device's
    discrete decisions, plus the anti-aliasing chain.  Returns (oracle, state, grads)."""
    op, _ = aa_opacity(sc, dtype)
    o, st, grads = forced_backward(dict(sc, opacity=op.reshape(np.asarray(sc["opacity"]).shape)), dtype, base, final_T,
                                   n_contrib, g)
    return o, st, aa_backward(sc, st, grads)
