"""Per-Gaussian rounding bounds of the rasterizer backward (TEST INFRASTRUCTURE ONLY).

Truth: the fp64 backward of gpsg_oracle.c run on the fp32 forward state (means2D, conic_opacity, tile lists, final_T,
n_contrib) that the device itself used -- `fp64_state`.  Its continuous inputs are then exactly the device's, so a correct
fp32 backward differs from it only by its own rounding (and by ex2.approx / rcp.approx), and every gradient element gets
its own bound

    |fp32 - fp64| <= 2^-24 * Mag

Compositing (A.6): oracle_render_backward_mag accumulates every (pixel, Gaussian) term of the gradient with all factors
in absolute value, weighted by its rounding count: the MAG_* operation counts in gpsg_oracle.c, plus one step per
transmittance recovery T /= (1 - alpha) the pixel made before reaching the term, each carrying the error of that alpha
amplified by 1 / (1 - alpha).  A summation tree of depth d adds at most d * u * sum|terms| (`absum`): the device's tree is
16 fma per lane + one shuffle + one atomic per warp and tile (8 warps per tile), so d <= 17 + 8 * tiles_touched; a
serial sum over a Gaussian's pixels has d = nterm.  Mag_2D = mag + d * absum.

Projection chain (A.7 + A.8): per Gaussian, the exact fp64 Jacobian J of u = (ndc_x, ndc_y, conic_x, 2 conic_y, conic_w)
with respect to its inputs (means3D, scales, rots or cov3D), by torch.func.jacrev + vmap over raster_torch64.project.
Then Mag_3D = |J|^T Mag_2D + C_CHAIN * kappa * |J|^T |g_2D|: the propagated compositing error plus the chain's own
roundings, kappa = (ac + b^2) / |ac - b^2| the conditioning of the conic inversion (a, b, c = cov2D + 0.3), which amplifies
the rounding of `denom` and of everything computed from it; C_CHAIN counts the fp32 operations on the longest path of the
chain (view transform 3, J 3, A 2, Sigma 3 (scale / rotation: + R 3), A Sigma 3, A Sigma A^T 3, denom 2, denom2inv 3,
dL_da / db / dc 6, dL_dcov3D 4, dL_dA 3, dL_dJ 3, dL_dt 4, dL_dmean 3, dL_dN 4, dL_dR 1, dL_dq 9) -> 64.
The absolute Jacobian is taken stage by stage wherever the fp32 chain forms a difference whose exact value is small:
conic -> (a, b, c) with the term magnitudes of A.7 ((denom - ac) rounds like ac, not like b^2), (a, b, c) -> cov3D with
|J| |W| for A = J W, and cov3D -> (scales, rots) by the A.8 formulas in absolute value (the rotation gradient of a nearly
isotropic Gaussian is ~0, its fp32 value is not).  Without these three the fp32 oracle exceeds the bound by up to 5x on
nearly isotropic splats.
"""
import numpy as np
import torch

from oracle import raster_torch64 as rt
from oracle.raster_oracle import RasterOracle

U = 2.0 ** -24
C_CHAIN = 64.0
DEVICE_LEAVES = 17          # 16 fma per lane + 1 shuffle before the first atomic
DEVICE_PER_TILE = 8         # one partial sum per warp (4 per CTA, two CTAs per tile)

COLS = dict(dL_dmean2D=slice(0, 2), dL_dconic=slice(2, 5), dL_dopacity=slice(5, 6), dL_dcolors=slice(6, 9))


def fp64_state(base, final_T, n_contrib, colors=None):
    """The fp64 oracle's state on the fp32 forward state `base` (RasterOracle('f32').forward, bit-identical to the
    device's for the visible Gaussians): means2D, conic_opacity and the inputs upcast exactly, the tile lists of `base`,
    the device's final_T / n_contrib.  `colors` replaces the colours (SH: the fp64 colours; the device's own fp32 colours
    are then bounded through oracle_render_backward_mag's col_err)."""
    st = dict(base)
    for k in ("means2D", "conic_opacity", "depth", "cov3D"):
        st[k] = np.ascontiguousarray(base[k], np.float64)
    st["inputs"] = {k: (np.ascontiguousarray(v, np.float64) if isinstance(v, np.ndarray) else v)
                    for k, v in base["inputs"].items()}
    if colors is not None:                  # colours the device computes itself (SH): the fp64 ones
        st["inputs"]["colors"] = np.ascontiguousarray(colors, np.float64)
    st["final_T"] = np.ascontiguousarray(np.asarray(final_T, np.float64).reshape(base["H"], base["W"]))
    st["n_contrib"] = np.ascontiguousarray(np.asarray(n_contrib).reshape(base["H"], base["W"]), np.uint32)
    return st


def projection_jacobian(st, vis):
    """J [n, 5, 9] of u = (ndc_x, ndc_y, conic_x, 2 conic_y, conic_w) with respect to (means3D, cov3D) of the visible
    Gaussians `vis`, their covariances c6 [n, 6] (fp64, from scales / rots when there is no cov3D_precomp), and kappa [n]."""
    i = st["inputs"]
    cam = rt.camera(st)
    T = lambda a: torch.from_numpy(np.ascontiguousarray(np.asarray(a, np.float64)[vis]))
    m3 = T(i["means3D"])
    if i["cov3D_precomp"] is not None:
        c6 = T(i["cov3D_precomp"])
    else:
        c6 = rt.cov3d(T(i["scales"]), T(i["rots"]), float(i["scale_mod"]))

    def v_of(m, c):                     # (ndc, cov2D + 0.3): the intermediates the fp32 chain goes through
        ndc, _, _, abc = rt.project(cam, m[None], c[None])
        return torch.cat([ndc[0], abc[0]])

    def con_of(abc):                    # conic inversion, with the backward's 1 / (det^2 + 1e-7) regulariser
        a, b, c = abc[0], abc[1], abc[2]
        det = a * c - b * b
        k = (det * det / (det * det + float(np.float32(0.0000001)))).detach()
        a, b, c = ((k * v + ((1 - k) * v).detach()) for v in (a, b, c))
        det = a * c - b * b
        return torch.stack([c / det, -2.0 * b / det, a / det])

    jm, jc = torch.func.vmap(torch.func.jacrev(v_of, argnums=(0, 1)))(m3, c6)
    with torch.no_grad():
        abc = torch.func.vmap(v_of)(m3, c6)[:, 2:]
    jabc = torch.func.vmap(torch.func.jacrev(con_of))(abc)
    a, b, c = abc[:, 0].numpy(), abc[:, 1].numpy(), abc[:, 2].numpy()
    kappa = (a * c + b * b) / np.abs(a * c - b * b)
    # d(a, b, c)/d(cov3D) is A (x) A with A = J W; the fp32 A rounds relative to |J| |W|, not to |A| (W J can cancel), so
    # the stage is bounded with A_abs = |J| |W| in place of A
    V = cam["view"].numpy()
    t = np.asarray(i["means3D"], np.float64)[vis] @ V[:3, :3] + V[3, :3]
    fx, fy = cam["W"] / (2.0 * cam["tanfovx"]), cam["H"] / (2.0 * cam["tanfovy"])
    limx, limy = float(np.float32(1.3)) * cam["tanfovx"], float(np.float32(1.3)) * cam["tanfovy"]
    tz = t[:, 2]
    tx, ty = np.clip(t[:, 0] / tz, -limx, limx) * tz, np.clip(t[:, 1] / tz, -limy, limy) * tz
    Wr = np.abs(V[:3, :3].T)                                    # |W(r, k)|
    A0 = np.abs(fx / tz)[:, None] * Wr[0] + np.abs(fx * tx / tz ** 2)[:, None] * Wr[2]
    A1 = np.abs(fy / tz)[:, None] * Wr[1] + np.abs(fy * ty / tz ** 2)[:, None] * Wr[2]
    pairs = ((0, 0), (0, 1), (0, 2), (1, 1), (1, 2), (2, 2))        # cov3D entry (p, q); off-diagonals stand for both
    row_a = np.stack([(1 if p == q else 2) * A0[:, p] * A0[:, q] for p, q in pairs], 1)
    row_b = np.stack([A0[:, p] * A1[:, q] + (A0[:, q] * A1[:, p] if p != q else 0) for p, q in pairs], 1)
    row_c = np.stack([(1 if p == q else 2) * A1[:, p] * A1[:, q] for p, q in pairs], 1)
    jc_abs = np.stack([row_a, row_b, row_c], 1)                    # [n, (a, b, c), 6]
    J = torch.cat([jm, jc], 2).numpy()
    J[:, 2:, 3:] = np.maximum(np.abs(J[:, 2:, 3:]), jc_abs)
    # A.7 computes dL/d(a, b, c) term by term, with (denom - a c) for -b^2 and (denom + 2 b^2) for a c + b^2: their
    # rounding is relative to the terms, so the stage is bounded with the terms' magnitudes ([n, conic k, abc j])
    den = np.abs(a * c - b * b)
    d2i = 1.0 / (den * den + float(np.float32(0.0000001)))
    ab, ac_ = np.abs(b), np.abs(a * c)
    terms = np.stack([np.stack([c * c, 2 * ab * c, den + ac_], 1),
                      np.stack([2 * ab * c, 2 * (den + 2 * b * b), 2 * np.abs(a) * ab], 1),
                      np.stack([den + ac_, 2 * np.abs(a) * ab, a * a], 1)], 2) * d2i[:, None, None]
    return J, np.maximum(np.abs(jabc.numpy()), terms), kappa


# fp32 operations on the longest path from dL_dcov3D to dL_dscales / dL_drots: dL_dN 4, dL_dR 1, dL_dq 9 (dL_ds: 4 + 3 + 1)
C_ROT = 16.0


def _abs_cov_to_scale_rot(dcov, scales, rots, mod):
    """The A.8 step dL_dcov3D -> (dL_dscales, dL_drots) of gpsg_oracle.c with every factor in absolute value and every
    difference a - b as |a| + |b|: it bounds |J|^T dcov for dcov >= 0 and the rounding of that step, term by term."""
    q = np.abs(rots)
    r, x, y, z = q[:, 0], q[:, 1], q[:, 2], q[:, 3]
    R = np.stack([1 + 2 * (y * y + z * z), 2 * (x * y + r * z), 2 * (x * z + r * y),
                  2 * (x * y + r * z), 1 + 2 * (x * x + z * z), 2 * (y * z + r * x),
                  2 * (x * z + r * y), 2 * (y * z + r * x), 1 + 2 * (x * x + y * y)], 1).reshape(-1, 3, 3)
    sv = np.abs(mod * scales)
    d = dcov
    dS = np.stack([d[:, 0], 0.5 * d[:, 1], 0.5 * d[:, 2], 0.5 * d[:, 1], d[:, 3], 0.5 * d[:, 4],
                   0.5 * d[:, 2], 0.5 * d[:, 4], d[:, 5]], 1).reshape(-1, 3, 3)
    dN = 2 * np.einsum("nab,nbi->nai", dS, R * sv[:, None, :])
    dsc = abs(mod) * np.einsum("nai,nai->ni", dN, R)
    dR = dN * sv[:, None, :]
    e = lambda a_, i_: dR[:, a_, i_]
    dq = np.stack([
        2 * (z * e(0, 1) + y * e(0, 2) + z * e(1, 0) + x * e(1, 2) + y * e(2, 0) + x * e(2, 1)),
        2 * (y * e(0, 1) + z * e(0, 2) + y * e(1, 0) + 2 * x * e(1, 1) + r * e(1, 2) + z * e(2, 0) + r * e(2, 1) + 2 * x * e(2, 2)),
        2 * (2 * y * e(0, 0) + x * e(0, 1) + r * e(0, 2) + x * e(1, 0) + z * e(1, 2) + r * e(2, 0) + z * e(2, 1) + 2 * y * e(2, 2)),
        2 * (2 * z * e(0, 0) + r * e(0, 1) + x * e(0, 2) + r * e(1, 0) + 2 * z * e(1, 1) + y * e(1, 2) + x * e(2, 0) + y * e(2, 1))], 1)
    return dsc, dq


def grad_bounds(st, out, depth):
    """Per-element bounds (already multiplied by 2^-24) of every gradient of `out` = RasterOracle('f64').backward_mag(st)
    for an fp32 backward whose per-Gaussian summation depth is `depth` [P].  Returns dict name -> bound array.
    dL_dcov3D is bounded on both paths (the device returns it on request)."""
    P = st["P"]
    i = st["inputs"]
    M2 = out["mag"] + np.asarray(depth, np.float64)[:, None] * out["absum"]
    B = {k: M2[:, s].reshape(out[k].shape) for k, s in COLS.items()}
    vis = st["radii"] > 0
    B["dL_dmeans3D"], B["dL_dcov3D"] = np.zeros((P, 3)), np.zeros((P, 6))
    B["dL_dscales"], B["dL_drots"] = np.zeros((P, 3)), np.zeros((P, 4))
    if vis.any():
        Jv, Jc, kappa = projection_jacobian(st, vis)
        g2 = np.abs(np.concatenate([out["dL_dmean2D"], out["dL_dconic"]], 1)[vis])
        m2 = np.concatenate([B["dL_dmean2D"], B["dL_dconic"]], 1)[vis]
        # the fp32 chain goes through dL/d(ndc) and dL/d(a, b, c): the bound is taken stage by stage, |J2|^T |J1|^T,
        # which keeps what cancels between the a, b and c paths of the composite Jacobian
        aJc = np.abs(Jc)
        mv = np.concatenate([m2[:, :2], np.einsum("nkj,nk->nj", aJc, m2[:, 2:])], 1)
        gv = np.concatenate([g2[:, :2], np.einsum("nkj,nk->nj", aJc, g2[:, 2:])], 1)
        aJ = np.abs(Jv)
        M3 = np.einsum("nkm,nk->nm", aJ, mv) + C_CHAIN * kappa[:, None] * np.einsum("nkm,nk->nm", aJ, gv)
        B["dL_dmeans3D"][vis], B["dL_dcov3D"][vis] = M3[:, :3], M3[:, 3:]
        if i["cov3D_precomp"] is None:
            dcov = np.abs(out["dL_dcov3D"][vis])
            s, q = np.asarray(i["scales"], np.float64)[vis], np.asarray(i["rots"], np.float64)[vis]
            ms, mq = _abs_cov_to_scale_rot(M3[:, 3:] + C_ROT * dcov, s, q, float(i["scale_mod"]))
            B["dL_dscales"][vis], B["dL_drots"][vis] = ms, mq
    return {k: U * v for k, v in B.items()}


def ratios(got, want, bound):
    """Per-Gaussian worst |got - want| / bound over the tensor's columns (0 where both sides are 0, inf where the bound
    is 0 but the error is not)."""
    want = np.asarray(want, np.float64).reshape(want.shape[0], -1)
    got = np.asarray(got, np.float64).reshape(want.shape[0], -1)
    bound = np.asarray(bound, np.float64).reshape(want.shape[0], -1)
    err = np.abs(got - want)
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.where(err == 0, 0.0, err / bound)
    return np.where(np.isnan(r), np.inf, r).max(1) if r.size else np.zeros(want.shape[0])


def device_depth(base, nterm):
    """Summation depth of the device's accumulation of each Gaussian's terms (see the module docstring)."""
    return np.minimum(nterm.astype(np.float64), DEVICE_LEAVES + DEVICE_PER_TILE * base["tiles_touched"].astype(np.float64))


def exempt_sets(st, nthreads):
    """Gaussians whose gradient may legitimately differ by more than rounding: evaluated by a pixel where an
    `alpha < 1/255` / `power > 0` decision lies within fp32 rounding of its threshold (RasterOracle.margins with the fp32
    eps; the backward takes no transmittance decision).  Returns (shared, own, margins)."""
    m = RasterOracle("f64").margins(st, eps=dict(T=0.0), nthreads=nthreads)
    return m["taint"] & ~m["taint_own"], m["taint_own"], m
