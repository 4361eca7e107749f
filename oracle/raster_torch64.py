"""Independent fp64 *autograd* restatement of the rasterizer forward (TEST INFRASTRUCTURE ONLY).

Purpose: SURVEY.md Appendix A's backward formulas (A.6-A.8) are recalled, not verifiable against
the absent `diff-gaussian-rasterization` source.  This module restates only the FORWARD in its
maths form (Sigma3D = R S^2 R^T, Sigma2D = J W Sigma3D W^T J^T + 0.3 I, front-to-back compositing
with the 1/255, 0.99 and T<1e-4 rules) in differentiable fp64 torch and lets autograd derive
every gradient.  tests/test_oracle_backward.py checks gpsg_oracle.c's hand-written backward
against it -- that is what pins the backward formulas.

Two upstream conventions are reproduced on purpose (documented in Appendix A.6/A.7):
  * the min(0.99, o*G) clamp is ignored by the derivative (straight-through);
  * when t.x/t.z is clamped to +-1.3 tanfov, t.x is treated as independent of t.z and gets zero grad.
Discrete decisions (cull, radius, tile lists, sort order) are piecewise constant and taken from
the C oracle's state.  Usable only for small cases (python loop over tiles).
"""
import numpy as np
import torch


def _rotmat(q):
    r, x, y, z = q[:, 0], q[:, 1], q[:, 2], q[:, 3]
    R = torch.stack([
        1 - 2 * (y * y + z * z), 2 * (x * y - r * z), 2 * (x * z + r * y),
        2 * (x * y + r * z), 1 - 2 * (x * x + z * z), 2 * (y * z - r * x),
        2 * (x * z - r * y), 2 * (y * z + r * x), 1 - 2 * (x * x + y * y)], -1)
    return R.reshape(-1, 3, 3)


def cov3d(scales, rots, scale_mod=1.0):
    """Sigma3D = R diag(mod*s)^2 R^T as the 6 upper-triangle entries [P,6] (xx, xy, xz, yy, yz, zz)."""
    R = _rotmat(rots)
    N = R @ torch.diag_embed(scales * scale_mod)
    S = N @ N.transpose(1, 2)
    return torch.stack([S[:, 0, 0], S[:, 0, 1], S[:, 0, 2], S[:, 1, 1], S[:, 1, 2], S[:, 2, 2]], -1)


def camera(st):
    """The camera of a RasterOracle state as fp64 tensors: dict(view, proj, W, H, tanfovx, tanfovy)."""
    i = st["inputs"]
    dt = torch.float64
    return dict(view=torch.tensor(np.asarray(i["view"], np.float64).reshape(4, 4), dtype=dt),    # tensor as passed: W2V^T
                proj=torch.tensor(np.asarray(i["proj"], np.float64).reshape(4, 4), dtype=dt),
                W=st["W"], H=st["H"], tanfovx=float(i["tanfovx"]), tanfovy=float(i["tanfovy"]))


def project(cam, means3D, c6, denom_eps=0.0):
    """A.2 per Gaussian (every Gaussian independent of the others): world means [P,3] and covariances [P,6] ->
    (ndc [P,2], pixel means [P,2], conic (x, y, w) [P,3], cov2D + 0.3 as (a, b, c) [P,3]).  See render_autograd for the
    frustum clamp and `denom_eps`."""
    dt = torch.float64
    view, proj, W, H = cam["view"], cam["proj"], cam["W"], cam["H"]
    tanx, tany = cam["tanfovx"], cam["tanfovy"]
    fx, fy = W / (2.0 * tanx), H / (2.0 * tany)
    P = means3D.shape[0]
    hom = torch.cat([means3D, torch.ones(P, 1, dtype=dt)], 1)
    t = (hom @ view)[:, :3]                       # row-vector convention == M p
    ph = hom @ proj
    pw = 1.0 / (ph[:, 3] + float(np.float32(0.0000001)))
    ndc = ph[:, :2] * pw[:, None]
    pix = torch.stack([((ndc[:, 0] + 1.0) * W - 1.0) * 0.5, ((ndc[:, 1] + 1.0) * H - 1.0) * 0.5], 1)
    Sigma = torch.stack([c6[:, 0], c6[:, 1], c6[:, 2], c6[:, 1], c6[:, 3], c6[:, 4], c6[:, 2], c6[:, 4], c6[:, 5]], -1)
    Sigma = Sigma.reshape(-1, 3, 3)
    limx, limy = float(np.float32(1.3)) * tanx, float(np.float32(1.3)) * tany
    tz = t[:, 2]
    rx, ry = t[:, 0] / tz, t[:, 1] / tz
    cx = (rx < -limx) | (rx > limx)
    cy = (ry < -limy) | (ry > limy)
    tx = torch.where(cx, (rx.clamp(-limx, limx) * tz).detach(), t[:, 0])
    ty = torch.where(cy, (ry.clamp(-limy, limy) * tz).detach(), t[:, 1])
    zero = torch.zeros_like(tz)
    J = torch.stack([fx / tz, zero, -fx * tx / (tz * tz), zero, fy / tz, -fy * ty / (tz * tz)], -1).reshape(-1, 2, 3)
    Wrot = view[:3, :3].T                          # maths world->view rotation
    A = J @ Wrot
    cov = A @ Sigma @ A.transpose(1, 2)
    k03 = float(np.float32(0.3))
    a, b, c = cov[:, 0, 0] + k03, cov[:, 0, 1], cov[:, 1, 1] + k03
    abc = torch.stack([a, b, c], 1)
    det = a * c - b * b
    if denom_eps:
        k = (det * det / (det * det + denom_eps)).detach()
        a, b, c = ((k * v + ((1 - k) * v).detach()) for v in (a, b, c))
        det = a * c - b * b
    return ndc, pix, torch.stack([c / det, -b / det, a / det], 1), abc


def render_autograd(st, means3D, colors, opacity, scales, rots, scale_mod=1.0, cov3D=None, denom_eps=0.0):
    """st: state dict of RasterOracle('f64').forward (supplies view/proj/camera + the discrete binning).
    Tensor args: fp64 torch tensors (requires_grad as desired).  `cov3D` [P,6] (see `cov3d`), when given, replaces the
    scale/rotation covariance, as cov3D_precomp does; one symmetric off-diagonal entry stands for both Sigma_ab and Sigma_ba.
    `denom_eps` > 0 scales the gradient through the conic by det^2 / (det^2 + denom_eps) without changing the image: the
    regulariser of the hand-written backward's 1/(det^2 + 1e-7).  Returns image [3,H,W] fp64."""
    i = st["inputs"]
    W, H = st["W"], st["H"]
    dt = torch.float64
    bg = torch.tensor(np.asarray(i["bg"], np.float64), dtype=dt)
    c6 = cov3d(scales, rots, scale_mod) if cov3D is None else cov3D
    _, pix, con, _ = project(camera(st), means3D, c6, denom_eps)
    conx, cony, conz = con[:, 0], con[:, 1], con[:, 2]
    op = opacity.reshape(-1)

    ranges = st["ranges"]
    vals = torch.as_tensor(st["vals"].astype(np.int64))
    gx = (W + 15) // 16
    img = bg[:, None, None].expand(3, H, W).clone()
    thr_a = float(np.float32(1.0) / np.float32(255.0))
    for tile in range(ranges.shape[0]):
        s, e = int(ranges[tile, 0]), int(ranges[tile, 1])
        ty0, tx0 = (tile // gx) * 16, (tile % gx) * 16
        ys = torch.arange(ty0, min(ty0 + 16, H), dtype=dt)
        xs = torch.arange(tx0, min(tx0 + 16, W), dtype=dt)
        if e <= s or len(ys) == 0 or len(xs) == 0:
            continue
        ids = vals[s:e]
        py, px = torch.meshgrid(ys, xs, indexing="ij")
        px, py = px.reshape(-1, 1), py.reshape(-1, 1)
        dx = pix[ids, 0][None] - px
        dy = pix[ids, 1][None] - py
        power = -0.5 * (conx[ids][None] * dx * dx + conz[ids][None] * dy * dy) - cony[ids][None] * dx * dy
        G = torch.exp(power)
        raw = op[ids][None] * G
        alpha = raw + (raw.clamp(max=float(np.float32(0.99))) - raw).detach()      # straight-through clamp
        keep = (power <= 0) & (alpha.detach() >= thr_a)
        alpha = torch.where(keep, alpha, torch.zeros_like(alpha))
        # transmittance with the T<1e-4 stop rule (decision is piecewise constant)
        with torch.no_grad():
            Tn = torch.cumprod(1 - alpha, 1)
            stop = (Tn < float(np.float32(0.0001))) & keep
            dead = torch.cumsum(stop.to(torch.int64), 1) > 0
        alpha = torch.where(dead, torch.zeros_like(alpha), alpha)
        T_excl = torch.cumprod(torch.cat([torch.ones(alpha.shape[0], 1, dtype=dt), 1 - alpha[:, :-1]], 1), 1)
        w = alpha * T_excl
        C = w @ colors[ids]
        T_fin = T_excl[:, -1] * (1 - alpha[:, -1])
        out = C + T_fin[:, None] * bg[None]
        img[:, ty0:ty0 + len(ys), tx0:tx0 + len(xs)] = out.T.reshape(3, len(ys), len(xs))
    return img
