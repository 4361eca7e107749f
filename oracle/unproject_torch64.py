"""Independent fp64 torch restatement of the fused unprojection (TEST INFRASTRUCTURE ONLY).

Restates flow2depth + depth2pc (reference lib/utils.py:87-119, as lib/network.py:64-69 calls them) from their maths, in
differentiable CPU torch, so that d/d flow comes from autograd rather than from a hand-written backward:

  * depth = -(offset - flow) / Tf_x * mask[:, 0],  offset = ref_intr cx - intr cx;   pts_valid = depth != 0;
  * z = 1 / (depth + 1e-8), pixel centres u, v = 0.5 .. S - 0.5 (linspace), p = ((u - cx) z / fx, (v - cy) z / fy, z);
  * xyz = R^T p - R^T t with R, t the first three rows of extr.

dtype=float64 is the maths.  dtype=float32 is the reference's own fp32 chain in its op order (`offset - flow`, negate,
`/ Tf_x`, `* mask`; `(u - cx) * z / fx`): depth and pts_valid of a correct fp32 kernel are bit-identical to it, since
only a subtraction, a negation, an IEEE division and a multiplication are involved.

`mutant=` perturbs the restatement the way a wrong kernel would (MUTANTS), so the tests can show that the bounds of
`bounds` reject each such kernel."""
import torch

F64 = torch.float64
EPS = 2.0 ** -24
K_XYZ = 32                     # xyz: |got - fp64| <= K_XYZ 2^-24 (|R^T| |p| + |R^T| |t|) per component
K_GRAD = 64                    # d/d flow: K_GRAD 2^-24 times the sum of the magnitudes of its terms
MUTANTS = ("pixel_corner", "cx_cy_swapped", "R_not_Rt", "mask_channel_1", "z_not_z2_backward", "tf_sign_dropped")


class _RecipZBackward(torch.autograd.Function):
    """z = 1 / a whose backward returns -g z instead of -g z^2 (the "z instead of z^2" mutant)."""

    @staticmethod
    def forward(ctx, a):
        z = 1.0 / a
        ctx.save_for_backward(z)
        return z

    @staticmethod
    def backward(ctx, g):
        z, = ctx.saved_tensors
        return -g * z


def pixel_centres(S, dtype):
    return torch.linspace(0.5, S - 0.5, S, dtype=dtype)


def unproject(flow, mask, intr, extr, ref_intr, tf_x, dtype=F64, mutant=None):
    """flow[B,1,S,S], mask[B,C,S,S], intr[B,3,3], extr[B,3|4,4], ref_intr[B,3,3], tf_x[B] (torch, any float dtype)
    -> depth[B,1,S,S], xyz[B,S*S,3], valid[B,S*S] in `dtype`; differentiable w.r.t. flow."""
    f, m, K, E, Kr = (t.to(dtype) for t in (flow, mask, intr, extr, ref_intr))
    tf = tf_x.to(dtype).reshape(-1)
    B, _, S, _ = f.shape
    if mutant == "tf_sign_dropped":
        tf = tf.abs()
    offset = (Kr[:, 0, 2] - K[:, 0, 2])[:, None, None, None]
    depth = -(offset - f) / tf[:, None, None, None]
    ch = 1 if mutant == "mask_channel_1" and m.shape[1] > 1 else 0
    depth = depth * m[:, ch:ch + 1]
    c = pixel_centres(S, dtype)
    if mutant == "pixel_corner":
        c = c - 0.5
    v, u = torch.meshgrid(c, c, indexing="ij")
    a = depth[:, 0] + 1e-8
    z = _RecipZBackward.apply(a) if mutant == "z_not_z2_backward" else 1.0 / a
    cx, cy = K[:, 0, 2, None, None], K[:, 1, 2, None, None]
    if mutant == "cx_cy_swapped":
        cx, cy = cy, cx
    px = (u - cx) * z / K[:, 0, 0, None, None]
    py = (v - cy) * z / K[:, 1, 1, None, None]
    p = torch.stack([px, py, z], -1).reshape(B, S * S, 3)
    R, t = E[:, :3, :3], E[:, :3, 3]
    Rt = R if mutant == "R_not_Rt" else R.transpose(1, 2)
    xyz = p @ Rt.transpose(1, 2) - (Rt @ t[..., None]).transpose(1, 2)
    return depth, xyz, (depth != 0).reshape(B, -1)


def forward_and_grad(flow, mask, intr, extr, ref_intr, tf_x, g_xyz=None, g_depth=None, dtype=F64, mutant=None):
    """`unproject` and d <(xyz, depth), (g_xyz, g_depth)> / d flow by autograd (None = that output gets no gradient)."""
    fl = flow.detach().to(dtype).requires_grad_(True)
    depth, xyz, valid = unproject(fl, mask, intr, extr, ref_intr, tf_x, dtype, mutant)
    loss = 0.0
    if g_xyz is not None:
        loss = loss + (xyz * g_xyz.to(dtype)).sum()
    if g_depth is not None:
        loss = loss + (depth * g_depth.to(dtype)).sum()
    grad = torch.autograd.grad(loss, fl)[0] if torch.is_tensor(loss) else None
    return depth.detach(), xyz.detach(), valid, grad


def bounds(depth, mask, intr, extr, tf_x, g_xyz=None, g_depth=None):
    """Per-element bounds, from the fp64 depth: xyz [B,S*S,3] and d/d flow [B,1,S,S].

    xyz_k: K_XYZ 2^-24 (sum_j |R_jk| |p_j| + sum_j |R_jk| |t_j|) -- p carries a few roundings of its own (sub, add, two
    divisions, a product), the dot products three more.  d/d flow = (z^2 (u'/fx (R g)_0 + v'/fy (R g)_1 + (R g)_2) +
    g_depth) * mask / Tf_x up to sign, u' = u - cx: K_GRAD 2^-24 |mask / Tf_x| times the same sum of absolute values."""
    d = depth.to(F64)[:, 0]
    K, E = intr.to(F64), extr.to(F64)
    B, S, _ = d.shape
    c = pixel_centres(S, F64)
    v, u = torch.meshgrid(c, c, indexing="ij")
    z = 1.0 / (d + 1e-8)
    ax = (u - K[:, 0, 2, None, None]).abs() / K[:, 0, 0, None, None].abs()
    ay = (v - K[:, 1, 2, None, None]).abs() / K[:, 1, 1, None, None].abs()
    p = torch.stack([ax * z.abs(), ay * z.abs(), z.abs()], -1).reshape(B, S * S, 3)
    Ra, ta = E[:, :3, :3].abs(), E[:, :3, 3].abs()
    out = {"xyz": K_XYZ * EPS * (p @ Ra + (ta[:, None, :] @ Ra))}
    scale = (mask.to(F64)[:, 0] / tf_x.to(F64).reshape(-1)[:, None, None]).abs()
    mag = torch.zeros_like(d)
    if g_xyz is not None:
        gp = (g_xyz.to(F64).abs() @ Ra.transpose(1, 2)).reshape(B, S, S, 3)       # |R| |g|
        mag = z * z * (ax * gp[..., 0] + ay * gp[..., 1] + gp[..., 2])
    if g_depth is not None:
        mag = mag + g_depth.to(F64)[:, 0].abs()
    out["grad"] = (K_GRAD * EPS * scale * mag)[:, None]
    return out
