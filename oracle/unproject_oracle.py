"""CPU oracle (numpy) of the fused unprojection.  TEST INFRASTRUCTURE ONLY.

Restates reference lib/utils.py:112-119 (flow2depth) and :87-109 (depth2pc) as used by lib/network.py:64-69.
PINNED by tests/golden/unproject_golden.npz, which tests/golden/make_unproject_golden.py produced by calling the
reference's own functions (imported from a checkout of the original project), incl. autograd gradients."""
import numpy as np


def unproject(flow, mask, intr, extr, ref_intr, tf_x, dtype=np.float64):
    """flow[B,1,S,S], mask[B,C,S,S], intr[B,3,3], extr[B,>=3,4], ref_intr[B,3,3], tf_x[B] -> depth, xyz[B,S*S,3], valid"""
    f = np.asarray(flow, dtype); m = np.asarray(mask, dtype)[:, :1]
    K = np.asarray(intr, dtype); E = np.asarray(extr, dtype); Kr = np.asarray(ref_intr, dtype); tf = np.asarray(tf_x, dtype)
    B, _, S, _ = f.shape
    offset = (Kr[:, 0, 2] - K[:, 0, 2])[:, None, None, None]
    depth = -(offset - f) / tf[:, None, None, None]
    depth = depth * m
    d = depth[:, 0]
    v, u = np.meshgrid(np.linspace(0.5, S - 0.5, S, dtype=dtype), np.linspace(0.5, S - 0.5, S, dtype=dtype), indexing="ij")
    z = 1.0 / (d + dtype(1e-8))
    px = (u[None] - K[:, 0, 2][:, None, None]) * z / K[:, 0, 0][:, None, None]
    py = (v[None] - K[:, 1, 2][:, None, None]) * z / K[:, 1, 1][:, None, None]
    p = np.stack([px, py, z], 1).reshape(B, 3, S * S)
    R, t = E[:, :3, :3], E[:, :3, 3:]
    Rt = np.transpose(R, (0, 2, 1))
    xyz = Rt @ p - Rt @ t
    return depth, np.transpose(xyz, (0, 2, 1)), (depth != 0).reshape(B, -1)


def unproject_backward(depth, mask, intr, extr, tf_x, dL_dxyz, dL_ddepth=None, dtype=np.float64):
    d = np.asarray(depth, dtype)[:, 0]; m = np.asarray(mask, dtype)[:, 0]
    K = np.asarray(intr, dtype); E = np.asarray(extr, dtype); tf = np.asarray(tf_x, dtype)
    B, S, _ = d.shape
    v, u = np.meshgrid(np.linspace(0.5, S - 0.5, S, dtype=dtype), np.linspace(0.5, S - 0.5, S, dtype=dtype), indexing="ij")
    z = 1.0 / (d + dtype(1e-8))
    g = np.asarray(dL_dxyz, dtype).reshape(B, S, S, 3)
    gp = np.einsum('brk,bsvk->bsvr', E[:, :3, :3], g)              # R g
    dz = gp[..., 0] * (u[None] - K[:, 0, 2][:, None, None]) / K[:, 0, 0][:, None, None] \
        + gp[..., 1] * (v[None] - K[:, 1, 2][:, None, None]) / K[:, 1, 1][:, None, None] + gp[..., 2]
    dd = -dz * z * z
    if dL_ddepth is not None:
        dd = dd + np.asarray(dL_ddepth, dtype)[:, 0]
    return (dd * m / tf[:, None, None])[:, None]
