"""Seeded inputs for the unprojection tests and the per-element checks they are held to.

`SWEEP` is what tests/test_unproject_fp64_gpu.py runs on the device; tests/test_unproject_torch64_cpu.py shows on the
same cases that each mutant of oracle/unproject_torch64.py breaks a check, i.e. that these checks would reject a kernel
with that bug.  Every case has per-item ref_intr offsets, both signs of Tf_x across its items (or across the sweep for
B = 1), cx != cy, a mask whose channel 1 differs from channel 0, and a few pixels with flow == offset exactly."""
import itertools

import numpy as np
import torch

from oracle import unproject_torch64 as ut

BATCHES = (1, 2, 4)
SIZES = (1, 7, 24, 255, 256, 257, 1024)
MASKS = tuple(itertools.product((1, 3), ("binary", "soft", "zero"), (3, 4)))     # (C, kind, extr rows)
GRAD_MODES = ("xyz", "depth", "both")


def make_case(B, S, C, kind, rows, seed):
    """-> dict of fp32 CPU tensors: flow[B,1,S,S], mask[B,C,S,S], intr, extr[B,rows,4], ref_intr, tf_x[B], and the
    incoming gradients g_xyz[B,S*S,3], g_depth[B,1,S,S]."""
    rng = np.random.default_rng(seed)
    f32 = np.float32
    intr = np.zeros((B, 3, 3), f32)
    intr[:, 0, 0], intr[:, 1, 1] = S * rng.uniform(0.8, 1.6, B) + 1, S * rng.uniform(0.8, 1.6, B) + 1
    intr[:, 0, 2], intr[:, 1, 2] = S * rng.uniform(0.4, 0.6, B) + 0.25, S * rng.uniform(0.4, 0.6, B) + 0.35
    intr[:, 2, 2] = 1
    ref_intr = intr.copy()
    ref_intr[:, 0, 2] = intr[:, 0, 2] * rng.uniform(0.7, 1.3, B).astype(f32)        # within 2x: offset is exact
    offset = ref_intr[:, 0, 2] - intr[:, 0, 2]                                       # fp32, as the kernel forms it
    tf = (rng.uniform(300, 500, B) * np.where((np.arange(B) + seed) % 2 == 0, 1, -1)).astype(f32)
    extr = np.zeros((B, rows, 4), f32)
    for b in range(B):
        q, r = np.linalg.qr(rng.standard_normal((3, 3)))
        extr[b, :3, :3] = q * np.sign(np.diag(r))
        extr[b, :3, 3] = rng.uniform(-2, 2, 3)
    if rows == 4:
        extr[:, 3, 3] = 1
    inv_depth = rng.uniform(0.3, 2.0, (B, 1, S, S))
    flow = (offset[:, None, None, None] + tf[:, None, None, None] * inv_depth).astype(f32)
    n0 = max(1, S // 64)
    rows0, cols0 = rng.integers(0, max(1, S // 5), (B, n0)), rng.integers(0, S, (B, n0))
    for b in range(B):                                                               # depth exactly 0 at mask 1
        flow[b, 0, rows0[b], cols0[b]] = offset[b]
    if kind == "binary":
        mask = (rng.uniform(0, 1, (B, C, S, S)) < 0.7).astype(f32)
    elif kind == "soft":
        mask = rng.uniform(0.01, 0.99, (B, C, S, S)).astype(f32)
    else:
        mask = np.zeros((B, C, S, S), f32)
    if kind != "zero":
        mask[:, 0, :max(1, S // 5)] = 1                                                # where flow == offset
    g_xyz = rng.standard_normal((B, S * S, 3)).astype(f32)
    g_depth = rng.standard_normal((B, 1, S, S)).astype(f32)
    T = torch.from_numpy
    return {"flow": T(flow), "mask": T(mask), "intr": T(intr), "extr": T(extr), "ref_intr": T(ref_intr),
            "tf_x": T(tf), "g_xyz": T(g_xyz), "g_depth": T(g_depth)}


def _sweep():
    out = []
    for i, (S, B) in enumerate(itertools.product(SIZES, BATCHES)):
        C, kind, rows = MASKS[i % len(MASKS)]
        out.append((B, S, C, kind, rows, 500 + i))
    return out


SWEEP = _sweep()


def case_id(case):
    B, S, C, kind, rows, _ = case
    return f"B{B}-S{S}-C{C}-{kind}-E{rows}x4"


def _args(inp):
    return inp["flow"], inp["mask"], inp["intr"], inp["extr"], inp["ref_intr"], inp["tf_x"]


def _grads(mode, inp):
    return (inp["g_xyz"] if mode != "depth" else None), (inp["g_depth"] if mode != "xyz" else None)


def reference(inp):
    """fp32 depth / valid in the reference's op order, fp64 xyz and d/d flow per gradient mode, and the bounds."""
    d32, _, v32 = ut.unproject(*_args(inp), dtype=torch.float32)
    ref = {"depth": d32, "valid": v32}
    for mode in GRAD_MODES:
        depth, xyz, _, g = ut.forward_and_grad(*_args(inp), *_grads(mode, inp))
        b = ut.bounds(depth, inp["mask"], inp["intr"], inp["extr"], inp["tf_x"], *_grads(mode, inp))
        ref["xyz"], ref["grad_" + mode] = xyz, g
        ref["bound_xyz"], ref["bound_grad_" + mode] = b["xyz"], b["grad"]
    return ref


def stand_in(inp, mutant=None):
    """What an fp32 kernel with bug `mutant` would return: the fp32 restatement (mutated) and its autograd."""
    out = {}
    for mode in GRAD_MODES:
        out["depth"], out["xyz"], out["valid"], out["grad_" + mode] = ut.forward_and_grad(
            *_args(inp), *_grads(mode, inp), dtype=torch.float32, mutant=mutant)
    return out


def ratios(ref, got):
    """depth / valid: 0 when bit-identical to the fp32 restatement, else inf; xyz and d/d flow: worst err / bound
    (0 where equal, inf where the bound is 0, as for d/d flow at mask 0)."""
    out = {}
    for k, v in got.items():
        v = v.detach().cpu()
        if k in ("depth", "valid"):
            same = v.dtype == ref[k].dtype and v.shape == ref[k].shape and torch.equal(
                v.view(torch.int32) if k == "depth" else v, ref[k].view(torch.int32) if k == "depth" else ref[k])
            out[k] = 0.0 if same else float("inf")
            continue
        err = (v.to(torch.float64) - ref[k]).abs()
        r = torch.where(err == 0, torch.zeros_like(err), err / ref["bound_" + k])
        out[k] = float(r.max()) if r.numel() else 0.0
    return out
