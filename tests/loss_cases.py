"""Seeded image pairs for the photometric-loss tests and the per-element checks they are held to.

`SWEEP` is what tests/test_loss_fp64_gpu.py runs on the device; tests/test_loss_torch64_cpu.py shows on the same cases
that each mutant of oracle/loss_torch64.py breaks a bound, i.e. that these checks would reject a kernel with that bug.
Sizes cross the 32-px tile and the 5-px halo in every combination (1 .. 69 on each axis); planes go past 6."""
import itertools

import numpy as np
import torch

from oracle import loss_torch64 as lt

KINDS = ("flat", "flat_bright", "zero_var", "ties", "noise", "smooth")
SIZES = (1, 5, 6, 11, 31, 32, 33, 37, 69)
SHAPE_OF_PLANES = {1: (1, 1), 3: (1, 3), 6: (2, 3), 96: (32, 3)}


def image_pair(kind, shape, seed):
    """(img, gt) float32 [B,C,H,W] in [0,1] ([-1,1] for kind 'signed')."""
    rng = np.random.default_rng(seed)
    B, C, H, W = shape
    if kind == "flat":                                   # two constant images: zero variance everywhere
        gt, img = np.full(shape, 0.6), np.full(shape, 0.4)
    elif kind == "flat_bright":                          # bright flat gt, the render a little off it
        gt = np.full(shape, 0.95)
        img = np.clip(gt + rng.normal(0, 0.01, shape), 0, 1)
    elif kind == "zero_var":                             # 8x8 constant blocks, equal in half of them, and a black corner
        blk = lambda: np.kron(rng.uniform(0, 1, (B, C, H // 8 + 1, W // 8 + 1)), np.ones((8, 8)))[..., :H, :W]
        gt = blk()
        img = np.where(blk() > 0.5, gt, blk())
        gt[..., : H // 3, : W // 3] = 0.0
        img[..., : H // 3, : W // 3] = 0.0
    elif kind == "ties":                                 # x == y exactly on about half of the pixels
        gt = rng.uniform(0, 1, shape)
        img = np.where(rng.uniform(0, 1, shape) < 0.5, gt, np.clip(gt + rng.normal(0, 0.1, shape), 0, 1))
    elif kind == "noise":
        gt, img = rng.uniform(0, 1, shape), rng.uniform(0, 1, shape)
    elif kind == "smooth":                               # low-frequency content, noisy render, a black region
        yy, xx = np.meshgrid(np.linspace(0, 4, H), np.linspace(0, 4, W), indexing="ij")
        gt = 0.5 + 0.4 * np.sin(yy * 1.7 + np.arange(C)[:, None, None]) * np.cos(xx * 2.3)
        gt = np.broadcast_to(gt, shape).copy()
        gt[..., : H // 4, W // 2:] = 0.0
        img = np.clip(gt + rng.normal(0, 0.05, shape), 0, 1)
    elif kind == "signed":
        gt = rng.uniform(-1, 1, shape)
        img = np.clip(gt + rng.normal(0, 0.3, shape), -1, 1)
    else:
        raise ValueError(kind)
    return img.astype(np.float32), gt.astype(np.float32)


def _sweep():
    cases = []
    for i, (H, W) in enumerate(itertools.product(SIZES, SIZES)):
        planes = (1, 3, 6)[i % 3]
        cases.append((KINDS[(i // 3) % 6], SHAPE_OF_PLANES[planes] + (H, W), 100 + i))
    for i, (H, W) in enumerate(((32, 32), (33, 37), (69, 69), (5, 6))):
        cases.append((KINDS[(2 * i + 1) % 6], SHAPE_OF_PLANES[96] + (H, W), 200 + i))
    cases.append(("signed", (1, 3, 37, 69), 300))
    cases.append(("signed", (2, 3, 33, 6), 301))
    return cases


SWEEP = _sweep()
LARGE = [("smooth", (1, 3, 1024, 1024), 400), ("flat_bright", (1, 3, 1024, 512), 401), ("noise", (1, 1, 512, 1024), 402)]


def case_id(case):
    kind, shape, _ = case
    return f"{kind}-{'x'.join(map(str, shape))}"


KEYS = ("loss", "l1", "ssim", "ssim_per_image", "dmaps_img", "dmaps_gt", "grad_img", "grad_gt")


def reference(img, gt, w_l1=0.8, w_ssim=0.2, g=1.0):
    """Everything the device returns, in fp64, and the bound each is held to (under "bound")."""
    img, gt = torch.as_tensor(img), torch.as_tensor(gt)
    ref, ref["grad_img"], ref["grad_gt"] = lt.forward_and_grads(img, gt, w_l1, w_ssim)
    ref["grad_img"], ref["grad_gt"] = g * ref["grad_img"], g * ref["grad_gt"]
    ref["dmaps_img"], ref["dmaps_gt"] = lt.dmaps(ref["moments"])
    ref["bound"] = lt.bounds(img, gt, ref["moments"], w_l1, w_ssim, g)
    return ref


def outputs_of(d):
    return {k: v for k, v in d.items() if k in KEYS}


def ratios(ref, got):
    """Worst |got - ref| / bound of every quantity in `got` (0 where they agree exactly, inf where the bound is 0)."""
    out = {}
    for k, v in got.items():
        err = (torch.as_tensor(v).detach().cpu().to(torch.float64).reshape(ref[k].shape) - ref[k]).abs()
        bnd = torch.as_tensor(ref["bound"][k], dtype=torch.float64)
        r = torch.where(err == 0, torch.zeros_like(err), err / bnd)
        out[k] = float(r.max()) if r.numel() else 0.0
    return out
