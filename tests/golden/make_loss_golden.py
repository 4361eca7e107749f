"""Generate tests/golden/loss_golden.npz from the REFERENCE's own lib/loss.py (l1_loss, ssim) and the combination of
train_stage2.py:70-72, on the CPU in float64 and float32, with autograd gradients w.r.t. the rendered image.

Run with GPSG_REFERENCE naming a checkout of the original project:  python tests/golden/make_loss_golden.py"""
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.environ["GPSG_REFERENCE"])
from lib.loss import gaussian, l1_loss, ssim  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))


def case(rng, shape, smooth):
    gt = rng.uniform(0, 1, shape)
    if smooth:                                   # image-like: low-frequency content + a flat (zero-variance) region
        yy, xx = np.meshgrid(np.linspace(0, 3, shape[-2]), np.linspace(0, 3, shape[-1]), indexing="ij")
        gt = 0.5 + 0.4 * np.sin(yy * 2.1 + np.arange(shape[1])[:, None, None]) * np.cos(xx * 1.7)
        gt = np.broadcast_to(gt, shape).copy()
        gt[..., : shape[-2] // 3, : shape[-1] // 3] = 0.0
    img = np.clip(gt + rng.normal(0, 0.08, shape), 0, 1)
    img[..., -3:, -3:] = gt[..., -3:, -3:]       # exact ties: |x - y| = 0 -> subgradient 0
    return img, gt


def main():
    rng = np.random.default_rng(1314)
    out = {"window": gaussian(11, 1.5).numpy()}
    for name, shape, smooth in (("noise", (2, 3, 40, 52), False), ("smooth", (1, 3, 70, 33), True), ("tiny", (1, 3, 7, 5), False)):
        img, gt = case(rng, shape, smooth)
        out[f"{name}_img"], out[f"{name}_gt"] = img.astype(np.float32), gt.astype(np.float32)
        for dt, tag in ((torch.float64, "f64"), (torch.float32, "f32")):
            x = torch.tensor(out[f"{name}_img"]).to(dt).requires_grad_(True)
            y = torch.tensor(out[f"{name}_gt"]).to(dt)
            Ll1 = l1_loss(x, y)
            s = ssim(x, y)
            loss = 0.8 * Ll1 + 0.2 * (1.0 - s)
            loss.backward()
            out[f"{name}_{tag}_l1"], out[f"{name}_{tag}_ssim"] = Ll1.item(), s.item()
            out[f"{name}_{tag}_loss"], out[f"{name}_{tag}_grad"] = loss.item(), x.grad.numpy()
            if shape[0] > 1:
                out[f"{name}_{tag}_ssim_per_image"] = ssim(x.detach(), y, size_average=False).numpy()
    np.savez_compressed(os.path.join(HERE, "loss_golden.npz"), **out)
    print({k: (v.shape if hasattr(v, "shape") else v) for k, v in out.items()})


if __name__ == "__main__":
    main()
