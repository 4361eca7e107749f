"""Generate tests/golden/corr_golden.npz from the REFERENCE's own PyTorch correlation block.

Run with GPSG_REFERENCE naming a checkout of the original project:
    python tests/golden/make_corr_golden.py
It imports `CorrBlock1D` from reference core/corr.py:110-156 -- the in-repo twin of the CUDA
`CorrBlockFast1D`/`corr_sampler` path (README.md:34: same results) -- runs it on seeded inputs on the CPU in
fp64, and stores inputs, the [B,36,H,W] lookup, every pyramid level, and per-level d(loss)/d(volume) obtained
by autograd with each level made a leaf (== what corr_sampler.backward must return)."""
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.environ["GPSG_REFERENCE"])
from core.corr import CorrBlock1D  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))


def main():
    rng = np.random.default_rng(1314)
    B, D, H, W = 2, 24, 3, 40
    f1 = torch.tensor(rng.standard_normal((B, D, H, W)))
    f2 = torch.tensor(rng.standard_normal((B, D, H, W)))
    xs = np.broadcast_to(np.arange(W, dtype=np.float64), (B, H, W))
    ys = np.broadcast_to(np.arange(H, dtype=np.float64)[:, None], (B, H, W))
    cx = xs + rng.normal(0, 6.0, (B, H, W))
    cx[0, 0, :6] = [-7.5, -4.0, 0.0, W - 1.0, W + 3.25, 2.0]       # out-of-range / integer / border cases
    coords = torch.tensor(np.stack([cx, ys], 1))
    blk = CorrBlock1D(f1, f2, num_levels=4, radius=4)
    levels = [blk.corr_pyramid[i].detach().clone().requires_grad_(True) for i in range(4)]
    for i in range(4):
        blk.corr_pyramid[i] = levels[i]
    out = blk(coords)                                               # [B,36,H,W] (.float() in the reference)
    gout = torch.tensor(rng.standard_normal(tuple(out.shape)))
    (out.double() * gout).sum().backward()
    np.savez_compressed(
        os.path.join(HERE, "corr_golden.npz"), fmap1=f1.numpy(), fmap2=f2.numpy(), coords=coords.numpy(),
        out=out.detach().numpy(), grad_out=gout.numpy(),
        **{f"level{i}": levels[i].detach().numpy().reshape(B, H, W, -1) for i in range(4)},
        **{f"grad_level{i}": levels[i].grad.numpy().reshape(B, H, W, -1) for i in range(4)})
    print("wrote corr_golden.npz", out.shape, out.dtype)


if __name__ == "__main__":
    main()
