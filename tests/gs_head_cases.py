"""Cases of the regressor-tail tests: the golden cases (tests/golden/gs_head_golden.npz, the reference's own module in
fp64) and seeded sweeps, as (src, img, depth, params) fp32 CPU tensors with params in gs_head.params_of order."""
import os
from dataclasses import dataclass, field

import numpy as np
import torch

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "gs_head_golden.npz")
GOLDEN_CASES = ("default", "rot_zero", "saturate", "clamp", "nonsquare")
SHAPES = ((32, 52, 3, 3), (32,), (32, 32, 3, 3), (32,), (4, 32, 1, 1), (4,), (32, 32, 3, 3), (32,), (3, 32, 1, 1), (3,),
          (32, 32, 3, 3), (32,), (1, 32, 1, 1), (1,))


@dataclass
class Case:
    id: str
    B: int
    H: int
    W: int
    seed: int = 0
    special: str = ""            # "", "positive", "nan_depth", "inf_depth"
    extra: dict = field(default_factory=dict)


def golden(name):
    """(src, img, depth, params, want) of a golden case; want = dict(rot, scale, opacity) in fp64."""
    z = np.load(GOLDEN)
    ps = [torch.from_numpy(z[f"{name}_p{i}"] if f"{name}_p{i}" in z.files else z[f"base_p{i}"]) for i in range(14)]
    src, img, depth = (torch.from_numpy(z[f"{name}_{k}"]) for k in ("src", "img", "depth"))
    return src, img, depth, ps, {k: torch.from_numpy(z[f"{name}_{k}"]) for k in ("rot", "scale", "opacity")}


def params(seed, positive=False):
    """Conv2d's default init (uniform in +-1/sqrt(fan_in), weights and biases), seeded; positive: magnitudes only."""
    g = torch.Generator().manual_seed(seed)
    out = []
    for i, s in enumerate(SHAPES):
        fan_in = int(np.prod(SHAPES[i if len(s) == 4 else i - 1][1:]))
        p = (torch.rand(s, generator=g) * 2 - 1) / fan_in ** 0.5
        out.append(p.abs() if positive else p)
    return out


def inputs(case):
    g = torch.Generator().manual_seed(1000 + case.seed)
    B, H, W = case.B, case.H, case.W
    src = torch.randn(B, 48, H // 2, W // 2, generator=g)
    img = torch.rand(B, 3, H, W, generator=g) * 2 - 1
    depth = torch.rand(B, 1, H, W, generator=g)
    if case.special == "positive":
        src, img = src.abs(), img.abs()
    if case.special in ("nan_depth", "inf_depth"):
        depth[0, 0, H // 2, W - 3] = float("nan") if case.special == "nan_depth" else float("inf")
        depth[-1, 0, 0, 0] = float("nan") if case.special == "nan_depth" else float("inf")
    return src, img, depth, params(case.seed, case.special == "positive")


SWEEP = [Case("tiny_10x6", 1, 10, 6, 1), Case("b2_18x34", 2, 18, 34, 2), Case("row_8x66", 1, 8, 66, 3),
         Case("positive_12x20", 1, 12, 20, 4, "positive"), Case("nan_depth_14x36", 2, 14, 36, 5, "nan_depth"),
         Case("inf_depth_12x10", 1, 12, 10, 6, "inf_depth")]
