"""Cases of the encoder-stem tests: the golden cases (tests/golden/encoder_golden.npz, the reference's own
UnetExtractor in fp64) and seeded sweeps, as (x, params) fp32 CPU tensors with params in encoder.params_of order."""
import os
from dataclasses import dataclass

import numpy as np
import torch

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "encoder_golden.npz")
GOLDEN_CASES = ("rgb_16x24", "depth_16x24", "rgb_17x9", "depth_17x9", "rgb_1x1", "depth_1x1", "depth_zero",
                "zero_var_group", "offset")


def shapes(cin):
    blk = ((32, 32, 3, 3), (32,), (32,), (32,)) * 2
    return ((32, cin, 5, 5), (32,), (32,), (32,)) + blk * 2


@dataclass
class Case:
    id: str
    cin: int
    B: int
    H: int
    W: int
    seed: int = 0
    special: str = ""          # "", "positive", "trunc_bits", "nan", "inf"


def golden(name):
    """(x, params, x1) of a golden case; x1 fp64."""
    z = np.load(GOLDEN)
    x = torch.from_numpy(z[f"{name}_x"])
    cin = x.shape[1]
    ps = [torch.from_numpy(z[f"{name}_p{i}"] if f"{name}_p{i}" in z.files else z[f"c{cin}_p{i}"]) for i in range(20)]
    return x, ps, torch.from_numpy(z[f"{name}_x1"])


def _low_bits_set(t):
    """t with the 13 mantissa bits below TF32's precision all set: truncating them loses almost a full TF32 ulp, while
    rounding to nearest moves by 2^-13 of one."""
    return (t.contiguous().view(torch.int32) | 0x1FFF).view(torch.float32)


def params(seed, cin, special=""):
    """Conv2d's default init (uniform in +-1/sqrt(fan_in)), GroupNorm weights in +-[0.5, 1.5] and biases in [-0.5, 0.5],
    seeded; positive / trunc_bits: positive convolution weights (trunc_bits: with the low mantissa bits set)."""
    g = torch.Generator().manual_seed(seed)
    out = []
    for s in shapes(cin):
        if len(s) == 4:
            fan_in = s[1] * s[2] * s[3]
            p = (torch.rand(s, generator=g) * 2 - 1) / fan_in ** 0.5
            if special in ("positive", "trunc_bits"):
                p = p.abs()
            if special == "trunc_bits":
                p = _low_bits_set(p)
            out.append(p)
            last_fan = fan_in
        elif len(out) % 4 == 1:                                      # convolution bias
            out.append((torch.rand(s, generator=g) * 2 - 1) / last_fan ** 0.5)
        elif len(out) % 4 == 2:                                      # GroupNorm weight
            sign = torch.where(torch.rand(s, generator=g) < 0.15, -1.0, 1.0)
            out.append(sign * (0.5 + torch.rand(s, generator=g)))
        else:                                                        # GroupNorm bias
            out.append(torch.rand(s, generator=g) - 0.5)
    return out


def inputs(case):
    g = torch.Generator().manual_seed(1000 + case.seed)
    x = torch.rand(case.B, case.cin, case.H, case.W, generator=g)
    if case.cin == 3 and case.special not in ("positive", "trunc_bits"):
        x = x * 2 - 1
    if case.special == "trunc_bits":
        x = _low_bits_set(x * 0.5 + 0.5)
    if case.special in ("nan", "inf"):
        x[0, 0, case.H // 2, case.W - 2] = float("nan") if case.special == "nan" else float("inf")
    return x, params(case.seed, case.cin, case.special)


SWEEP = [Case("rgb_tiny_10x6", 3, 1, 10, 6, 1), Case("depth_b2_18x34", 1, 2, 18, 34, 2),
         Case("rgb_positive_12x20", 3, 1, 12, 20, 3, "positive"), Case("rgb_trunc_bits_8x8", 3, 1, 8, 8, 4, "trunc_bits"),
         Case("depth_nan_14x12", 1, 2, 14, 12, 5, "nan"), Case("rgb_inf_9x11", 3, 2, 9, 11, 6, "inf")]
