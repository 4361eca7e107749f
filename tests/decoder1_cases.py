"""Cases of the decoder1 tests: the golden cases (tests/golden/decoder1_golden.npz, the reference's own ResidualBlocks and
nn.Upsample in fp64) and seeded sweeps, as (s, f_i, f_d, params) fp32 CPU tensors with params in decoder.params_of
order."""
import os
from dataclasses import dataclass

import numpy as np
import torch

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "decoder1_golden.npz")
GOLDEN_CASES = ("b1_6x8", "b1_9x5", "b2_1x1", "zero_var_group", "offset")


def shapes():
    blk0 = ((48, 128, 3, 3), (48,), (48,), (48,), (48, 48, 3, 3), (48,), (48,), (48,),
            (48, 128, 1, 1), (48,), (48,), (48,))
    blk1 = ((48, 48, 3, 3), (48,), (48,), (48,)) * 2
    return blk0 + blk1


@dataclass
class Case:
    id: str
    B: int
    Hs: int
    Ws: int
    seed: int = 0
    special: str = ""          # "", "nan", "inf"


def golden(name):
    """(s, f_i, f_d, params, out) of a golden case; out fp64."""
    z = np.load(GOLDEN)
    t = lambda k: torch.from_numpy(z[k])
    ps = [t(f"{name}_p{i}" if f"{name}_p{i}" in z.files else f"p{i}") for i in range(20)]
    return t(f"{name}_s"), t(f"{name}_fi"), t(f"{name}_fd"), ps, t(f"{name}_out")


def params(seed):
    """Conv2d's default init range (uniform in +-1/sqrt(fan_in)) for weights and biases, GroupNorm weights in +-[0.5, 1.5]
    and biases in [-0.5, 0.5], seeded."""
    g = torch.Generator().manual_seed(seed)
    out, fan = [], 1
    for i, s in enumerate(shapes()):
        k = i % 4
        if k == 0:
            fan = s[1] * s[2] * s[3]
            out.append((torch.rand(s, generator=g) * 2 - 1) / fan ** 0.5)
        elif k == 1:
            out.append((torch.rand(s, generator=g) * 2 - 1) / fan ** 0.5)
        elif k == 2:
            sign = torch.where(torch.rand(s, generator=g) < 0.15, -1.0, 1.0)
            out.append(sign * (0.5 + torch.rand(s, generator=g)))
        else:
            out.append(torch.rand(s, generator=g) - 0.5)
    return out


def inputs(case):
    """s [B,64,Hs,Ws] like a decoder output (ReLU'd, so >= 0), f_i and f_d [B,32,2Hs,2Ws] like encoder features; a
    "nan" / "inf" case puts one non-finite value into sample 0 of f_i."""
    g = torch.Generator().manual_seed(1000 + case.seed)
    s = torch.rand(case.B, 64, case.Hs, case.Ws, generator=g) * 2
    f_i = torch.rand(case.B, 32, 2 * case.Hs, 2 * case.Ws, generator=g) * 2
    f_d = torch.rand(case.B, 32, 2 * case.Hs, 2 * case.Ws, generator=g) * 2
    if case.special in ("nan", "inf"):
        f_i[0, 3, case.Hs, 2 * case.Ws - 1] = float("nan") if case.special == "nan" else float("inf")
    return s, f_i, f_d, params(case.seed)


SWEEP = [Case("tiny_3x2", 1, 3, 2, 1), Case("b2_5x7", 2, 5, 7, 2), Case("nan_4x6", 2, 4, 6, 5, "nan"),
         Case("inf_3x5", 2, 3, 5, 6, "inf")]
