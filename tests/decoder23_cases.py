"""Cases of the decoder3 / decoder2 tests: the golden cases (tests/golden/decoder23_golden.npz, the reference's own
ResidualBlocks and nn.Upsample in fp64) and seeded sweeps, as fp32 CPU tensors with params in
decoder.deep_params_of order.  Sizes are decoder3's [H,W]; decoder2 runs at [2H,2W]."""
import os
from dataclasses import dataclass

import numpy as np
import torch

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "decoder23_golden.npz")
GOLDEN_CASES = ("b1_3x4", "b1_5x3", "b2_1x1", "zero_var_group", "offset")


def shapes(c):
    k = 192
    return ((c, k, 3, 3), (c,), (c,), (c,), (c, c, 3, 3), (c,), (c,), (c,), (c, k, 1, 1), (c,), (c,), (c,),
            (c, c, 3, 3), (c,), (c,), (c,), (c, c, 3, 3), (c,), (c,), (c,))


@dataclass
class Case:
    id: str
    B: int
    H: int
    W: int
    seed: int = 0
    special: str = ""          # "", "nan", "inf"


WEIGHT_SCALE = 1024.0     # golden convolution weights are integer multiples of 1 / WEIGHT_SCALE
CONV_IDX = (0, 4, 8, 12, 16)                     # the convolution weights in deep_params_of order
CONV_SEED = {"d3": 3000, "d2": 2000}             # + the parameter index


def _splitmix64(x):
    x = x + np.uint64(0x9E3779B97F4A7C15)
    x = (x ^ (x >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
    x = (x ^ (x >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
    return x ^ (x >> np.uint64(31))


def conv_weight(shape, seed):
    """A convolution weight of the golden file's modules: torch's default init range (uniform in +-1/sqrt(fan_in)),
    drawn as integer multiples of 1 / WEIGHT_SCALE from a splitmix64 stream, so it is exact and the same on every
    platform and library version; the file stores the seed, not the 0.67 M values."""
    n, fan = int(np.prod(shape)), int(np.prod(shape[1:]))
    k = int(WEIGHT_SCALE / fan ** 0.5)
    z = _splitmix64(np.arange(n, dtype=np.uint64) + np.full(n, seed, dtype=np.uint64) * np.uint64(1 << 32))
    q = (z % np.uint64(2 * k + 1)).astype(np.int64) - k
    return (q / WEIGHT_SCALE).astype(np.float32).reshape(shape)


def golden(name):
    """dict(f3i, f3d, f2i, f2d, p3, p2, out3, out2) of a golden case; out3 and out2 fp64, the parameters fp32."""
    z = np.load(GOLDEN)
    t = lambda k: torch.from_numpy(z[k])
    ps = {}
    for st, c in (("d3", 96), ("d2", 64)):
        ps[st] = [torch.from_numpy(conv_weight(shapes(c)[i], CONV_SEED[st] + i)) if i in CONV_IDX
                  else t(f"{name}_{st}p{i}" if f"{name}_{st}p{i}" in z.files else f"{st}p{i}") for i in range(20)]
    d = {k: t(f"{name}_{k}") for k in ("f3i", "f3d", "f2i", "f2d", "out3", "out2")}
    return dict(d, p3=ps["d3"], p2=ps["d2"])


def params(c, seed):
    """Conv2d's default init range (uniform in +-1/sqrt(fan_in)) for weights and biases, GroupNorm weights in +-[0.5, 1.5]
    and biases in [-0.5, 0.5], seeded."""
    g = torch.Generator().manual_seed(seed)
    out, fan = [], 1
    for i, s in enumerate(shapes(c)):
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
    """dict(f3i, f3d [B,96,H,W], f2i, f2d [B,48,2H,2W], s [B,96,H,W] (a decoder output: ReLU'd, so >= 0), p3, p2), like
    encoder features; a "nan" / "inf" case puts one non-finite value into sample 0 of f3i and of f2i."""
    g = torch.Generator().manual_seed(2000 + case.seed)
    B, H, W = case.B, case.H, case.W
    d = dict(f3i=torch.rand(B, 96, H, W, generator=g) * 2, f3d=torch.rand(B, 96, H, W, generator=g) * 2,
             f2i=torch.rand(B, 48, 2 * H, 2 * W, generator=g) * 2, f2d=torch.rand(B, 48, 2 * H, 2 * W, generator=g) * 2,
             s=torch.rand(B, 96, H, W, generator=g) * 2)
    if case.special in ("nan", "inf"):
        bad = float("nan") if case.special == "nan" else float("inf")
        d["f3i"][0, 5, H - 1, W // 2] = bad
        d["f2i"][0, 7, H, 2 * W - 1] = bad
    return dict(d, p3=params(96, case.seed), p2=params(64, 100 + case.seed))


def stage_args(d, stage, s=None):
    """(srcs, params) of one stage from an inputs() / golden() dict; decoder2 takes s (default d["s"])."""
    if stage == "d3":
        return (d["f3i"], d["f3d"]), d["p3"]
    return (d["s"] if s is None else s, d["f2i"], d["f2d"]), d["p2"]


SWEEP = [Case("tiny_2x3", 1, 2, 3, 1), Case("b2_3x5", 2, 3, 5, 2), Case("nan_3x4", 2, 3, 4, 5, "nan"),
         Case("inf_2x3", 2, 2, 3, 6, "inf")]
