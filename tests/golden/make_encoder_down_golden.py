"""Generate tests/golden/encoder_down_golden.npz from the REFERENCE's own ResidualBlock (core/extractor.py).

Run with GPSG_REFERENCE naming a checkout of the original project:  python tests/golden/make_encoder_down_golden.py
Builds res2 and res3 as UnetExtractor does with encoder_dim [32, 48, 96] (ResidualBlock(32, 48, stride 2) then
ResidualBlock(48, 48); ResidualBlock(48, 96, stride 2) then ResidualBlock(96, 96); norm_fn='group') with torch's seeded
default init, the GroupNorm weights and biases randomised (the defaults 1 and 0 would hide affine bugs), the convolution
weights rounded to multiples of 2^-12 (so the file stays small) and every parameter fp32; converts them to fp64 and runs
them on the CPU.  Per case `<name>_*`: the input `x` (fp32) and `out` (fp64), plus the parameters the case changes
(`p<i>`, index into gps_gaussian_b200.encoder.down_params_of order).  The base parameters `res2_p<i>` / `res3_p<i>`
(fp32) are shared by the cases of their stage, which the input's channel count names.
"""
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.environ["GPSG_REFERENCE"])
from core.extractor import ResidualBlock  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
DIMS = {"res2": (32, 48), "res3": (48, 96)}


def _zero_var_bias(p):
    p = p.clone()
    p[:8] = p[0]                       # conv1 bias equal over the first GroupNorm group: with a zero input, zero variance
    return p


# name: (stage, B, H, W, input, {param index: transform of the base tensor})
CASES = {
    "res2_9x5": ("res2", 1, 9, 5, "relu", {}),
    "res2_b2_6x8": ("res2", 2, 6, 8, "relu", {}),
    "res2_1x1": ("res2", 1, 1, 1, "relu", {}),
    "res2_zero_var_group": ("res2", 1, 3, 4, "zero", {1: _zero_var_bias}),
    "res2_offset": ("res2", 1, 4, 3, "offset", {}),
    "res3_5x3": ("res3", 1, 5, 3, "relu", {}),
    "res3_1x1": ("res3", 2, 1, 1, "relu", {}),
    "res3_offset": ("res3", 1, 3, 2, "offset", {}),
}


def params_of(stage):
    b0, b1 = stage
    return [b0.conv1.weight, b0.conv1.bias, b0.norm1.weight, b0.norm1.bias,
            b0.conv2.weight, b0.conv2.bias, b0.norm2.weight, b0.norm2.bias,
            b0.downsample[0].weight, b0.downsample[0].bias, b0.norm3.weight, b0.norm3.bias,
            b1.conv1.weight, b1.conv1.bias, b1.norm1.weight, b1.norm1.bias,
            b1.conv2.weight, b1.conv2.bias, b1.norm2.weight, b1.norm2.bias]


def make_module(cin, c, seed):
    torch.manual_seed(seed)
    st = torch.nn.Sequential(ResidualBlock(cin, c, norm_fn="group", stride=2), ResidualBlock(c, c, norm_fn="group"))
    g = torch.Generator().manual_seed(seed + 1)
    with torch.no_grad():
        for mod in st.modules():
            if isinstance(mod, torch.nn.GroupNorm):
                sign = torch.where(torch.rand(mod.weight.shape, generator=g) < 0.15, -1.0, 1.0)
                mod.weight.copy_(sign * (0.5 + torch.rand(mod.weight.shape, generator=g)))
                mod.bias.copy_(torch.rand(mod.bias.shape, generator=g) - 0.5)
            elif isinstance(mod, torch.nn.Conv2d):
                mod.weight.copy_(torch.round(mod.weight * 4096) / 4096)
        for p in st.parameters():
            p.copy_(p.float())
    return st.double().eval()


def make_input(kind, shape, rng):
    if kind == "zero":
        return np.zeros(shape, np.float32)
    if kind == "offset":
        return (1000.0 + 0.01 * rng.standard_normal(shape)).astype(np.float32)
    return np.maximum(rng.standard_normal(shape), 0).astype(np.float32)


def main():
    mods = {name: make_module(cin, c, 41 + i) for i, (name, (cin, c)) in enumerate(DIMS.items())}
    base = {name: [p.detach().float().numpy().copy() for p in params_of(m)] for name, m in mods.items()}
    rng = np.random.default_rng(2029)
    out = {f"{name}_p{i}": b for name, bs in base.items() for i, b in enumerate(bs)}
    for name, (stage, B, H, W, kind, changes) in CASES.items():
        ps = params_of(mods[stage])
        with torch.no_grad():
            for i, p in enumerate(ps):
                p.copy_(torch.from_numpy(base[stage][i]).double())
                if i in changes:
                    p.copy_(changes[i](p).float().double())
        x = make_input(kind, (B, DIMS[stage][0], H, W), rng)
        with torch.no_grad():
            y = mods[stage](torch.from_numpy(x).double())
        out.update({f"{name}_x": x, f"{name}_out": y.numpy()})
        for i in changes:
            out[f"{name}_p{i}"] = ps[i].detach().float().numpy()
    path = os.path.join(HERE, "encoder_down_golden.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path), "bytes,", len(CASES), "cases")


if __name__ == "__main__":
    main()
