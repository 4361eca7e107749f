"""Generate tests/golden/decoder1_golden.npz from the REFERENCE's own ResidualBlock (core/extractor.py) and nn.Upsample.

Run with GPSG_REFERENCE naming a checkout of the original project:  python tests/golden/make_decoder1_golden.py
Builds decoder1 as lib/gs_parm_network.py does with the stage-2 config (ResidualBlock(32 + 32 + 64, 48) then
ResidualBlock(48, 48), norm_fn='group') and `up` = nn.Upsample(scale_factor=2, mode="bilinear"), with torch's seeded
default init, the GroupNorm weights and biases randomised (the defaults 1 and 0 would hide affine bugs), the convolution
weights rounded to multiples of 2^-12 (so the file stays small) and every parameter fp32; converts it to fp64 and runs
decoder1(cat(up(s), f_i, f_d)) on the CPU.  Per case `<name>_*`: the inputs `s`, `fi`, `fd` (fp32) and `out` (fp64),
plus the parameters the case changes (`p<i>`, index into gps_gaussian_b200.decoder.params_of order).  The base
parameters `p<i>` (fp32) are shared by all cases.
"""
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.environ["GPSG_REFERENCE"])
from core.extractor import ResidualBlock  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))


def _zero_var_bias(p):
    p = p.clone()
    p[:8] = p[0]                       # conv1 bias equal over GroupNorm(6)'s first group
    return p


# name: (B, Hs, Ws, input, {param index: transform of the base tensor})
CASES = {
    "b1_6x8": (1, 6, 8, "uniform", {}),
    "b1_9x5": (1, 9, 5, "uniform", {}),
    "b2_1x1": (2, 1, 1, "uniform", {}),
    "zero_var_group": (1, 3, 4, "zero", {1: _zero_var_bias}),
    "offset": (1, 3, 4, "offset", {}),
}


def params_of(dec):
    b0, b1 = dec
    return [b0.conv1.weight, b0.conv1.bias, b0.norm1.weight, b0.norm1.bias,
            b0.conv2.weight, b0.conv2.bias, b0.norm2.weight, b0.norm2.bias,
            b0.downsample[0].weight, b0.downsample[0].bias, b0.norm3.weight, b0.norm3.bias,
            b1.conv1.weight, b1.conv1.bias, b1.norm1.weight, b1.norm1.bias,
            b1.conv2.weight, b1.conv2.bias, b1.norm2.weight, b1.norm2.bias]


def make_module(seed):
    torch.manual_seed(seed)
    dec = torch.nn.Sequential(ResidualBlock(32 + 32 + 64, 48, norm_fn="group"), ResidualBlock(48, 48, norm_fn="group"))
    g = torch.Generator().manual_seed(seed + 1)
    with torch.no_grad():
        for mod in dec.modules():
            if isinstance(mod, torch.nn.GroupNorm):
                sign = torch.where(torch.rand(mod.weight.shape, generator=g) < 0.15, -1.0, 1.0)
                mod.weight.copy_(sign * (0.5 + torch.rand(mod.weight.shape, generator=g)))
                mod.bias.copy_(torch.rand(mod.bias.shape, generator=g) - 0.5)
            elif isinstance(mod, torch.nn.Conv2d):
                mod.weight.copy_(torch.round(mod.weight * 4096) / 4096)
        for p in dec.parameters():
            p.copy_(p.float())
    return dec.double().eval()


def make_input(kind, shape, rng):
    if kind == "zero":
        return np.zeros(shape, np.float32)
    if kind == "offset":
        return (1000.0 + 0.01 * rng.standard_normal(shape)).astype(np.float32)
    return rng.uniform(0, 2, shape).astype(np.float32)


def main():
    dec = make_module(31)
    up = torch.nn.Upsample(scale_factor=2, mode="bilinear")
    base = [p.detach().float().numpy().copy() for p in params_of(dec)]
    rng = np.random.default_rng(2028)
    out = {f"p{i}": b for i, b in enumerate(base)}
    for name, (B, Hs, Ws, kind, changes) in CASES.items():
        ps = params_of(dec)
        with torch.no_grad():
            for i, p in enumerate(ps):
                p.copy_(torch.from_numpy(base[i]).double())
                if i in changes:
                    p.copy_(changes[i](p).float().double())
        s = make_input(kind, (B, 64, Hs, Ws), rng)
        fi = make_input(kind, (B, 32, 2 * Hs, 2 * Ws), rng)
        fd = make_input(kind, (B, 32, 2 * Hs, 2 * Ws), rng)
        with torch.no_grad():
            t = lambda a: torch.from_numpy(a).double()
            y = dec(torch.cat([up(t(s)), t(fi), t(fd)], dim=1))
        out.update({f"{name}_s": s, f"{name}_fi": fi, f"{name}_fd": fd, f"{name}_out": y.numpy()})
        for i in changes:
            out[f"{name}_p{i}"] = ps[i].detach().float().numpy()
    path = os.path.join(HERE, "decoder1_golden.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path), "bytes,", len(CASES), "cases")


if __name__ == "__main__":
    main()
