"""Generate tests/golden/decoder23_golden.npz from the REFERENCE's own ResidualBlock (core/extractor.py) and nn.Upsample.

Run with GPSG_REFERENCE naming a checkout of the original project:  python tests/golden/make_decoder23_golden.py
Builds decoder3 and decoder2 as lib/gs_parm_network.py does with the stage-2 config (ResidualBlock(96 + 96, 96) then
ResidualBlock(96, 96); ResidualBlock(48 + 48 + 96, 64) then ResidualBlock(64, 64); norm_fn='group') and `up` =
nn.Upsample(scale_factor=2, mode="bilinear"), with torch's seeded default init for the biases, the GroupNorm weights
and biases randomised (the defaults 1 and 0 would hide affine bugs), the convolution weights drawn in torch's default
init range as multiples of 2^-10 by tests/decoder23_cases.py's `conv_weight` (seeded and exact, so the file keeps only
the seeds) and every parameter fp32; converts them to fp64 and runs on the CPU
    out3 = decoder3(cat(f3i, f3d)),  out2 = decoder2(cat(up(out3), f2i, f2d)).
Per case `<name>_*`: the inputs `f3i`, `f3d`, `f2i`, `f2d` (fp32) and `out3`, `out2` (fp64), plus the parameters the
case changes (`d3p<i>` / `d2p<i>`, index into gps_gaussian_b200.decoder.deep_params_of order).  The base biases and
GroupNorm parameters `d3p<i>` / `d2p<i>` (fp32) are shared by all cases; the convolution weights (indices
decoder23_cases.CONV_IDX) are not stored: `conv_weight(shape, CONV_SEED[stage] + i)` rebuilds them.
"""
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.environ["GPSG_REFERENCE"])
from core.extractor import ResidualBlock  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from decoder23_cases import CONV_IDX, CONV_SEED, conv_weight  # noqa: E402


def _zero_var_bias(p):
    p = p.clone()
    p[:8] = p[0]                       # conv1 bias equal over the first GroupNorm group
    return p


# name: (B, H, W at decoder3, input, {(stage, param index): transform of the base tensor})
CASES = {
    "b1_3x4": (1, 3, 4, "uniform", {}),
    "b1_5x3": (1, 5, 3, "uniform", {}),
    "b2_1x1": (2, 1, 1, "uniform", {}),
    "zero_var_group": (1, 2, 3, "zero", {("d3", 1): _zero_var_bias, ("d2", 1): _zero_var_bias}),
    "offset": (1, 2, 3, "offset", {}),
}


def params_of(dec):
    b0, b1 = dec
    return [b0.conv1.weight, b0.conv1.bias, b0.norm1.weight, b0.norm1.bias,
            b0.conv2.weight, b0.conv2.bias, b0.norm2.weight, b0.norm2.bias,
            b0.downsample[0].weight, b0.downsample[0].bias, b0.norm3.weight, b0.norm3.bias,
            b1.conv1.weight, b1.conv1.bias, b1.norm1.weight, b1.norm1.bias,
            b1.conv2.weight, b1.conv2.bias, b1.norm2.weight, b1.norm2.bias]


def make_module(stage, cin, c, seed):
    torch.manual_seed(seed)
    dec = torch.nn.Sequential(ResidualBlock(cin, c, norm_fn="group"), ResidualBlock(c, c, norm_fn="group"))
    g = torch.Generator().manual_seed(seed + 1)
    with torch.no_grad():
        for mod in dec.modules():
            if isinstance(mod, torch.nn.GroupNorm):
                sign = torch.where(torch.rand(mod.weight.shape, generator=g) < 0.15, -1.0, 1.0)
                mod.weight.copy_(sign * (0.5 + torch.rand(mod.weight.shape, generator=g)))
                mod.bias.copy_(torch.rand(mod.bias.shape, generator=g) - 0.5)
        for i, p in enumerate(params_of(dec)):
            p.copy_(torch.from_numpy(conv_weight(tuple(p.shape), CONV_SEED[stage] + i)) if i in CONV_IDX else p.float())
    return dec.double().eval()


def make_input(kind, shape, rng):
    if kind == "zero":
        return np.zeros(shape, np.float32)
    if kind == "offset":
        return (1000.0 + 0.01 * rng.standard_normal(shape)).astype(np.float32)
    return rng.uniform(0, 2, shape).astype(np.float32)


def main():
    decs = {"d3": make_module("d3", 96 + 96, 96, 41), "d2": make_module("d2", 48 + 48 + 96, 64, 43)}
    up = torch.nn.Upsample(scale_factor=2, mode="bilinear")
    base = {st: [p.detach().float().numpy().copy() for p in params_of(d)] for st, d in decs.items()}
    rng = np.random.default_rng(2029)
    out = {f"{st}p{i}": b for st, bs in base.items() for i, b in enumerate(bs) if i not in CONV_IDX}
    for name, (B, H, W, kind, changes) in CASES.items():
        for st, dec in decs.items():
            with torch.no_grad():
                for i, p in enumerate(params_of(dec)):
                    p.copy_(torch.from_numpy(base[st][i]).double())
                    if (st, i) in changes:
                        p.copy_(changes[st, i](p).float().double())
        ins = {"f3i": make_input(kind, (B, 96, H, W), rng), "f3d": make_input(kind, (B, 96, H, W), rng),
               "f2i": make_input(kind, (B, 48, 2 * H, 2 * W), rng), "f2d": make_input(kind, (B, 48, 2 * H, 2 * W), rng)}
        t = lambda a: torch.from_numpy(a).double()
        with torch.no_grad():
            out3 = decs["d3"](torch.cat([t(ins["f3i"]), t(ins["f3d"])], dim=1))
            out2 = decs["d2"](torch.cat([up(out3), t(ins["f2i"]), t(ins["f2d"])], dim=1))
        out.update({f"{name}_{k}": v for k, v in ins.items()})
        out.update({f"{name}_out3": out3.numpy(), f"{name}_out2": out2.numpy()})
        for st, i in changes:
            out[f"{name}_{st}p{i}"] = params_of(decs[st])[i].detach().float().numpy()
    path = os.path.join(HERE, "decoder23_golden.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path), "bytes,", len(CASES), "cases")


if __name__ == "__main__":
    main()
