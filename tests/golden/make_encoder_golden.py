"""Generate tests/golden/encoder_golden.npz from the REFERENCE's own UnetExtractor (core/extractor.py).

Run with GPSG_REFERENCE naming a checkout of the original project:  python tests/golden/make_encoder_golden.py
Builds UnetExtractor(in_channel=Cin, encoder_dim=[32, 48, 96]) for Cin = 3 (image) and Cin = 1 (depth) with torch's
seeded default init, the GroupNorm weights and biases randomised (the defaults 1 and 0 would hide affine bugs), every
parameter rounded to fp32 and the module converted to fp64; runs its own forward on the CPU with a forward hook on
`res1` that captures the stem's output.  Per case `<name>_*`: the input `x` (fp32) and `x1` (fp64), plus the parameters
the case changes (`p<i>`, index into gps_gaussian_b200.encoder.params_of order).  The base parameters `c<Cin>_p<i>`
(fp32) are shared by the cases of that channel count.
"""
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.environ["GPSG_REFERENCE"])
from core.extractor import UnetExtractor  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))


def _zero_var_bias(p):
    p = p.clone()
    p[:4] = p[0]                       # in_ds bias equal over GroupNorm(8)'s first group
    return p


# name: (Cin, B, H, W, input, {param index: transform of the base tensor})
CASES = {
    "rgb_16x24": (3, 2, 16, 24, "uniform", {}),
    "depth_16x24": (1, 2, 16, 24, "uniform", {}),
    "rgb_17x9": (3, 2, 17, 9, "uniform", {}),
    "depth_17x9": (1, 2, 17, 9, "uniform", {}),
    "rgb_1x1": (3, 2, 1, 1, "uniform", {}),
    "depth_1x1": (1, 2, 1, 1, "uniform", {}),
    "depth_zero": (1, 2, 16, 24, "zero", {}),
    "zero_var_group": (3, 2, 12, 20, "zero", {1: _zero_var_bias}),
    "offset": (3, 2, 16, 24, "offset", {}),
}


def params_of(e):
    out = [e.in_ds[0].weight, e.in_ds[0].bias, e.in_ds[1].weight, e.in_ds[1].bias]
    for blk in e.res1:
        out += [blk.conv1.weight, blk.conv1.bias, blk.norm1.weight, blk.norm1.bias,
                blk.conv2.weight, blk.conv2.bias, blk.norm2.weight, blk.norm2.bias]
    return out


def make_module(cin, seed):
    torch.manual_seed(seed)
    m = UnetExtractor(in_channel=cin, encoder_dim=[32, 48, 96])
    g = torch.Generator().manual_seed(seed + 1)
    with torch.no_grad():
        for mod in m.modules():
            if isinstance(mod, torch.nn.GroupNorm):
                sign = torch.where(torch.rand(mod.weight.shape, generator=g) < 0.15, -1.0, 1.0)
                mod.weight.copy_(sign * (0.5 + torch.rand(mod.weight.shape, generator=g)))
                mod.bias.copy_(torch.rand(mod.bias.shape, generator=g) - 0.5)
        for p in m.parameters():
            p.copy_(p.float())
    return m.double().eval()


def make_input(kind, cin, B, H, W, rng):
    if kind == "zero":
        return np.zeros((B, cin, H, W), np.float32)
    if kind == "offset":
        return (1000.0 + 0.01 * rng.standard_normal((B, cin, H, W))).astype(np.float32)
    return rng.uniform(-1, 1, (B, cin, H, W)).astype(np.float32) if cin == 3 else \
        rng.uniform(0, 1, (B, cin, H, W)).astype(np.float32)


def main():
    mods = {cin: make_module(cin, 10 + cin) for cin in (1, 3)}
    base = {cin: [p.detach().float().numpy().copy() for p in params_of(m)] for cin, m in mods.items()}
    rng = np.random.default_rng(2027)
    out = {f"c{cin}_p{i}": b for cin, bs in base.items() for i, b in enumerate(bs)}
    for name, (cin, B, H, W, kind, changes) in CASES.items():
        m = mods[cin]
        ps = params_of(m)
        with torch.no_grad():
            for i, p in enumerate(ps):
                p.copy_(torch.from_numpy(base[cin][i]).double())
                if i in changes:
                    p.copy_(changes[i](p).float().double())
        x = make_input(kind, cin, B, H, W, rng)
        seen = {}
        hook = m.res1.register_forward_hook(lambda mod, inp, o: seen.setdefault("x1", o.detach().clone()))
        try:
            with torch.no_grad():
                m(torch.from_numpy(x).double())
        finally:
            hook.remove()
        out[f"{name}_x"] = x
        out[f"{name}_x1"] = seen["x1"].numpy()
        for i in changes:
            out[f"{name}_p{i}"] = ps[i].detach().float().numpy()
    path = os.path.join(HERE, "encoder_golden.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path), "bytes,", len(CASES), "cases")


if __name__ == "__main__":
    main()
