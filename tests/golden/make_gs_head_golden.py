"""Generate tests/golden/gs_head_golden.npz from the REFERENCE's own GSRegresser (lib/gs_parm_network.py).

Run with GPSG_REFERENCE naming a checkout of the original project:  python tests/golden/make_gs_head_golden.py
Builds the module with the stage-2 config's dimensions (decoder_dims [48, 64, 96], head_dim 32), seeds its weights
with torch's default init, converts it to fp64 and runs its own forward on the CPU with a forward hook that replaces
the decoder1 output by a seeded tensor, so the full-resolution tail (upsample, cat, out_conv, the three heads and
their activations) is the reference's code on known inputs.  Per case `<name>_*`: the tail's inputs `src` (decoder1
output [B,48,H/2,W/2]), `img`, `depth` (fp32 values), the outputs `rot`, `scale`, `opacity` (fp64), and the 1x1 layers
and biases the case changes (`p<i>`, index into gps_gaussian_b200.gs_head.params_of order).  The base weights `base_p<i>`
(fp32) are shared by every case.
"""
import os
import sys
import types

import numpy as np
import torch

sys.path.insert(0, os.environ["GPSG_REFERENCE"])
from lib.gs_parm_network import GSRegresser  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))

# name: (B, H, W, {param index: transform of the base tensor})
CASES = {
    "default": (1, 16, 24, {}),
    "rot_zero": (1, 16, 24, {4: lambda p: p * 0, 5: lambda p: p * 0}),                 # pre = 0: normalize's eps
    "saturate": (1, 16, 24, {8: lambda p: p * 400, 12: lambda p: p * 400}),            # softplus threshold, sigmoid 0/1
    "clamp": (1, 16, 24, {8: lambda p: p * 0.05, 9: lambda p: p * 0 + 0.008}),          # softplus on both sides of 0.01
    "nonsquare": (2, 24, 40, {}),                                                       # tiles do not divide 40
}


def params_of(r):
    return [r.out_conv.weight, r.out_conv.bias] + [t for h in (r.rot_head, r.scale_head, r.opacity_head)
                                                   for t in (h[0].weight, h[0].bias, h[2].weight, h[2].bias)]


def make_module():
    cfg = types.SimpleNamespace(raft=types.SimpleNamespace(encoder_dims=[32, 48, 96]),
                                gsnet=types.SimpleNamespace(encoder_dims=[32, 48, 96], decoder_dims=[48, 64, 96],
                                                            parm_head_dim=32))
    torch.manual_seed(7)
    m = GSRegresser(cfg, rgb_dim=3, depth_dim=1)
    with torch.no_grad():
        for p in m.parameters():
            p.copy_(p.float())                                    # fp32 values, as the kernels receive them
    return m.double().eval()


def run_case(m, base, rng, B, H, W, changes):
    ps = params_of(m)
    with torch.no_grad():
        for i, p in enumerate(ps):
            p.copy_(torch.from_numpy(base[i]).double())
            if i in changes:
                p.copy_(changes[i](p).float().double())
    src = rng.standard_normal((B, 48, H // 2, W // 2)).astype(np.float32)
    img = rng.uniform(-1, 1, (B, 3, H, W)).astype(np.float32)
    depth = rng.uniform(0, 1, (B, 1, H, W)).astype(np.float32)
    feats = [torch.from_numpy(rng.standard_normal((B, c, H // s, W // s))).double()
             for c, s in ((32, 2), (48, 4), (96, 8))]
    hook = m.decoder1.register_forward_hook(lambda mod, inp, out: torch.from_numpy(src).double())
    try:
        with torch.no_grad():
            rot, scale, opacity = m(torch.from_numpy(img).double(), torch.from_numpy(depth).double(), feats)
    finally:
        hook.remove()
    rec = dict(src=src, img=img, depth=depth, rot=rot.numpy(), scale=scale.numpy(), opacity=opacity.numpy())
    for i in changes:
        rec[f"p{i}"] = ps[i].detach().float().numpy()
    return rec


def main():
    m = make_module()
    base = [p.detach().float().numpy().copy() for p in params_of(m)]
    rng = np.random.default_rng(2026)
    out = {f"base_p{i}": b for i, b in enumerate(base)}
    for name, (B, H, W, changes) in CASES.items():
        for k, v in run_case(m, base, rng, B, H, W, changes).items():
            out[f"{name}_{k}"] = v
    path = os.path.join(HERE, "gs_head_golden.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path), "bytes,", len(CASES), "cases")


if __name__ == "__main__":
    main()
