"""Generate tests/golden/gs_head_grad_golden.npz from the REFERENCE's own GSRegresser (lib/gs_parm_network.py).

Run with GPSG_REFERENCE naming a checkout of the original project:  python tests/golden/make_gs_head_grad_golden.py
The module is built as in make_gs_head_golden.py (stage-2 dimensions, seeded default init, fp64 on the CPU).  A forward
hook replaces the decoder1 output by a seeded leaf `src` that requires grad, `depth` requires grad, and seeded upstream
gradients of rot, scale and opacity go into torch.autograd.backward, so the full-resolution tail's backward is the
reference's own autograd.  Per case `<name>_*`: the inputs `src`, `img`, `depth` and `g_rot`, `g_scale`, `g_opacity`
(fp32 values), the gradients `d_src`, `d_depth` and `g<i>` of parameter i in gps_gaussian_b200.gs_head.params_of order
(fp64), and the parameters the case changes (`p<i>`).  The gradients of the four 3x3 weights (`g0`, `g2`, `g6`, `g10`)
are stored as every `<name>_stride`-th element of the flattened tensor (a stride prime to 9 and to the channel counts,
so every tap and every channel pair appears), with `<name>_finite<i>`, the full tensor's isfinite mask, bit-packed;
every other gradient is stored whole.  The base weights are tests/golden/gs_head_golden.npz's `base_p<i>`: the same
seeded module, checked here.
"""
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from make_gs_head_golden import make_module, params_of  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))

# name: (B, H, W, {param index: transform of the base tensor}, special, stride of the 3x3 weight gradients)
CASES = {
    "default": (1, 8, 16, {}, "", 7),
    "rot_zero": (1, 8, 16, {4: lambda p: p * 0, 5: lambda p: p * 0}, "", 13),              # normalize's eps branch
    "saturate": (1, 8, 16, {8: lambda p: p * 400, 12: lambda p: p * 400}, "", 13),         # softplus threshold, sigmoid
    "clamp": (1, 8, 16, {8: lambda p: p * 0.05, 9: lambda p: p * 0 + 0.008}, "", 13),       # both sides of 0.01
    "nonsquare": (2, 8, 24, {}, "", 13),                                                    # two samples, H != W
    "nan_depth": (1, 8, 16, {}, "nan_depth", 13),                                           # one NaN depth pixel
    "inf_g_scale": (1, 8, 16, {}, "inf_g_scale", 13),                                       # inf upstream gradients
}
SAMPLED = (0, 2, 6, 10)                                                                     # out_w, *_w1


def run_case(m, base, rng, B, H, W, changes, special, stride):
    ps = params_of(m)
    with torch.no_grad():
        for i, p in enumerate(ps):
            p.copy_(torch.from_numpy(base[i]).double())
            if i in changes:
                p.copy_(changes[i](p).float().double())
            p.grad = None
    src = rng.standard_normal((B, 48, H // 2, W // 2)).astype(np.float32)
    img = rng.uniform(-1, 1, (B, 3, H, W)).astype(np.float32)
    depth = rng.uniform(0, 1, (B, 1, H, W)).astype(np.float32)
    gs = [rng.standard_normal((B, c, H, W)).astype(np.float32) for c in (4, 3, 1)]
    if special == "nan_depth":
        depth[0, 0, H // 2, W - 3] = np.nan
    if special == "inf_g_scale":
        gs[1][0, :, 5, 7] = np.inf                    # all three channels: at least one is below the clamp
        gs[1][0, 0, 6, 2] = -np.inf
    feats = [torch.from_numpy(rng.standard_normal((B, c, H // s, W // s))).double()
             for c, s in ((32, 2), (48, 4), (96, 8))]
    s = torch.from_numpy(src).double().requires_grad_()
    d = torch.from_numpy(depth).double().requires_grad_()
    hook = m.decoder1.register_forward_hook(lambda mod, inp, out: s)
    try:
        outs = m(torch.from_numpy(img).double(), d, feats)
        torch.autograd.backward(outs, [torch.from_numpy(g).double() for g in gs])
    finally:
        hook.remove()
    rec = dict(src=src, img=img, depth=depth, g_rot=gs[0], g_scale=gs[1], g_opacity=gs[2], d_src=s.grad.numpy(),
               d_depth=d.grad.numpy())
    for i, p in enumerate(ps):
        g = p.grad.numpy()
        if i in SAMPLED:
            rec[f"g{i}"] = g.reshape(-1)[::stride].copy()
            rec[f"finite{i}"] = np.packbits(np.isfinite(g).reshape(-1))
        else:
            rec[f"g{i}"] = g.copy()
    rec["stride"] = np.int64(stride)
    for i in changes:
        rec[f"p{i}"] = ps[i].detach().float().numpy()
    return rec


def main():
    m = make_module().train()
    base = [p.detach().float().numpy().copy() for p in params_of(m)]
    fwd = np.load(os.path.join(HERE, "gs_head_golden.npz"))
    assert all(np.array_equal(b, fwd[f"base_p{i}"]) for i, b in enumerate(base)), "base weights differ from the forward's"
    rng = np.random.default_rng(2027)
    out = {}
    for name, (B, H, W, changes, special, stride) in CASES.items():
        for k, v in run_case(m, base, rng, B, H, W, changes, special, stride).items():
            out[f"{name}_{k}"] = v
    path = os.path.join(HERE, "gs_head_grad_golden.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path), "bytes,", len(CASES), "cases")


if __name__ == "__main__":
    main()
