"""Cases of the regressor-tail backward tests: the golden cases (tests/golden/gs_head_grad_golden.npz, the reference's
own module's autograd in fp64) and seeded upstream gradients for the forward's cases (gs_head_cases)."""
import os

import numpy as np
import torch

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "gs_head_grad_golden.npz")
BASE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "gs_head_golden.npz")     # shared base weights
GOLDEN_CASES = ("default", "rot_zero", "saturate", "clamp", "nonsquare", "nan_depth", "inf_g_scale")
GRAD_KEYS = ("d_src", "d_depth", "out_w", "out_b", "rot_w1", "rot_b1", "rot_w2", "rot_b2", "scale_w1", "scale_b1",
             "scale_w2", "scale_b2", "opacity_w1", "opacity_b1", "opacity_w2", "opacity_b2")
SAMPLED = ("out_w", "rot_w1", "scale_w1", "opacity_w1")     # stored as every `stride`-th element, with a finiteness mask


def golden(name):
    """(src, img, depth, params, grads, want, finite, stride) of a golden case: grads = (g_rot, g_scale, g_opacity) fp32;
    want = dict(GRAD_KEYS) in fp64, whole tensors except SAMPLED ones, which hold `pick(k, full, stride)`; finite =
    the isfinite mask of every whole gradient."""
    z, base = np.load(GOLDEN), np.load(BASE)
    ps = [torch.from_numpy(z[f"{name}_p{i}"] if f"{name}_p{i}" in z.files else base[f"base_p{i}"]) for i in range(14)]
    src, img, depth = (torch.from_numpy(z[f"{name}_{k}"]) for k in ("src", "img", "depth"))
    grads = [torch.from_numpy(z[f"{name}_{k}"]) for k in ("g_rot", "g_scale", "g_opacity")]
    want = dict(d_src=torch.from_numpy(z[f"{name}_d_src"]), d_depth=torch.from_numpy(z[f"{name}_d_depth"]))
    finite = {}
    for i, k in enumerate(GRAD_KEYS[2:]):
        want[k] = torch.from_numpy(z[f"{name}_g{i}"])
        if k in SAMPLED:
            n = ps[i].numel()
            finite[k] = torch.from_numpy(np.unpackbits(z[f"{name}_finite{i}"])[:n].astype(bool)).view(ps[i].shape)
        else:
            finite[k] = torch.isfinite(want[k])
    finite["d_src"], finite["d_depth"] = torch.isfinite(want["d_src"]), torch.isfinite(want["d_depth"])
    return src, img, depth, ps, grads, want, finite, int(z[f"{name}_stride"])


def pick(k, t, stride):
    """The elements of gradient `k` that the golden stores: every `stride`-th of the flattened tensor for SAMPLED keys."""
    return t.reshape(-1)[::stride] if k in SAMPLED else t


def upstream(B, H, W, seed):
    """Seeded upstream gradients (g_rot [B,4,H,W], g_scale [B,3,H,W], g_opacity [B,1,H,W]), fp32 CPU."""
    g = torch.Generator().manual_seed(5000 + seed)
    return [torch.randn(B, c, H, W, generator=g) for c in (4, 3, 1)]
