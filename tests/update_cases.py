"""Closed-form update-block parameters and inputs, shared by tests/golden/make_update_golden.py and the update tests.

Every value is a small integer over a power of two, so it is exact in fp16, fp32 and fp64 alike and the golden file
stores only outputs: the 1.4 M parameters are rebuilt here from (seed, tensor index)."""
import torch

F64 = torch.float64
HID = 96
PARAM_SHAPES = ((64, 36, 1, 1), (64,), (64, 64, 3, 3), (64,), (64, 2, 7, 7), (64,), (64, 64, 3, 3), (64,),
                (126, 128, 3, 3), (126,), (96, 224, 3, 3), (96,), (96, 224, 3, 3), (96,), (96, 224, 3, 3), (96,),
                (256, 96, 3, 3), (256,), (2, 256, 3, 3), (2,), (256, 96, 3, 3), (256,), (576, 256, 1, 1), (576,))
# single-iteration cases (B, H, W) and the loop case (B, H, W, iters)
STEP_CASES = ((1, 1, 1), (2, 3, 5), (1, 9, 7), (2, 9, 7))
LOOP_CASE = (1, 6, 20, 3)
FMAP_D = 32


def _pattern(n, seed, mod=255):
    """n integers in [-(mod // 2), mod // 2], a fixed hash of (index, seed)."""
    i = torch.arange(n, dtype=torch.int64)
    return ((i * 7919 + seed * 104729 + (i * i) % 977) % mod - mod // 2).to(F64)


def params(seed=0):
    """The 24 parameters in update.params_of order, fp64: weights of magnitude ~ 1 / sqrt(fan-in), biases ~ 0.1, all
    multiples of 2^-12."""
    out = []
    for k, s in enumerate(PARAM_SHAPES):
        n = 1
        for d in s:
            n *= d
        v = _pattern(n, seed * 31 + k)
        if len(s) == 4:
            fan = s[1] * s[2] * s[3]
            scale = 2.0 ** -round(torch.log2(torch.tensor(127.0 * fan ** 0.5)).item())
        else:
            scale = 2.0 ** -10
        out.append((v * scale).view(s))
    return out


def inputs(B, H, W, seed=1):
    """dict(corr [B,36,H,W], coords1 [B,2,H,W], net [B,96,H,W], czrq [B,288,H,W]), fp64, fp16-exact except coords1's
    sub-ulp fractions (which the fp16 flow rounding must drop)."""
    corr = _pattern(B * 36 * H * W, seed, 61).view(B, 36, H, W) * 2.0 ** -4
    net = _pattern(B * HID * H * W, seed + 1, 255).view(B, HID, H, W) * 2.0 ** -7
    czrq = _pattern(B * 3 * HID * H * W, seed + 2, 255).view(B, 3 * HID, H, W) * 2.0 ** -7
    ys, xs = torch.meshgrid(torch.arange(H, dtype=F64), torch.arange(W, dtype=F64), indexing="ij")
    g = torch.stack([xs, ys])[None].repeat(B, 1, 1, 1)
    coords1 = g + _pattern(B * 2 * H * W, seed + 3, 101).view(B, 2, H, W) * (2.0 ** -5 + 2.0 ** -19)
    return dict(corr=corr, coords1=coords1, net=net, czrq=czrq)


def fmaps(B, H, W, seed=2):
    """fmap1, fmap2 [B,32,H,W] of the loop case, multiples of 2^-6."""
    f1 = _pattern(B * FMAP_D * H * W, seed, 63).view(B, FMAP_D, H, W) * 2.0 ** -6
    f2 = _pattern(B * FMAP_D * H * W, seed + 5, 63).view(B, FMAP_D, H, W) * 2.0 ** -6
    return f1, f2
