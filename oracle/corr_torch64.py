"""Independent fp64 torch restatement of the 1-D correlation block (TEST INFRASTRUCTURE ONLY).

Restates `CorrBlockFast1D` (reference core/corr.py:31-61) and the `corr_sampler` lookup (SURVEY.md Appendix B) from
their maths, in differentiable fp64 CPU torch, so that every gradient (per pyramid level and w.r.t. the feature maps)
comes from autograd rather than from a hand-written backward:

  * volume  C[b,h,x,y] = sum_d F1[b,d,h,x] F2[b,d,h,y] / sqrt(D), with sqrt(D) taken in fp32 as the reference does;
  * pyramid level l+1 = mean of adjacent pairs of level l along y, width floor(W_l / 2) (avg_pool2d([1,2]));
  * lookup  out[i] = tap(xf-r+i) (1-dx) + tap(xf-r+i+1) dx, i in [0, 2r], xf = floor(x), dx = x - xf, taps outside
    [0, W2) are 0; level l samples at x / 2^l.

`floor` is taken in fp64 and converted to int64, so coordinates far past 2^31 (where a 32-bit `(int)floorf` saturates)
are well defined: their window lies wholly outside the row and the output is 0.  Callers pass the fp32 coordinate the
kernels see; `.double()` of it is exact, and so is the division by 2^l, so `dx` is the kernels' `dx`.

Tensors are created on the device of the inputs: CPU by default, the GPU where a check is too large for the CPU.

`amp=True` rounds to fp16 at the reference's op boundaries under autocast (einsum result, the division, each pooled
level): the pyramid the reference holds when it is handed fp16 feature maps.  The rounding is straight-through (the
gradient is the fp64 derivative of the unrounded op), so gradients are the same with and without it.
Pinned by tests/test_corr_torch64_cpu.py against tests/golden/corr_golden.npz."""
import torch

F64 = torch.float64


def _fp16(t):
    """Round to fp16 in the value, identity in the gradient."""
    return t + (t.detach().to(torch.float16).to(F64) - t.detach())


def sqrt_d(D):
    """torch.sqrt(torch.tensor(D).float()): the reference's divisor, an fp32 value."""
    return float(torch.sqrt(torch.tensor(D, dtype=torch.float32)))


def volume(f1, f2, amp=False):
    """f1 [B,D,H,W1], f2 [B,D,H,W2] -> level-0 volume [B,H,W1,W2] (fp64)."""
    c = torch.einsum("bdhx,bdhy->bhxy", f1.to(F64), f2.to(F64))
    div = sqrt_d(f1.shape[1])
    if amp:
        return _fp16(_fp16(c) / div)
    return c / div


def pool(v, amp=False):
    """avg_pool2d([1,2], stride [1,2]) along the last axis: [..., W] -> [..., W // 2]."""
    n = v.shape[-1] // 2
    p = 0.5 * (v[..., 0:2 * n:2] + v[..., 1:2 * n:2])
    return _fp16(p) if amp else p


def pyramid(f1, f2, levels=4, amp=False):
    """[volume, pool(volume), ...]: `levels` tensors [B,H,W1,W2 >> l] (floor widths, as the reference's views)."""
    lv = [volume(f1, f2, amp)]
    for _ in range(levels - 1):
        lv.append(pool(lv[-1], amp))
    return lv


def sample(vol, x, r):
    """corr_sampler.forward: vol [B,H,W1,W2], x [B,H,W1] (level coordinates) -> [B,2r+1,H,W1] (fp64).

    A non-finite x gives a non-finite output row (dx is NaN); its taps are read from a clamped index."""
    vol = vol.to(F64)
    B, H, W1, W2 = vol.shape
    x = x.to(F64)
    fl = torch.floor(x)
    dx = (x - fl).unsqueeze(-1)                                           # exact: x and floor(x) share a binade
    xf = torch.nan_to_num(fl, nan=0.0).clamp(-2.0 ** 62, 2.0 ** 62).to(torch.int64)
    k = xf.unsqueeze(-1) - r + torch.arange(2 * r + 2, dtype=torch.int64, device=vol.device)  # taps xf-r .. xf+r+1, [B,H,W1,2r+2]
    inside = (k >= 0) & (k < W2)
    if W2 == 0:
        taps = torch.zeros(k.shape, dtype=F64, device=vol.device) + 0.0 * vol.sum()
    else:
        taps = torch.where(inside, torch.gather(vol, 3, k.clamp(0, W2 - 1)), torch.zeros((), dtype=F64))
    out = taps[..., :-1] * (1.0 - dx) + taps[..., 1:] * dx
    return out.permute(0, 3, 1, 2)


def lookup(levels, coords_x, r):
    """CorrBlockFast1D.__call__: levels [B,H,W1,W2>>l], coords_x [B,H,W1] (or [B,1,H,W1] / [B,2,H,W1], x channel used)
    -> [B, len(levels)*(2r+1), H, W1]."""
    c = coords_x.to(F64)
    if c.dim() == 4:
        c = c[:, 0]
    return torch.cat([sample(v, c / 2 ** l, r) for l, v in enumerate(levels)], 1)


def level_grads(shapes, coords_x, r, grad_out):
    """d<lookup(levels, coords_x, r), grad_out>/d level, by autograd: one fp64 tensor per shape in `shapes`."""
    lv = [torch.zeros(s, dtype=F64, device=grad_out.device, requires_grad=True) for s in shapes]
    out = lookup(lv, coords_x, r)
    return list(torch.autograd.grad(out, lv, grad_out.to(F64), allow_unused=True))


def fold(grads, W2):
    """Level-0 gradient [B,H,W1,W2] from per-level gradients `grads` (None for a level without one): element j of level
    l is the mean of level-0 elements j 2^l .. j 2^l + 2^l - 1."""
    g = None
    for l, gl in enumerate(grads):
        if gl is None:
            continue
        if g is None:
            g = torch.zeros(tuple(gl.shape[:3]) + (W2,), dtype=F64, device=gl.device)
        n = gl.shape[-1]
        g[..., :n << l] += (gl.to(F64) / 2 ** l).repeat_interleave(1 << l, dim=-1)
    return g


def fmap_grads_from_levels(f1, f2, grads):
    """Closed form of d/dfmap given per-level gradients: G = fold(grads), dF1 = sum_y G F2 / sqrt(D) and
    dF2 = sum_x G F1 / sqrt(D)."""
    f1, f2 = f1.to(F64), f2.to(F64)
    g = fold(grads, f2.shape[3])
    div = sqrt_d(f1.shape[1])
    return (torch.einsum("bhxy,bdhy->bdhx", g, f2) / div, torch.einsum("bhxy,bdhx->bdhy", g, f1) / div)
