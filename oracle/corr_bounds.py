"""Per-element bounds for the correlation block against the fp64 restatement (TEST INFRASTRUCTURE ONLY).

Every check takes the inputs the device actually saw and evaluates the restatement (oracle/corr_torch64.py) in fp64 on
the device of its inputs.  Notation: u = 2^-24 (half an fp32 ulp at 1), div = sqrt_d(D) (the reference's fp32 sqrt(D)),
S = the exact contraction (fp64: a product of two fp32 values is exact in it, and D products sum to within D 2^-53 of S,
which the factor (1 + 2^-20) on every accumulation bound below covers).

Level 0 as an interval
----------------------
The device computes level 0 as R(acc) with acc the fp32 accumulator of S and R the dtype's chain:
  fp32  R(t) = RN32(t / div)                          (corr.cu: round_to<float>(round_to<float>(acc) / div))
  fp16  R(t) = RN16(RN32(RN16(t) / div))              (the reference's autocast chain: einsum in fp16, division in fp16;
                                                       corr.cu's round_to<half> pair, corr_tc.cu's div_rn_fast(rh(acc)))
Every step of R is monotone, so |acc - S| <= E gives R(S - E) <= device <= R(S + E).  Where both ends round to the same
value the device must equal it bit for bit.  div_rn_fast (reciprocal plus one Markstein correction) returns the correctly
rounded quotient for these operands, so R is the same for both kernels.
  * FFMA kernels: acc is one serial chain of D fmaf's starting from 0.  A recursive dot product of n terms errs by at
    most n u sum|x_i y_i| (Jeannerod & Rump 2013, with or without FMA, barring underflow): E = D u sum_d |F1 F2|.
  * wgmma kernel: the tensor core's fp32 accumulation is not guaranteed to round to nearest; with one ulp (2u) per
    step instead of half of one, E = D 2^-23 sum_d |F1 F2|.
R is evaluated in fp64: t / div is rounded once more there, so the low end is moved down and the high end up by 2^-50
relative before the fp32 rounding, which can only widen the interval (and does so only when t / div lies within 2^-50 of
an fp32 rounding midpoint).  RN16 is taken in one step from fp64 (no detour through fp32).

Pooled levels: bit-exact
------------------------
Level l+1 is avg_pool2d([1,2]) of the device's own level l in the same dtype: (a + b) in fp32, halved, rounded to the
dtype.  The floor width drops the last column of an odd level.

Build backward
--------------
dF1 = F2 g^T / div (K = W2 terms per element) and dF2 = F1 g / div (K = W1): the same interval with
  fp32  R(t) = RN32(t / div),    fp16  R(t) = RN16(RN32(t / div)),
and E = K u sum|g F| (FFMA) or K 2^-23 sum|g F| (wgmma).

fp32 block forward
------------------
Each lookup output is an fp32 interpolation of two device level values prev, cur.  With v the fp64 lookup of the fp64
pyramid of the fp32 feature maps,
    |out - v| <= 2^-22 (|prev| + |cur|) + (1 - dx) E_l[a] + dx E_l[b],
the first term the fp32 interpolation (1 - dx, two products, one sum; see tests/test_corr_amp_gpu.py) and the second the
error of the device's level values at taps a, b:
  * E_0 = (D + 1) u A_0, A_0 = sum_d |F1| |F2| / div: D u A_0 for the accumulation, u |acc / div| <= u A_0 for the
    division (to first order; the u^2 terms are inside the factor (1 + 2^-20));
  * E_{l+1}[j] = 1/2 (E_l[2j] + E_l[2j+1]) + u 1/2 (|v_l[2j]| + |v_l[2j+1]|): the average carries the two errors, and
    its one rounding errs by u of its magnitude.

fp32 block feature-map gradients
--------------------------------
The path from the incoming gradients G_k of N lookups to dF1 in fp32:
  1. each lookup's backward writes a level-gradient element a dx + b (1 - dx) of two incoming gradients, within
     2^-22 (|a| + |b|) of its exact value (tests/test_corr_amp_gpu.py).  Not 2u of |a| dx + |b| (1 - dx): dx and 1 - dx
     are fp32 values, and for a level coordinate in (-1, 1) either can carry an absolute rounding error near u that
     no weighted magnitude bounds (dx = RN32(x + 1) for x = -2^-30 is 1, its 1 - dx is 0).  So this term is bounded
     with the unweighted fold A_lk = sum_y U_lk |F2| / div, U_lk the fold of |a| + |b|;
  2. autograd sums the N lookups' fp32 gradients of each level: N - 1 roundings, each within u of a partial sum, which
     is bounded by the unsigned level gradient;
  3. _BuildPyramid.backward folds each pooled level's gradient into the level below with one fp32 add per level (the
     halving is exact): up to levels - 1 = 3 roundings for level 0, none for a level without a gradient;
  4. the build backward accumulates K terms (K = W2 for dF1, W1 for dF2): K u sum|g F|;
  5. the division rounds once: u.
With U the level-0 gradient folded from unsigned terms (|G_k| with the weights dx, 1 - dx), A = sum_y U |F2| / div bounds
every partial sum of steps 2-5, so per element
    |dF1 - ref| <= C u A + 2^-22 A_lk,    C = (N - 1) + folds + K + 1,
and dF2 is the same with F1 and a sum over x.

Emulation
---------
`emulate_*` run the same chain in fp32 (fp16 where the device rounds to it) on the CPU, and `MUTANTS` name one defect
each that a kernel or corr.py could have; tests/test_corr_bounds_cpu.py checks that the emulation passes every check
and that every mutant fails at least one.
"""
from dataclasses import dataclass, field

import torch
import torch.nn.functional as F

from oracle import corr_torch64 as ct

F64 = torch.float64
U = 2.0 ** -24
E32 = 2.0 ** -22
SAFE = 1.0 + 2.0 ** -20          # covers the fp64 restatement's own rounding and second-order terms
WIDEN = 2.0 ** -50


@dataclass
class Check:
    name: str
    ok: bool
    worst: float                  # worst |got - centre| / half-width (intervals), err / bound (bounds), mismatches (exact)
    info: dict = field(default_factory=dict)

    def require(self):
        assert self.ok, f"{self.name}: worst {self.worst:.3g} {self.info}"
        return self


# ---------------------------------------------------------------------------------------------------------------------
# rounding in fp64
# ---------------------------------------------------------------------------------------------------------------------
def rn32(v):
    return v.to(torch.float32).to(F64)


def rn16(v):
    """v (fp64) rounded to the nearest fp16, ties to even, in one step (fp16 subnormals included)."""
    _, e = torch.frexp(v)
    e = torch.where(v == 0, torch.full_like(e, -100), e) - 1
    ulp = torch.exp2(e.clamp_min(-14).to(F64) - 10)
    return torch.round(v / ulp) * ulp


def _rn32_dir(q, side):
    """RN32 of the real quotient that fp64 `q` approximates to 2^-53: side -1 takes a value at or below it, +1 above."""
    return rn32(q + side * q.abs() * WIDEN) if side else rn32(q)


def chain(t, div, dtype, pre16, side=0):
    """The level-0 (pre16=True) or build-backward (pre16=False) rounding chain applied to fp64 t."""
    if dtype == torch.float32:
        return _rn32_dir(t / div, side)
    a = rn16(t) if pre16 else t
    return rn16(_rn32_dir(a / div, side))


def interval(S, M, K, div, dtype, acc_u, pre16):
    """(low, centre, high) device values for an accumulation S of K terms with sum of magnitudes M."""
    E = K * acc_u * M * SAFE
    return chain(S - E, div, dtype, pre16, -1), chain(S, div, dtype, pre16), chain(S + E, div, dtype, pre16, 1)


def check_interval(name, got, lo, mid, hi):
    got = got.detach().to(lo.device, F64)
    if got.shape != lo.shape:
        return Check(name, False, float("inf"), dict(shape=tuple(got.shape), want=tuple(lo.shape)))
    if got.numel() == 0:
        return Check(name, True, 0.0, dict(n=0, wide=0.0))
    inside = (got >= lo) & (got <= hi)
    den = torch.where(got > mid, hi - mid, mid - lo)
    ratio = torch.where(got == mid, torch.zeros_like(got), (got - mid).abs() / den)
    ratio = torch.nan_to_num(ratio, nan=float("inf"), posinf=float("inf"))
    wide = float((lo != hi).double().mean())                   # share of elements whose interval is not one value
    off = float((got != mid).double().mean())                   # share not equal to the chain applied to S
    return Check(name, bool(inside.all()), float(ratio.max()),
                 dict(n=got.numel(), outside=int((~inside).sum()), wide=wide, off=off))


def check_bound(name, got, ref, bound):
    got = got.detach().to(ref.device, F64)
    if got.shape != ref.shape:
        return Check(name, False, float("inf"), dict(shape=tuple(got.shape), want=tuple(ref.shape)))
    if got.numel() == 0:
        return Check(name, True, 0.0, dict(n=0))
    err = (got - ref).abs()
    ratio = torch.where(err == 0, torch.zeros_like(err), err / bound)
    ratio = torch.nan_to_num(ratio, nan=float("inf"), posinf=float("inf"))
    worst = float(ratio.max())
    return Check(name, worst <= 1.0, worst, dict(n=got.numel(), over=int((ratio > 1).sum())))


# ---------------------------------------------------------------------------------------------------------------------
# build forward and backward
# ---------------------------------------------------------------------------------------------------------------------
def _contract(f1, f2):
    return torch.einsum("bdhx,bdhy->bhxy", f1, f2)


def check_level0(name, got, f1, f2, dtype, wgmma=False, device=None):
    """got: the device's level 0 [B,H,W1,W2]; f1, f2 the feature maps it was built from."""
    dev = device or got.device
    a1, a2 = f1.detach().to(dev, F64), f2.detach().to(dev, F64)
    D = a1.shape[1]
    lo, mid, hi = interval(_contract(a1, a2), _contract(a1.abs(), a2.abs()), D, ct.sqrt_d(D), dtype,
                           2 * U if wgmma else U, True)
    return check_interval(name, got, lo, mid, hi)


def check_pooled(name, levels):
    """levels[l+1] == avg_pool2d(levels[l], [1,2]) bit for bit, in the levels' dtype and on their device."""
    worst, ok, info = 0, True, {}
    for l in range(len(levels) - 1):
        a, got = levels[l].detach(), levels[l + 1].detach()
        w = a.shape[-1] // 2
        if got.shape != a.shape[:-1] + (w,) or got.dtype != a.dtype:
            return Check(name, False, float("inf"), dict(level=l + 1, shape=tuple(got.shape)))
        if w == 0:
            continue
        want = F.avg_pool2d(a, (1, 2))
        it = {torch.float16: torch.int16, torch.float32: torch.int32}[a.dtype]
        bad = int((got.contiguous().view(it) != want.contiguous().view(it)).sum())
        bad += int((~torch.isfinite(got)).sum())
        worst = max(worst, bad)
        if bad:
            ok = False
            info[f"level{l + 1}"] = bad
    return Check(name, ok, float(worst), info)


def check_build_backward(name, d1, d2, f1, f2, g, dtype, wgmma=False, device=None):
    """d1, d2: the device's dF1, dF2 for the level-0 gradient g."""
    dev = device or d1.device
    a1, a2, gg = (t.detach().to(dev, F64) for t in (f1, f2, g))
    D, W1, W2 = a1.shape[1], a1.shape[3], a2.shape[3]
    div = ct.sqrt_d(D)
    acc_u = 2 * U if wgmma else U
    S1, M1 = (torch.einsum("bhxy,bdhy->bdhx", p, q) for p, q in ((gg, a2), (gg.abs(), a2.abs())))
    S2, M2 = (torch.einsum("bhxy,bdhx->bdhy", p, q) for p, q in ((gg, a1), (gg.abs(), a1.abs())))
    return (check_interval(name + " dF1", d1, *interval(S1, M1, W2, div, dtype, acc_u, False)),
            check_interval(name + " dF2", d2, *interval(S2, M2, W1, div, dtype, acc_u, False)))


# ---------------------------------------------------------------------------------------------------------------------
# the fp32 block
# ---------------------------------------------------------------------------------------------------------------------
def level_errors(f1, f2, levels):
    """fp64 pyramid of fp64 feature maps and the bounds E_l on the fp32 device levels' errors."""
    D = f1.shape[1]
    lv = ct.pyramid(f1, f2, levels)
    E = [(D + 1) * U * SAFE * _contract(f1.abs(), f2.abs()) / ct.sqrt_d(D)]
    for l in range(levels - 1):
        n = lv[l].shape[-1] // 2
        e, v = E[l], lv[l].abs()
        E.append(0.5 * SAFE * (e[..., 0:2 * n:2] + e[..., 1:2 * n:2]) + U * 0.5 * (v[..., 0:2 * n:2] + v[..., 1:2 * n:2]))
    return lv, E


def _tap_sums(levels, cx, r):
    """Per level, |prev| + |cur| of every lookup output: the lookup of |level| at floor(x / 2^l) and floor + 1."""
    out = []
    for l, v in enumerate(levels):
        fl = torch.floor(cx / 2 ** l)
        out.append(ct.sample(v.abs(), fl, r) + ct.sample(v.abs(), fl + 1, r))
    return torch.cat(out, 1)


def check_block_forward(name, out, dev_levels, lv64, E, cx, r):
    """out: one fp32 lookup [B, L(2r+1), H, W1] of the device levels `dev_levels` at level-0 x coordinates cx [B,H,W1]."""
    dev = lv64[0].device
    cx = cx.to(dev, F64)
    v = ct.lookup(lv64, cx, r)
    bound = E32 * _tap_sums([t.detach().to(dev, F64) for t in dev_levels], cx, r) + ct.lookup(E, cx, r)
    return check_bound(name, out, v, bound)


def block_grad_reference(f1, f2, coords, gs, levels, r, only_level=None, device=None):
    """fp64 autograd through the restatement and the per-element bounds on dF1, dF2 (see the module docstring).
    coords: level-0 x coordinates [B,H,W1] of each lookup; gs: each lookup's incoming gradient, or (only_level) the
    gradient of that level.  Returns ((ref1, bound1), (ref2, bound2))."""
    dev = device or f1.device
    a1 = f1.detach().to(dev, F64).requires_grad_(True)
    a2 = f2.detach().to(dev, F64).requires_grad_(True)
    D, W1, W2 = a1.shape[1], a1.shape[3], a2.shape[3]
    lv = ct.pyramid(a1, a2, levels)
    shapes = [v.shape for v in lv]
    if only_level is None:
        cs = [c.to(dev, F64) for c in coords]
        gs = [g.to(dev, F64) for g in gs]
        loss = sum((ct.lookup(lv, c, r) * g).sum() for c, g in zip(cs, gs))
        Ul = [0] * levels
        Ulk = [0] * levels
        for c, g in zip(cs, gs):
            Ul = [x + y for x, y in zip(Ul, ct.level_grads(shapes, c, r, g.abs()))]
            rd = 2 * r + 1
            for l in range(levels):                   # |a| + |b|: the backward at floor(x / 2^l) and floor + 1
                leaf = torch.zeros(shapes[l], dtype=F64, device=dev, requires_grad=True)
                fl = torch.floor(c / 2 ** l)
                gl = g[:, l * rd:(l + 1) * rd].abs()
                Ulk[l] = Ulk[l] + sum(torch.autograd.grad(ct.sample(leaf, x, r), leaf, gl)[0] for x in (fl, fl + 1))
        n_sum, folds = len(cs) - 1, levels - 1
    else:
        g = gs[0].to(dev, F64)
        loss = (lv[only_level] * g).sum()
        Ul = [g.abs() if l == only_level else None for l in range(levels)]
        Ulk = None
        n_sum, folds = 0, 0
    d1, d2 = torch.autograd.grad(loss, (a1, a2))
    div = ct.sqrt_d(D)
    b1, b2 = a1.detach().abs(), a2.detach().abs()
    Ug = ct.fold(Ul, W2)
    A1 = torch.einsum("bhxy,bdhy->bdhx", Ug, b2) / div
    A2 = torch.einsum("bhxy,bdhx->bdhy", Ug, b1) / div
    bound1 = (n_sum + folds + W2 + 1) * U * SAFE * A1
    bound2 = (n_sum + folds + W1 + 1) * U * SAFE * A2
    if Ulk is not None:
        Gk = ct.fold(Ulk, W2)
        bound1 = bound1 + E32 * SAFE * torch.einsum("bhxy,bdhy->bdhx", Gk, b2) / div
        bound2 = bound2 + E32 * SAFE * torch.einsum("bhxy,bdhx->bdhy", Gk, b1) / div
    return (d1, bound1), (d2, bound2)


# ---------------------------------------------------------------------------------------------------------------------
# CPU emulation of the chain, and its mutants
# ---------------------------------------------------------------------------------------------------------------------
MUTANTS = {
    "pool_unrounded": "fp16: a pooled level averaged from the previous level before its rounding to fp16",
    "pool_shifted": "pooling pairs shifted by one column: (2j+1, 2j+2)",
    "pool_odd_tail": "an odd level's trailing column kept: ceil width, the last pair padded with 0",
    "level0_once16": "fp16: level 0 rounded once, RN16(acc / div), instead of the reference's two roundings",
    "fold_no_half": "the fold adds a pooled level's gradient without its 1/2",
    "fold_half_twice": "the fold applies 1/2 twice to the gradient of level 2 and above",
    "drop_lookup": "one lookup's level gradients dropped from the sum",
    "dx_swapped": "dx and 1 - dx swapped in the lookup backward",
    "g_transposed": "dF1 contracts g^T instead of g (seen where W1 == W2)",
    "no_div": "the build backward without its 1 / sqrt(D)",
}


def _r(v, dtype):
    return v.to(dtype).float()


def emulate_pyramid(f1, f2, levels, dtype, mutant=None):
    """fp32/fp16 feature maps (CPU) -> the FFMA kernel's levels, in `dtype`."""
    f1, f2 = f1.float(), f2.float()
    D = f1.shape[1]
    div = torch.tensor(D, dtype=torch.float32).sqrt()
    acc = torch.zeros(f1.shape[0], f1.shape[2], f1.shape[3], f2.shape[3])
    for d in range(D):                                           # one fp32 chain per output, in d order
        acc = acc + f1[:, d, :, :, None] * f2[:, d, :, None, :]
    once = dtype == torch.float32 or mutant == "level0_once16"
    unrounded = (acc if once else _r(acc, dtype)) / div         # the fp32 value before the rounding to dtype
    lv = [_r(unrounded, dtype)]
    for _ in range(levels - 1):
        src = unrounded if mutant == "pool_unrounded" else lv[-1]
        w = src.shape[-1]
        if mutant == "pool_shifted":
            n = (w - 1) // 2
            p = (src[..., 1:2 * n + 1:2] + src[..., 2:2 * n + 2:2]) * 0.5
            p = torch.cat([p, torch.zeros(p.shape[:-1] + (w // 2 - n,))], -1)
        elif mutant == "pool_odd_tail" and w % 2:
            s = torch.cat([src, torch.zeros(src.shape[:-1] + (1,))], -1)
            p = (s[..., 0::2] + s[..., 1::2]) * 0.5
        else:
            n = w // 2
            p = (src[..., 0:2 * n:2] + src[..., 1:2 * n:2]) * 0.5
        unrounded = p
        lv.append(_r(p, dtype))
    return [_r(v, dtype).to(dtype) for v in lv]


def emulate_build_backward(f1, f2, g, dtype, mutant=None):
    """The FFMA build backward: dF1 = F2 g^T / div, dF2 = F1 g / div, fp32 accumulation in K order, rounded to dtype."""
    f1, f2, g = f1.float(), f2.float(), g.float()
    D, W1, W2 = f1.shape[1], f1.shape[3], f2.shape[3]
    div = torch.tensor(D, dtype=torch.float32).sqrt()
    g1 = g.transpose(2, 3) if mutant == "g_transposed" else g
    d1 = torch.zeros(f1.shape)
    for y in range(W2):
        d1 = d1 + g1[:, None, :, :, y] * f2[:, :, :, y, None]
    d2 = torch.zeros(f2.shape)
    for x in range(W1):
        d2 = d2 + g[:, None, :, x, :] * f1[:, :, :, x, None]
    if mutant != "no_div":
        d1, d2 = d1 / div, d2 / div
    return d1.to(dtype), d2.to(dtype)


def _lookup_fwd(v, x, r):
    """fp32 lookup of one level at level coordinates x [B,H,W1] (corr_lookup_fwd_kernel)."""
    W2 = v.shape[-1]
    fl = torch.floor(x)
    dx = (x - fl).unsqueeze(-1)
    k = fl.long().unsqueeze(-1) - r + torch.arange(2 * r + 2)
    taps = torch.where((k >= 0) & (k < W2), torch.gather(v, 3, k.clamp(0, max(W2 - 1, 0))) if W2 else
                       torch.zeros(k.shape), torch.zeros(()))
    return (taps[..., :-1] * (1.0 - dx) + taps[..., 1:] * dx).permute(0, 3, 1, 2)


def _lookup_bwd(shape, x, r, go, mutant=None):
    """fp32 lookup backward of one level (corr_lookup_bwd_kernel): tap i gets go[i-1] dx + go[i] (1 - dx)."""
    W2 = shape[-1]
    fl = torch.floor(x)
    dx = (x - fl).unsqueeze(-1)
    om = 1.0 - dx
    if mutant == "dx_swapped":
        dx, om = om, dx
    go = go.permute(0, 2, 3, 1)                                 # [B,H,W1,rd]
    z = torch.zeros(go.shape[:-1] + (1,))
    t = torch.cat([z, go], -1) * dx + torch.cat([go, z], -1) * om    # taps 0 .. rd, each one product pair, one sum
    k = fl.long().unsqueeze(-1) - r + torch.arange(2 * r + 2)
    inside = (k >= 0) & (k < W2)
    gv = torch.zeros(shape)
    if W2:                                                       # a row's taps are distinct: each element gets one term
        gv.scatter_add_(3, torch.where(inside, k, torch.zeros_like(k)), torch.where(inside, t, torch.zeros(())))
    return gv


def emulate_block(f1, f2, coords, gs, levels, r, mutant=None, only_level=None):
    """fp32 block: pyramid, lookups at level-0 x coordinates `coords` (list of [B,H,W1]), their backward for incoming
    gradients `gs`, autograd's sum, the fold of _BuildPyramid.backward and the build backward.  Returns
    (levels, outs, dF1, dF2)."""
    lv = emulate_pyramid(f1, f2, levels, torch.float32, mutant)
    rd = 2 * r + 1
    outs = [torch.cat([_lookup_fwd(v, c / 2 ** l, r) for l, v in enumerate(lv)], 1) for c in coords]
    if only_level is None:
        grads = [None] * levels
        ks = range(len(coords) - 1) if mutant == "drop_lookup" else range(len(coords))
        for k in ks:
            for l, v in enumerate(lv):
                gl = _lookup_bwd(v.shape, coords[k] / 2 ** l, r, gs[k][:, l * rd:(l + 1) * rd], mutant)
                grads[l] = gl if grads[l] is None else grads[l] + gl
    else:
        grads = [gs[0].float() if l == only_level else None for l in range(levels)]
    g = None
    for l in range(levels - 1, -1, -1):                          # _BuildPyramid.backward's fold
        gl = grads[l]
        if g is not None:
            h = 1.0 if mutant == "fold_no_half" else (0.25 if mutant == "fold_half_twice" and l + 1 >= 2 else 0.5)
            up = torch.zeros(lv[l].shape)
            n = min(2 * g.shape[-1], up.shape[-1])               # < 2 g.shape[-1] only for pool_odd_tail
            up[..., :n] = (h * g).repeat_interleave(2, dim=-1)[..., :n]
            g = up if gl is None else gl + up
        else:
            g = gl
    d1, d2 = emulate_build_backward(f1, f2, g, torch.float32, mutant)
    return lv, outs, d1, d2
