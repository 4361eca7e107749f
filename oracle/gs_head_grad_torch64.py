"""fp64 autograd, fp32 emulation and per-element error bounds for the backward of the Gaussian-parameter regressor's
full-resolution tail (csrc/gs_head.cu, gpsg_gs_head_backward) -- TEST INFRASTRUCTURE ONLY.  The forward maths, its
emulation and the helpers (upsample2, conv, tf32, hulp, gamma, ratio) are oracle/gs_head_torch64.py's.

`backward64` is fp64 autograd through the same maths with torch's own activation
functions (F.relu, F.softplus, torch.clamp_max, F.normalize, torch.sigmoid, as the reference module calls them), so
masks and branches on NaN, inf and ties are torch's.  With `mid` given (the kernels' intermediate, NCHW) it is forced:
the heads read it and the out_conv ReLU's mask is taken from it, as the backward kernels do.  `emulate_backward` runs
the kernels' backward arithmetic in fp32 on TF32 operands with sums in a random order, the pixel sums of dW2 and of
the biases' gradients in fp64 as the kernels carry them (GRAD_MUTANTS inject errors).
`grad_bounds` bounds |kernel - backward64(mid)| per element, with Dw = hulp(w) and the reduction depth D of the
parameter-gradient sums (`reduction_depth`: 16 + 128 T + n for n CTAs of T tiles of 2 x 64 pixels each):
  h, pre   recomputed from mid as in the forward bounds (TF32 weights, mid already TF32), + the TF32 rounding of h;
  dpre     sigmoid: |g| (0.1 e_pre + 16u) (|d/dx y(1 - y)| < 0.1); softplus: |g| (25 e_pre + 32u) where the threshold
           (100 x vs 20) and the clamp (softplus vs 0.01, within the forward's softplus bound) are decided, 2 |g| where
           either is undecided, 0 where decidedly clamped; normalize: 3 |g| E / (n - E)^2 + 32u |g| / (n - E) where the
           eps branch is decided unclamped, |g| |1/eps32 - 1/eps| + 4u |g| / eps32 where decidedly clamped, inf else;
  dh       W2^T dpre with TF32 W2 (depth 5) and the ReLU mask; |v| + e where |z| <= e_z (undecided), + TF32 rounding;
  dmid     conv3x3^T of dh (depth 9 x 96) under mid's mask, + TF32 rounding;  dcat  conv3x3^T of dmid (depth 9 x 32);
  d_src    the upsample's adjoint of the dcat bound + gamma(52) of the magnitudes;  d_depth  dcat's channel 51;
           `src_stage` also checks d_src against the fp64 adjoint of the kernels' own dcat, gamma(52) of the magnitudes;
  weights  the weight gradient of the magnitude fields: sum (|G| Dx + DG |X| + DG Dx) + gamma(2 (D + 1)) sum (|G| +
           DG)(|X| + Dx) for G in (dpre, dh, dmid), X in (h, mid, cat), D the reduction depth.
"""
import math

import numpy as np
import torch
import torch.nn.functional as F

from oracle.gs_head_torch64 import (F64, U, _conv32, _heads, _pad, conv, emulate, gamma, hulp, ratio, relu, tf32,  # noqa: F401
                                    upsample2)

PARAM_NAMES = ("out_w", "out_b", "rot_w1", "rot_b1", "rot_w2", "rot_b2", "scale_w1", "scale_b1", "scale_w2", "scale_b2",
               "opacity_w1", "opacity_b1", "opacity_w2", "opacity_b2")
GRAD_KEYS = ("d_src", "d_depth") + PARAM_NAMES
GRAD_MUTANTS = ("tap_not_flipped", "upsample_adjoint_align_corners", "mid_mask_from_dmid", "partial_dropped",
                "softplus_no_threshold", "sigmoid_from_pre")
EPS32 = float(np.float32(1e-12))


class _ForcedMid(torch.autograd.Function):
    """Value `mid`; gradient to z masked by mid as the ReLU's threshold_backward on its result."""

    @staticmethod
    def forward(ctx, z, mid):
        ctx.save_for_backward(mid)
        return mid.clone()

    @staticmethod
    def backward(ctx, g):
        mid, = ctx.saved_tensors
        return torch.where(mid <= 0, torch.zeros_like(g), g), None


def _grads_of(grads, b):
    return [g[b:b + 1].to(F64) for g in grads]


def backward64(src, img, depth, params, grads, mid=None):
    """fp64 autograd of the tail: dict(d_src, d_depth, out_w, ..., opacity_b2) for upstream gradients grads = (g_rot,
    g_scale, g_opacity); `mid` [B,32,H,W] forces the intermediate (see the module docstring).  One batch element at a
    time, the parameter gradients summed in fp64."""
    ps = [p.detach().to(F64).requires_grad_() for p in params]
    d_src, d_depth = [], []
    for b in range(src.shape[0]):
        s = src[b:b + 1].detach().to(F64).requires_grad_()
        d = depth[b:b + 1].detach().to(F64).requires_grad_()
        x = torch.cat([upsample2(s), img[b:b + 1].to(F64), d], 1)
        z = conv(x, ps[0], ps[1])
        m = F.relu(z) if mid is None else _ForcedMid.apply(z, mid[b:b + 1].to(F64))
        pre = [conv(F.relu(conv(m, w1, b1)), w2, b2) for w1, b1, w2, b2 in _heads(ps)]
        outs = (F.normalize(pre[0], dim=1), torch.clamp_max(F.softplus(pre[1], beta=100, threshold=20), 0.01),
                torch.sigmoid(pre[2]))
        torch.autograd.backward(outs, _grads_of(grads, b))
        d_src.append(s.grad)
        d_depth.append(d.grad)
    out = dict(d_src=torch.cat(d_src), d_depth=torch.cat(d_depth))
    out.update({n: p.grad for n, p in zip(PARAM_NAMES, ps)})
    return out


def _up_adjoint(g, h, w):
    """The adjoint of upsample2 from [B,C,2h,2w] to [B,C,h,w] in g's dtype (every weight multiplied in)."""
    with torch.enable_grad():
        x = torch.zeros(g.shape[0], g.shape[1], h, w, dtype=g.dtype, device=g.device, requires_grad=True)
        upsample2(x).backward(g)
    return x.grad


def _flipT(w):
    return w.transpose(0, 1).flip(2, 3)


def _wsum32(G, X, k, gen, drop=0, acc_dtype=torch.float32):
    """sum over pixels of G [B,N,H,W] x im2col_k(X) [B,C k k,H W] of fp32 products, pixels in a random order, in
    `acc_dtype` -> fp32 [N, C k k]; `drop` leaves out that many pixels (a lost partial)."""
    B, N = G.shape[:2]
    cols = F.unfold(_pad(X, k), k)                                      # [B, C k k, HW]
    g = G.reshape(B, N, -1)
    acc = torch.zeros(N, cols.shape[1], dtype=acc_dtype)
    order = torch.randperm(B * g.shape[2], generator=gen).tolist()
    for i in order[:len(order) - drop]:
        bb, p = divmod(i, g.shape[2])
        acc = acc + (g[bb, :, p, None] * cols[bb, None, :, p]).to(acc_dtype)
    return acc.to(torch.float32)


def _sum64(G, gen):
    """sum over pixels of fp32 G [B,N,H,W] in fp64, pixels in a random order -> fp32 [N] (the kernels' bias sums)."""
    g = G.permute(1, 0, 2, 3).reshape(G.shape[1], -1).to(F64)
    acc = torch.zeros(G.shape[1], dtype=F64)
    for p in torch.randperm(g.shape[1], generator=gen).tolist():
        acc = acc + g[:, p]
    return acc.to(torch.float32)


def emulate_backward(src, img, depth, params, grads, seed=0, mutant=None):
    """The backward kernels' arithmetic on the CPU in fp32 (TF32 operands, random summation orders), on the forward
    emulation's own intermediate: dict(GRAD_KEYS..., mid, dcat) with mid the TF32 intermediate it used and dcat
    [B,52,H,W] the transposed out_conv's result that d_src and d_depth come from."""
    assert mutant is None or mutant in GRAD_MUTANTS, mutant
    src, img, depth = (t.to(torch.float32).cpu() for t in (src, img, depth))
    ps = [p.to(torch.float32).cpu() for p in params]
    gr = [g.to(torch.float32).cpu() for g in grads]
    m = tf32(emulate(src, img, depth, ps, seed=seed)["mid"])
    gen = torch.Generator().manual_seed(seed + 1)
    hs, pre = [], []
    for w1, b1, w2, b2 in _heads(ps):
        h = tf32(relu(_conv32(m, w1, b1, gen)))
        hs.append(h)
        pre.append(_conv32(h, w2, b2, gen))
    p, g = pre[0], gr[0]
    n = p.pow(2).sum(1, keepdim=True).sqrt()
    d = torch.where(n < EPS32, torch.full_like(n, EPS32), n)
    coef = torch.where(n >= EPS32, (-(g * p).sum(1, keepdim=True) / (d * d)) / n, torch.zeros_like(n))
    dp0 = g / d + p * coef
    v, g = pre[1], gr[1]
    z = v * 100
    sp = torch.where(z > 20, v, torch.log1p(torch.exp(z)) / 100)
    ds = torch.where(sp <= np.float32(0.01).item(), g, torch.zeros_like(g))
    ez = torch.exp(z)
    dp1 = ds * ez / (ez + 1) if mutant == "softplus_no_threshold" else torch.where(z > 20, ds, ds * ez / (ez + 1))
    y = pre[2] if mutant == "sigmoid_from_pre" else 1 / (1 + torch.exp(-pre[2]))
    dp2 = gr[2] * (1 - y) * y
    dps = (dp0, dp1, dp2)
    dh = []
    for (w1, b1, w2, b2), h, dp in zip(_heads(ps), hs, dps):
        w2r = tf32(w2).reshape(w2.shape[0], -1)
        acc = torch.zeros_like(h)
        for o in range(w2r.shape[0]):
            acc = acc + w2r[o].view(1, -1, 1, 1) * dp[:, o:o + 1]
        dh.append(tf32(torch.where(h <= 0, torch.zeros_like(acc), acc)))
    dh = torch.cat(dh, 1)
    w1all = torch.cat([w1 for w1, _, _, _ in _heads(ps)], 0)                 # [96, 32, 3, 3]
    wt = w1all.transpose(0, 1) if mutant == "tap_not_flipped" else _flipT(w1all)
    r = _conv32(dh, wt, torch.zeros(32), gen)
    dmid = tf32(torch.where((r if mutant == "mid_mask_from_dmid" else m) <= 0, torch.zeros_like(r), r))
    dcat = _conv32(dmid, _flipT(ps[0]), torch.zeros(52), gen)
    H, W = img.shape[-2:]
    dsrc_in = dcat[:, :48]
    if mutant == "upsample_adjoint_align_corners":
        with torch.enable_grad():
            x = torch.zeros(dcat.shape[0], 48, H // 2, W // 2, requires_grad=True)
            upsample2(x, align_corners=True).backward(dsrc_in)
        d_src = x.grad
    else:
        d_src = _up_adjoint(dsrc_in, H // 2, W // 2)
    out = dict(d_src=d_src, d_depth=dcat[:, 51:52], mid=m, dcat=dcat)
    dw1 = _wsum32(dh, m, 3, gen, drop=64 if mutant == "partial_dropped" else 0).view(96, 32, 3, 3)
    db1 = _sum64(dh, gen)
    cat = tf32(torch.cat([upsample2(src), img, depth], 1))
    out["out_w"] = _wsum32(dmid, cat, 3, gen).view(32, 52, 3, 3)
    out["out_b"] = _sum64(dmid, gen)
    for k, (name, dp, h) in enumerate(zip(("rot", "scale", "opacity"), dps, hs)):
        out[name + "_w1"] = dw1[32 * k:32 * k + 32]
        out[name + "_b1"] = db1[32 * k:32 * k + 32]
        out[name + "_w2"] = _wsum32(dp, h, 1, gen, acc_dtype=F64).view(dp.shape[1], 32, 1, 1)
        out[name + "_b2"] = _sum64(dp, gen)
    return out


def src_stage(dcat):
    """(want, bound) of d_src given the kernels' own dcat [B,>=48,H,W]: the upsample's adjoint in fp64 and the error of
    the kernels' gather, at most 25 products of exact dyadic weights summed in fp32, gamma(52) of the magnitudes.  This
    checks the last stage alone; the end-to-end bound of `grad_bounds` carries the TF32 error of the whole chain, which
    is as large as a wrong interpolation weight would be."""
    H, W = dcat.shape[-2:]
    d = dcat[:, :48].to(F64)
    want = _up_adjoint(d, H // 2, W // 2)
    return want, torch.nan_to_num(gamma(52) * _up_adjoint(d.abs(), H // 2, W // 2), nan=float("inf"))


def reduction_depth(B, H, W, ctas=132):
    """Longest chain of fp32 additions a parameter-gradient element goes through in the backward kernels."""
    tiles = B * math.ceil(H / 2) * math.ceil(W / 64)
    n = max(min(tiles, ctas), 1)
    return 16 + 128 * math.ceil(tiles / n) + n


def _cv(x, w, transpose=False):
    p = (w.shape[-1] - 1) // 2
    return F.conv_transpose2d(x, w, padding=p) if transpose else F.conv2d(x, w, padding=p)


def _gemm_err(a, da, w, n, transpose=False, b=None):
    """|kernel - exact| of conv(a, w) (+ b) with TF32 weights when the kernel's operand is within da of a (already TF32)."""
    aa, wa, dw = a.abs(), w.abs(), hulp(w)
    prod = _cv(da, wa, transpose) + _cv(aa + da, dw, transpose)
    tot = _cv(aa, wa, transpose) + prod
    if b is not None:
        tot = tot + b.abs().view(1, -1, 1, 1)
    return prod + gamma(2 * (n + 1)) * tot


def _wgrad(x, g, shape):
    return torch.nn.grad.conv2d_weight(x, shape, g, padding=(shape[-1] - 1) // 2)


def grad_bounds(src, img, depth, params, grads, mid, ctas=132):
    """Per-element bounds dict(GRAD_KEYS...) on the backward kernels' results against backward64(..., mid=mid), fp64 on
    the inputs' device; `mid` is the kernels' intermediate [B,32,H,W], `ctas` the SM count of the device."""
    B, _, H, W = img.shape
    gw = gamma(2 * (reduction_depth(B, H, W, ctas) + 1))
    ps = [p.detach().to(F64) for p in params]
    heads = _heads(ps)
    w1all = torch.cat([h[0] for h in heads], 0)
    acc = {}

    def add(k, v):
        acc[k] = acc[k] + v if k in acc else v

    d_src, d_depth = [], []
    with torch.no_grad(), torch.backends.cudnn.flags(enabled=False):
        for b in range(B):
            m = mid[b:b + 1].to(F64)
            g = _grads_of(grads, b)
            hs, Ehs, zs, ezs, pre, epre = [], [], [], [], [], []
            for w1, b1, w2, b2 in heads:
                z = _cv(m, w1) + b1.view(1, -1, 1, 1)
                ez = _gemm_err(m, torch.zeros_like(m), w1, 9 * 32, b=b1)
                h = relu(z)
                Eh = ez + hulp(h.abs() + ez)
                zs.append(z), ezs.append(ez), hs.append(h), Ehs.append(Eh)
                pre.append(_cv(h, w2) + b2.view(1, -1, 1, 1))
                epre.append(_gemm_err(h, Eh, w2, 33, b=b2))
            # dpre
            p, E0, gr = pre[0], epre[0], g[0]
            n = p.pow(2).sum(1, keepdim=True).sqrt()
            E = E0.pow(2).sum(1, keepdim=True).sqrt()
            gn = gr.pow(2).sum(1, keepdim=True).sqrt()
            dd = torch.where(n < 1e-12, torch.full_like(n, 1e-12), n)
            dp0 = gr / dd + p * torch.where(n >= 1e-12, (-(gr * p).sum(1, keepdim=True) / (dd * dd)) / n,
                                            torch.zeros_like(n))
            lo, hi = min(1e-12, EPS32), max(1e-12, EPS32)
            slack = E + 4 * U * n
            un = n - slack > hi
            cl = n + slack < lo
            e_un = 3 * gn * E / (n - E).clamp(min=1e-300) ** 2 + 32 * U * gn / (n - E).clamp(min=1e-300)
            e_cl = gr.abs() * (abs(1 / EPS32 - 1e12) + 4 * U / EPS32)
            e0 = torch.where(un, e_un.expand_as(p), torch.where(cl, e_cl, torch.full_like(p, float("inf"))))
            v, E1, gs = pre[1], epre[1], g[1]
            t = 100 * v
            sp = F.softplus(v, beta=100, threshold=20)
            dp1 = torch.where(sp <= 0.01, gs, torch.zeros_like(gs)) * torch.where(t > 20, torch.ones_like(t),
                                                                                  torch.sigmoid(t))
            e_sp = E1 + 1e-10 + U * (v.abs() + E1) + 8 * U * (sp.abs() + E1)
            und = ((sp - 0.01).abs() <= e_sp + 2.0 ** -30) | ((t - 20).abs() <= 100 * E1 + U * (t.abs() + 100 * E1))
            e1 = torch.where(und, 2 * gs.abs(),
                             torch.where(sp <= 0.01, gs.abs() * (25 * E1 + 32 * U), torch.zeros_like(gs)))
            y = torch.sigmoid(pre[2])
            dp2 = g[2] * (1 - y) * y
            e2 = g[2].abs() * (0.1 * epre[2] + 16 * U)
            dps, edps = (dp0, dp1, dp2), (e0, e1, e2)
            # dh
            dh, Edh = [], []
            for (w1, b1, w2, b2), h, z, ez, dp, edp in zip(heads, hs, zs, ezs, dps, edps):
                v = _cv(dp, w2, transpose=True)
                ev = _gemm_err(dp, edp, w2, 5, transpose=True)
                off = h <= 0
                e = torch.where((z.abs() <= ez) & ~torch.isnan(z), v.abs() + ev, torch.where(off, 0 * ev, ev))
                d = torch.where(off, torch.zeros_like(v), v)
                dh.append(d), Edh.append(e + hulp(d.abs() + e))
            dh, Edh = torch.cat(dh, 1), torch.cat(Edh, 1)
            # dmid, dcat
            r = _cv(dh, w1all, transpose=True)
            er = _gemm_err(dh, Edh, w1all, 9 * 96, transpose=True)
            on = ~(m <= 0)
            dmid = torch.where(on, r, torch.zeros_like(r))
            e = torch.where(on, er, torch.zeros_like(er))
            Edm = e + hulp(dmid.abs() + e)
            dcat = _cv(dmid, ps[0], transpose=True)
            ec = _gemm_err(dmid, Edm, ps[0], 9 * 32, transpose=True)
            d_depth.append(ec[:, 51:52])
            d_src.append(_up_adjoint(ec[:, :48], H // 2, W // 2)
                         + gamma(52) * _up_adjoint(dcat[:, :48].abs() + ec[:, :48], H // 2, W // 2))
            # parameter gradients
            for k, (name, h, Eh, dp, edp) in enumerate(zip(("rot", "scale", "opacity"), hs, Ehs, dps, edps)):
                ad, ah = dp.abs(), h.abs()
                ein = lambda x, y: torch.einsum("bohw,bchw->oc", x, y).view(x.shape[1], y.shape[1], 1, 1)
                add(name + "_w2", ein(ad, Eh) + ein(edp, ah + Eh) + gw * ein(ad + edp, ah + Eh))
                add(name + "_b2", edp.sum((0, 2, 3)) + gw * (ad + edp).sum((0, 2, 3)))
                sl = slice(32 * k, 32 * k + 32)
                add(name + "_w1", _wgrad(m.abs(), Edh[:, sl], (32, 32, 3, 3))
                    + gw * _wgrad(m.abs(), dh[:, sl].abs() + Edh[:, sl], (32, 32, 3, 3)))
                add(name + "_b1", Edh[:, sl].sum((0, 2, 3)) + gw * (dh[:, sl].abs() + Edh[:, sl]).sum((0, 2, 3)))
            s = src[b:b + 1].to(F64)
            cat = torch.cat([upsample2(s), img[b:b + 1].to(F64), depth[b:b + 1].to(F64)], 1).abs()
            dup = torch.cat([gamma(6) * upsample2(s.abs()), torch.zeros_like(cat[:, 48:])], 1)
            Dx = hulp(cat + dup) + dup
            ad = dmid.abs()
            add("out_w", _wgrad(cat + Dx, Edm, (32, 52, 3, 3)) + _wgrad(Dx, ad, (32, 52, 3, 3))
                + gw * _wgrad(cat + Dx, ad + Edm, (32, 52, 3, 3)))
            add("out_b", Edm.sum((0, 2, 3)) + gw * (ad + Edm).sum((0, 2, 3)))
    out = dict(d_src=torch.cat(d_src), d_depth=torch.cat(d_depth), **acc)
    return {k: torch.nan_to_num(out[k], nan=float("inf")) for k in GRAD_KEYS}
