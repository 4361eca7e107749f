"""Independent fp64 torch restatement of the Gaussian-parameter regressor's full-resolution tail (TEST INFRASTRUCTURE
ONLY), its TF32 emulation and per-element error bounds for csrc/gs_head.cu.

Maths (reference lib/gs_parm_network.py, GSRegresser.forward from `self.up(up1)` on), with params in
gps_gaussian_b200.gs_head.params_of order (out_w, out_b, rot_w1, rot_b1, rot_w2, rot_b2, scale_..., opacity_...):
  up      bilinear x2, align_corners=False: source s = (d + 0.5) / 2 - 0.5 clamped at 0, i0 = floor(s), i1 = min(i0 + 1,
          n - 1), weights 1 - (s - i0), s - i0, separably in y and x;
  mid     relu(conv3x3(cat[up, img, depth]) + out_b), zero padding of the concatenated tensor;
  h       relu(conv3x3(mid) + b1) per head;  pre = conv1x1(h) + b2 per head (rot 4, scale 3, opacity 1 channels);
  rot     pre / max(||pre||_2, 1e-12);  scale = min(softplus_100(pre), 0.01) with softplus_100(x) = x where 100 x > 20,
          log1p(exp(100 x)) / 100 elsewhere;  opacity = sigmoid(pre).  ReLU and min keep NaN.
Convolutions are im2col (F.unfold) + matmul, so a non-finite input only reaches the outputs whose window holds it.

`forward64` evaluates this in the inputs' dtype (pass fp64; fp32 inputs widen exactly).  `emulate` runs the kernels'
arithmetic on the CPU: every convolution operand rounded to TF32 (round to nearest, ties away, as cvt.rna.tf32.f32),
exact fp32 products, fp32 accumulation over the K terms in a random order, then the bias, the activations in fp32.
Its `mutant` argument swaps in one deliberate error (MUTANTS) so the tests can show that each breaks a check.

Bounds.  u = 2^-24, gamma(n) = n u / (1 - n u), hulp(x) = half a TF32 ulp of x (2^(e - 12) for |x| in [2^(e-1), 2^e)).
For one convolution with true operands w (fp32 weights, exact) and a (true activations) where the kernel's fp32 operand
a32 is within d of a:  |rna(w) - w| <= Dw = hulp(w) and |rna(a32) - a| <= Da = hulp(|a| + d) + d (a RN flip caused by d
is inside this).  Per output, with the sums over the window and the input channels (conv2d of the magnitude fields):
      e = sum (|w| Da + Dw |a| + Dw Da) + gamma(2 (n + 1)) (sum |w||a| + sum (|w| Da + Dw |a| + Dw Da) + |b|)
(n = K terms; the factor 2 allows an accumulator that truncates rather than rounds).  ReLU is 1-Lipschitz, so e carries
to the next convolution as its d: out_conv (n = 9 x 52, d = gamma(6) up(|src|) on the upsampled channels, 0 on img and
depth) -> the three 3x3 heads (n = 9 x 32) -> the 1x1 convolutions (n = 32).  Activations, from the pre-activation
bound e: sigmoid is 1/4-Lipschitz (+ 8u for its fp32 evaluation); softplus_100 is 1-Lipschitz (+ u |x| for the rounding
of 100 x, 8u |softplus| for expf / log1pf / the division, 1e-10 for the threshold's 2e-11 step) and the clamp adds
|0.01f - 0.01| < 2^-30; normalize moves by at most 2 E / ||pre|| for a pre-activation error vector of norm E (its Jacobian
at the fp64 point has norm 1 / ||pre||; the factor 2 makes the first-order bound hold for any E), capped at 2, E / 1e-12
where pre = 0, + 8u for its fp32 evaluation.  A bound that meets inf or NaN is inf.
"""
import numpy as np
import torch
import torch.nn.functional as F

F64 = torch.float64
U = 2.0 ** -24
MUTANTS = ("align_corners", "edge_pad", "truncate", "softplus_no_threshold", "normalize_no_eps", "relu_drops_nan",
           "heads_swapped")


def gamma(n):
    return n * U / (1.0 - n * U)


# ---- the maths -------------------------------------------------------------------------------------------------------

def _src_index(n_dst, n_src, align_corners=False):
    d = torch.arange(n_dst, dtype=F64)
    if align_corners:
        s = d * ((n_src - 1) / (n_dst - 1)) if n_dst > 1 else torch.zeros_like(d)
    else:
        s = ((d + 0.5) * 0.5 - 0.5).clamp(min=0.0)
    i0 = s.floor().long().clamp(max=n_src - 1)
    i1 = torch.where(i0 < n_src - 1, i0 + 1, i0)
    l1 = s - i0.to(F64)
    return i0, i1, 1.0 - l1, l1


def upsample2(x, align_corners=False):
    """Bilinear x2 of [B,C,h,w] in x's dtype, weights in that dtype (they are 0, 0.25, 0.75 or 1: exact)."""
    B, C, h, w = x.shape
    y0, y1, ly0, ly1 = (t.to(x.device) for t in _src_index(2 * h, h, align_corners))
    x0, x1, lx0, lx1 = (t.to(x.device) for t in _src_index(2 * w, w, align_corners))
    ly0, ly1 = ly0.to(x.dtype)[:, None], ly1.to(x.dtype)[:, None]
    lx0, lx1 = lx0.to(x.dtype), lx1.to(x.dtype)
    r0, r1 = x[:, :, y0], x[:, :, y1]
    return ly0 * (lx0 * r0[..., x0] + lx1 * r0[..., x1]) + ly1 * (lx0 * r1[..., x0] + lx1 * r1[..., x1])


def _pad(x, k, edge=False):
    p = (k - 1) // 2
    return F.pad(x, (p, p, p, p), mode="replicate" if edge else "constant") if p else x


def conv(x, w, b=None, edge_pad=False):
    """'Same' convolution with zero padding (edge_pad: replicated borders), as im2col + matmul in x's dtype."""
    B, C, H, W = x.shape
    k = w.shape[-1]
    cols = F.unfold(_pad(x, k, edge_pad), k)                         # [B, C k k, H W]
    out = torch.matmul(w.reshape(w.shape[0], -1).to(x.dtype), cols).view(B, w.shape[0], H, W)
    return out if b is None else out + b.to(x.dtype).view(1, -1, 1, 1)


def relu(x):
    return torch.where(x < 0, torch.zeros_like(x), x)


def softplus100(x):
    return torch.where(x * 100 > 20, x, torch.log1p(torch.exp(x * 100)) / 100)


def clamp_max(x, m):
    return torch.where(x > m, torch.full_like(x, m), x)


def normalize(x, eps=1e-12):
    n = x.pow(2).sum(1, keepdim=True).sqrt()
    return x / torch.where(n < eps, torch.full_like(n, eps), n)


def _heads(params):
    return [(params[2 + 4 * i], params[3 + 4 * i], params[4 + 4 * i], params[5 + 4 * i]) for i in range(3)]


def forward64(src, img, depth, params):
    """dict(rot, scale, opacity, scale_pre, pre, mid) in the inputs' dtype (everything is converted to fp64)."""
    src, img, depth = (t.to(F64) for t in (src, img, depth))
    ps = [p.to(F64) for p in params]
    mid = relu(conv(torch.cat([upsample2(src), img, depth], 1), ps[0], ps[1]))
    pre = [conv(relu(conv(mid, w1, b1)), w2, b2) for w1, b1, w2, b2 in _heads(ps)]
    sp = softplus100(pre[1])
    return dict(rot=normalize(pre[0]), scale=clamp_max(sp, 0.01), opacity=torch.sigmoid(pre[2]), scale_pre=sp,
                pre=torch.cat(pre, 1), mid=mid)


# ---- the kernels' arithmetic -------------------------------------------------------------------------------------

def tf32(x, truncate=False):
    """fp32 tensor rounded to TF32 (10 explicit mantissa bits): round to nearest, ties away (cvt.rna.tf32.f32); inf and
    NaN unchanged.  truncate: chop the low 13 bits instead."""
    x = x.to(torch.float32).contiguous()
    bits = x.view(torch.int32)
    r = bits if truncate else bits + 0x1000
    r = r & ~0x1FFF
    finite = torch.isfinite(x)
    return torch.where(finite, r.view(torch.float32), x)


def _conv32(x, w, b, gen, truncate=False, edge_pad=False):
    """fp32 convolution on TF32 operands: exact products, fp32 sums over the K terms in a random order, then + b."""
    B, C, H, W = x.shape
    k = w.shape[-1]
    cols = F.unfold(_pad(tf32(x, truncate), k, edge_pad), k)          # [B, K, HW]
    wm = tf32(w, truncate).reshape(w.shape[0], -1)                    # [Cout, K]
    acc = torch.zeros(B, w.shape[0], H * W, dtype=torch.float32)
    for j in torch.randperm(cols.shape[1], generator=gen).tolist():
        acc = acc + wm[None, :, j, None] * cols[:, None, j]
    return (acc + b.to(torch.float32).view(1, -1, 1)).view(B, w.shape[0], H, W)


def emulate(src, img, depth, params, seed=0, mutant=None):
    """The kernels' result on the CPU in fp32 (see the module docstring); `mutant` in MUTANTS injects one error."""
    assert mutant is None or mutant in MUTANTS, mutant
    gen = torch.Generator().manual_seed(seed)
    src, img, depth = (t.to(torch.float32).cpu() for t in (src, img, depth))
    ps = [p.to(torch.float32).cpu() for p in params]
    tr, edge = mutant == "truncate", mutant == "edge_pad"
    act = (lambda x: torch.fmax(x, torch.zeros_like(x))) if mutant == "relu_drops_nan" else relu
    x = torch.cat([upsample2(src, mutant == "align_corners"), img, depth], 1)
    mid = act(_conv32(x, ps[0], ps[1], gen, tr, edge))
    heads = _heads(ps)
    if mutant == "heads_swapped":
        heads[1], heads[2] = (heads[2][0],) + heads[1][1:], (heads[1][0],) + heads[2][1:]
    pre = [_conv32(act(_conv32(mid, w1, b1, gen, tr, edge)), w2, b2, gen, tr) for w1, b1, w2, b2 in heads]
    if mutant == "softplus_no_threshold":
        sp = torch.log1p(torch.exp(pre[1] * 100)) / 100
    else:
        sp = softplus100(pre[1])
    rot = normalize(pre[0], eps=0.0 if mutant == "normalize_no_eps" else 1e-12)
    return dict(rot=rot, scale=clamp_max(sp, np.float32(0.01).item()), opacity=torch.sigmoid(pre[2]), scale_pre=sp,
                pre=torch.cat(pre, 1), mid=mid)


# ---- bounds ----------------------------------------------------------------------------------------------------------

def hulp(x):
    """Half a TF32 ulp of |x| (0 at 0)."""
    m, e = torch.frexp(x.abs())
    return torch.where(m == 0, torch.zeros_like(x), torch.ldexp(torch.ones_like(x), e - 12))


def _conv_err(a, d, w, b, n):
    """Bound on |kernel - exact| of conv(a, w) + b when the kernel's fp32 operands are within d of a."""
    aa, wa = a.abs(), w.abs()
    Da = hulp(aa + d) + d
    Dw = hulp(w)
    prod = conv(Da, wa) + conv(aa, Dw) + conv(Da, Dw)
    return prod + gamma(2 * (n + 1)) * (conv(aa, wa) + prod + b.abs().view(1, -1, 1, 1))


def bounds(src, img, depth, params):
    """Per-element bounds dict(rot [B,4,H,W], scale [B,3,H,W], opacity [B,1,H,W]) on the kernels' results, and on the
    intermediates `emulate` exposes (scale_pre, pre [B,8,H,W], mid [B,32,H,W]), fp64 on the inputs' device."""
    src, img, depth = (t.to(F64) for t in (src, img, depth))
    ps = [p.to(F64) for p in params]
    with torch.no_grad():
        up = upsample2(src)
        x = torch.cat([up, img, depth], 1)
        d = torch.cat([gamma(6) * upsample2(src.abs()), torch.zeros_like(img), torch.zeros_like(depth)], 1)
        e_mid = _conv_err(x, d, ps[0], ps[1], 9 * 52)
        mid = relu(conv(x, ps[0], ps[1]))
        e_pre, pre = [], []
        for w1, b1, w2, b2 in _heads(ps):
            h = relu(conv(mid, w1, b1))
            e_h = _conv_err(mid, e_mid, w1, b1, 9 * 32)
            e_pre.append(_conv_err(h, e_h, w2, b2, 32))
            pre.append(conv(h, w2, b2))
        E = e_pre[0].pow(2).sum(1, keepdim=True).sqrt()
        r = pre[0].pow(2).sum(1, keepdim=True).sqrt()
        rot = torch.where(r > 0, 2 * E / r, E / 1e-12).clamp(max=2.0).expand_as(pre[0]) + 8 * U
        sp = softplus100(pre[1])
        scale_pre = e_pre[1] + 1e-10 + U * (pre[1].abs() + e_pre[1]) + 8 * U * (sp.abs() + e_pre[1])
        out = dict(rot=rot, scale=scale_pre + 2.0 ** -30, opacity=0.25 * e_pre[2] + 8 * U, scale_pre=scale_pre,
                   pre=torch.cat(e_pre, 1), mid=e_mid)
    return {k: torch.nan_to_num(v, nan=float("inf")) for k, v in out.items()}


def ratio(got, want, bound):
    """Worst |got - want| / bound where want is finite (0 where they agree exactly); inf when the NaN positions differ or
    an infinite want is not matched exactly."""
    got = torch.as_tensor(got).to(device=want.device, dtype=F64).reshape(want.shape)
    nan = torch.isnan(want)
    if not torch.equal(torch.isnan(got), nan):
        return float("inf")
    inf = torch.isinf(want)
    if not torch.equal(got[inf], want[inf]):
        return float("inf")
    err = (got - want).abs()
    r = torch.where(nan | inf | (err == 0), torch.zeros_like(err), err / bound.to(want.device))
    return float(r.max()) if r.numel() else 0.0
