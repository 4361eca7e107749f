"""Independent fp64 torch restatement of the UnetExtractor's half-resolution stem (TEST INFRASTRUCTURE ONLY), a CPU
emulation of the arithmetic of csrc/encoder_stem.cu in both precisions, and per-element error bounds for it.

Maths (reference core/extractor.py: in_ds + res1), params in gps_gaussian_b200.encoder.params_of order:
  y0 = conv5x5(x, stride 2, zero padding 2) + b;  x0 = relu(GN8(y0))
  per block (input v): y = conv3x3(v) + b;  h = relu(GN4(y));  y' = conv3x3(h) + b';  out = relu(v + relu(GN4(y')))
  GNg: per sample and group of 32 / g channels, mean and biased variance over the group's channels and pixels,
  (y - mean) / sqrt(var + 1e-5) * weight + bias per channel.  ReLU keeps NaN.
Convolutions are im2col (F.unfold) + matmul, so a non-finite input reaches only the outputs whose window holds it.

`forward64` evaluates this in fp64.  `emulate(x, params, mode)` runs the kernels' arithmetic on the CPU in fp32: mode
"tf32" rounds every convolution operand to TF32 (round to nearest, ties away); mode "fp16" rounds the operands and the
biases to fp16 and each convolution's output, bias included, to fp16.  Exact fp32 products, fp32 sums over the K terms
in a random order, the bias added in fp32.  GroupNorm as the kernels evaluate it: statistics in fp64 from the stored
values, A = fp32(weight rstd), C = fp32(bias - mean A), fp32(y A + C) (one rounding, as fmaf).  Its `mutant` argument
swaps in one deliberate error (MUTANTS) so the tests can show that each breaks a check.

Bounds (u = 2^-24, gamma(n) = n u / (1 - n u), hulp = half an ulp of the operand format: TF32 or fp16, both with 10
explicit mantissa bits, u_op = 2^-11 relative; fp16 adds 2^-25 absolute for its subnormals and inf above 65519):
  convolution  as oracle/gs_head_torch64.py: operands within d of the truth round to within Da = hulp(|a| + d) + d,
               weights within Dw = hulp(w); e = sum(|w| Da + Dw |a| + Dw Da) + gamma(2 (n + 1)) (sum |w||a| + that +
               |b|); fp16 mode adds hulp(|b|) for the bias and hulp(|y| + e) for the output rounding.
  GroupNorm    per group of N elements with errors E_i: the mean moves by Ebar = mean(E_i), each deviation by
               f_i = E_i + Ebar, the variance by dv = 2 mean(|y_i - mean| f_i) + mean(f_i^2), sigma = sqrt(var + eps)
               by ds = dv / sigma; with s = max(sqrt(eps), sigma - ds) (so the amplification is at most 1/sqrt(eps)),
               |weight| ((E + Ebar) / s + |y - mean| ds / (sigma s)); plus the evaluation: 3u ((|y| + E) |weight| / s
               + |bias| + (|mean| + Ebar) |weight| / s) for rounding A and C and the fused multiply-add, and 2^-40
               relative terms for the fp64 sums.
  ReLU         1-Lipschitz.
  residual     e_v + e_g + u |v + g|.
A bound that meets inf or NaN is inf.
"""
import torch
import torch.nn.functional as F

from oracle.gs_head_torch64 import gamma, hulp, ratio, tf32  # noqa: F401  (ratio is part of this module's interface)

F64 = torch.float64
U = 2.0 ** -24
EPS = 1e-5
KEYS = ("y0", "x0", "xb", "x1")
MUTANTS = ("in_ds_padding", "groups_swapped", "unbiased_var", "eps_outside_sqrt", "residual_dropped",
           "relu_drops_nan", "truncate")


# ---- the maths -------------------------------------------------------------------------------------------------------

def conv(x, w, b=None, stride=1, pad=None, pads=None):
    """Convolution with zero padding as im2col + matmul in x's dtype; pads = (left, right, top, bottom) overrides the
    symmetric `pad` (default (k - 1) / 2)."""
    B = x.shape[0]
    k = w.shape[-1]
    p = (k - 1) // 2 if pad is None else pad
    xp = F.pad(x, pads if pads is not None else (p, p, p, p))
    Ho = (xp.shape[2] - k) // stride + 1
    Wo = (xp.shape[3] - k) // stride + 1
    cols = F.unfold(xp, k, stride=stride)                          # [B, C k k, Ho Wo]
    out = torch.matmul(w.reshape(w.shape[0], -1).to(x.dtype), cols).view(B, w.shape[0], Ho, Wo)
    return out if b is None else out + b.to(x.dtype).view(1, -1, 1, 1)


def relu(x):
    return torch.where(x < 0, torch.zeros_like(x), x)


def group_norm(y, groups, weight, bias, eps=EPS):
    """GroupNorm from its definition, in y's dtype."""
    B, C, H, W = y.shape
    yg = y.reshape(B, groups, -1)
    mu = yg.mean(-1, keepdim=True)
    var = ((yg - mu) ** 2).mean(-1, keepdim=True)
    n = ((yg - mu) / torch.sqrt(var + eps)).view(B, C, H, W)
    return n * weight.to(y.dtype).view(1, -1, 1, 1) + bias.to(y.dtype).view(1, -1, 1, 1)


def _blocks(params):
    return [params[4 + 8 * k: 12 + 8 * k] for k in range(2)]


def forward64(x, params):
    """dict(y0, x0, xb, x1) in fp64: the in_ds convolution's output, in_ds's output, res1[0]'s and res1[1]'s outputs."""
    x = x.to(F64)
    ps = [p.to(F64) for p in params]
    y0 = conv(x, ps[0], ps[1], stride=2, pad=2)
    v = relu(group_norm(y0, 8, ps[2], ps[3]))
    out = dict(y0=y0, x0=v)
    for key, (w1, b1, g1, be1, w2, b2, g2, be2) in zip(("xb", "x1"), _blocks(ps)):
        h = relu(group_norm(conv(v, w1, b1), 4, g1, be1))
        v = relu(v + relu(group_norm(conv(h, w2, b2), 4, g2, be2)))
        out[key] = v
    return out


# ---- the kernels' arithmetic -------------------------------------------------------------------------------------

def _round(x, mode, truncate=False):
    x = x.to(torch.float32)
    return tf32(x, truncate) if mode == "tf32" else x.half().float()


def _conv32(x, w, b, gen, mode, stride=1, pad=None, pads=None, truncate=False):
    """fp32 convolution on rounded operands: exact products, fp32 sums over the K terms in a random order, + bias, and
    in fp16 mode the output rounded to fp16."""
    B = x.shape[0]
    k = w.shape[-1]
    p = (k - 1) // 2 if pad is None else pad
    xp = F.pad(_round(x, mode, truncate), pads if pads is not None else (p, p, p, p))
    Ho, Wo = (xp.shape[2] - k) // stride + 1, (xp.shape[3] - k) // stride + 1
    cols = F.unfold(xp, k, stride=stride)
    wm = _round(w, mode, truncate).reshape(w.shape[0], -1)
    acc = torch.zeros(B, w.shape[0], Ho * Wo, dtype=torch.float32)
    for j in torch.randperm(cols.shape[1], generator=gen).tolist():
        acc = acc + wm[None, :, j, None] * cols[:, None, j]
    bb = b.to(torch.float32) if mode == "tf32" else b.to(torch.float32).half().float()
    out = (acc + bb.view(1, -1, 1)).view(B, w.shape[0], Ho, Wo)
    return out if mode == "tf32" else out.half().float()


def _gn32(y, groups, weight, bias, mutant=None):
    B, C, H, W = y.shape
    yg = y.to(F64).reshape(B, groups, -1)
    n = yg.shape[-1]
    mu = yg.mean(-1, keepdim=True)
    var = ((yg - mu) ** 2).mean(-1, keepdim=True)
    if mutant == "unbiased_var":
        var = var * n / max(n - 1, 1)
    rstd = 1.0 / (torch.sqrt(var) + EPS) if mutant == "eps_outside_sqrt" else 1.0 / torch.sqrt(var + EPS)
    cpg = C // groups
    a64 = weight.to(F64).view(1, groups, cpg) * rstd                  # [B, G, cpg]
    A = a64.to(torch.float32).to(F64)
    Cc = (bias.to(F64).view(1, groups, cpg) - mu * a64).to(torch.float32).to(F64)
    out = yg.view(B, groups, cpg, -1) * A[..., None] + Cc[..., None]
    return out.to(torch.float32).view(B, C, H, W)


def emulate(x, params, mode="tf32", seed=0, mutant=None):
    """The kernels' result on the CPU in fp32 (see the module docstring): dict(y0, x0, xb, x1) and the raw outputs y1 ..
    y4 of the four 3x3 convolutions; `mutant` in MUTANTS injects one error."""
    assert mode in ("tf32", "fp16") and (mutant is None or mutant in MUTANTS), (mode, mutant)
    gen = torch.Generator().manual_seed(seed)
    x = x.to(torch.float32).cpu()
    ps = [p.to(torch.float32).cpu() for p in params]
    tr = mutant == "truncate"
    act = (lambda t: torch.fmax(t, torch.zeros_like(t))) if mutant == "relu_drops_nan" else relu
    g_in, g_res = (4, 8) if mutant == "groups_swapped" else (8, 4)
    if mutant == "in_ds_padding":                                    # the window one pixel off (padding 1 / 3)
        y0 = _conv32(x, ps[0], ps[1], gen, mode, stride=2, pads=(1, 3, 1, 3), truncate=tr)
    else:
        y0 = _conv32(x, ps[0], ps[1], gen, mode, stride=2, pad=2, truncate=tr)
    v = act(_gn32(y0, g_in, ps[2], ps[3], mutant))
    out = dict(y0=y0, x0=v)
    for k, (key, (w1, b1, g1, be1, w2, b2, g2, be2)) in enumerate(zip(("xb", "x1"), _blocks(ps))):
        ya = _conv32(v, w1, b1, gen, mode, truncate=tr)
        h = act(_gn32(ya, g_res, g1, be1, mutant))
        yb = _conv32(h, w2, b2, gen, mode, truncate=tr)
        g = act(_gn32(yb, g_res, g2, be2, mutant))
        v = act(g) if mutant == "residual_dropped" else act(v + g)
        out[key], out[f"y{2 * k + 1}"], out[f"y{2 * k + 2}"] = v, ya, yb
    return out


# ---- bounds ----------------------------------------------------------------------------------------------------------

def hulp_op(x, mode):
    """Half an ulp of |x| in the operand format: TF32, or fp16 (2^-25 below its normal range, inf above 65519)."""
    h = hulp(x)
    if mode == "tf32":
        return h
    a = x.abs()
    return torch.where(a >= 65520.0, torch.full_like(a, float("inf")), torch.clamp(h, min=2.0 ** -25))


def _conv_err(a, d, w, b, n, mode, stride=1, pad=None):
    aa, wa = a.abs(), w.abs()
    Da = hulp_op(aa + d, mode) + d
    Dw = hulp_op(w, mode)
    c = lambda t, k: conv(t, k, stride=stride, pad=pad)
    prod = c(Da, wa) + c(aa, Dw) + c(Da, Dw)
    e = prod + gamma(2 * (n + 1)) * (c(aa, wa) + prod + b.abs().view(1, -1, 1, 1))
    if mode == "fp16":
        e = e + hulp_op(b, mode).view(1, -1, 1, 1)
    return e


def _out_round(y, e, mode):
    return e if mode == "tf32" else e + hulp_op(y.abs() + e, mode)


def _gn_err(y, e, groups, weight, bias, out):
    B, C, H, W = y.shape
    cpg = C // groups
    yg, eg = y.reshape(B, groups, cpg, -1), e.reshape(B, groups, cpg, -1)
    red = lambda t: t.mean(dim=(2, 3), keepdim=True)
    mu = red(yg)
    dev = yg - mu
    var = red(dev * dev)
    ebar = red(eg) + 2.0 ** -40 * red(yg.abs())
    f = eg + ebar
    dv = 2 * red(dev.abs() * f) + red(f * f) + 2.0 ** -40 * (var + mu * mu)
    sig = torch.sqrt(var + EPS)
    ds = dv / sig
    s = torch.clamp(sig - ds, min=EPS ** 0.5)
    ga = weight.abs().view(1, groups, cpg, 1)
    ba = bias.abs().view(1, groups, cpg, 1)
    prop = ga * ((eg + ebar) / s + dev.abs() * ds / (sig * s))
    arith = 3 * U * ((yg.abs() + eg) * ga / s + ba + (mu.abs() + ebar) * ga / s)
    return (prop + arith).view(B, C, H, W)


def bounds(x, params, mode="tf32"):
    """Per-element bounds dict(y0, x0, xb, x1) on the kernels' results in `mode`, fp64 on the inputs' device."""
    x = x.to(F64)
    ps = [p.to(F64) for p in params]
    with torch.no_grad():
        cin = x.shape[1]
        y0 = conv(x, ps[0], ps[1], stride=2, pad=2)
        e0 = _out_round(y0, _conv_err(x, torch.zeros_like(x), ps[0], ps[1], 25 * cin, mode, stride=2, pad=2), mode)
        n0 = group_norm(y0, 8, ps[2], ps[3])
        v, ev = relu(n0), _gn_err(y0, e0, 8, ps[2], ps[3], n0)
        out = dict(y0=e0, x0=ev)
        for key, (w1, b1, g1, be1, w2, b2, g2, be2) in zip(("xb", "x1"), _blocks(ps)):
            y1 = conv(v, w1, b1)
            e1 = _out_round(y1, _conv_err(v, ev, w1, b1, 9 * 32, mode), mode)
            n1 = group_norm(y1, 4, g1, be1)
            h, eh = relu(n1), _gn_err(y1, e1, 4, g1, be1, n1)
            y2 = conv(h, w2, b2)
            e2 = _out_round(y2, _conv_err(h, eh, w2, b2, 9 * 32, mode), mode)
            n2 = group_norm(y2, 4, g2, be2)
            g, eg = relu(n2), _gn_err(y2, e2, 4, g2, be2, n2)
            ev = ev + eg + U * (v + g).abs()
            v = relu(v + g)
            out[key] = ev
    return {k: torch.nan_to_num(t, nan=float("inf")) for k, t in out.items()}


# ---- stage-local bounds --------------------------------------------------------------------------------------------
# The bounds above chain worst cases through four convolutions and five GroupNorms: each convolution can add its
# inputs' errors with aligned signs (sum |w| d), and each GroupNorm divides by its group's sigma, so past the first block
# they are valid but far from the errors that occur.  The kernels keep each convolution's raw output (y0 .. y4) in their
# workspace, so every stage is also checked on its own: its fp64 result from the kernels' stored input to that stage,
# within a bound on that stage's own arithmetic.  Together the stage checks pin the chain to fp64 step by step.

def _gn_arith(y, groups, weight, bias):
    """fp64 relu(GN(y)) of the stored values y, and a bound on the kernels' evaluation of it from the same y: the fp64
    statistics (2^-40 relative), A and C rounded to fp32 and the fused multiply-add (3u (|y| |A| + |bias| + |mean| |A|))."""
    B, C, H, W = y.shape
    cpg = C // groups
    yg = y.reshape(B, groups, cpg, -1)
    red = lambda t: t.mean(dim=(2, 3), keepdim=True)
    mu = red(yg)
    dev = yg - mu
    var = red(dev * dev)
    sig = torch.sqrt(var + EPS)
    ga = weight.abs().view(1, groups, cpg, 1)
    A = ga / sig
    dmu = 2.0 ** -40 * red(yg.abs())
    ds = 2.0 ** -40 * (var + mu * mu) / sig
    stats = ga * (dmu / sig + dev.abs() * ds / (sig * sig)) * 2
    arith = 3 * U * (yg.abs() * A + bias.abs().view(1, groups, cpg, 1) + mu.abs() * A)
    return relu(group_norm(y, groups, weight, bias)), (stats + arith).view(B, C, H, W)


def stage_checks(x, params, raws, mode="tf32"):
    """{stage: (want, bound)} for the kernels' stored convolution outputs raws = (y0, .., y4) (as fp32 or fp64 NCHW) and
    their x1: y0 from x; y1 from relu(GN8(y0)); y2 from relu(GN4(y1)); y3 from relu(relu(GN8(y0)) + relu(GN4(y2)));
    y4 from relu(GN4(y3)); x1 from y0, y2 and y4.  Each want is fp64 on the stored input; each bound covers the stage's
    own evaluation (operand rounding, fp32 sums, output rounding, the GroupNorm / ReLU / residual arithmetic)."""
    x = x.to(F64)
    ps = [p.to(F64) for p in params]
    ys = [r.to(F64).to(x.device) for r in raws]
    (w1a, b1a, g1a, be1a, w1b, b1b, g1b, be1b), (w2a, b2a, g2a, be2a, w2b, b2b, g2b, be2b) = _blocks(ps)
    with torch.no_grad():
        out = {}
        cin = x.shape[1]
        out["y0"] = (conv(x, ps[0], ps[1], stride=2, pad=2), None)
        y0 = out["y0"][0]
        out["y0"] = (y0, _out_round(y0, _conv_err(x, torch.zeros_like(x), ps[0], ps[1], 25 * cin, mode, 2, 2), mode))
        x0, e0 = _gn_arith(ys[0], 8, ps[2], ps[3])
        h1, e1 = _gn_arith(ys[1], 4, g1a, be1a)
        g2, e2 = _gn_arith(ys[2], 4, g1b, be1b)
        xb, eb = relu(x0 + g2), e0 + e2 + U * (x0 + g2).abs()
        h3, e3 = _gn_arith(ys[3], 4, g2a, be2a)
        g4, e4 = _gn_arith(ys[4], 4, g2b, be2b)
        for key, v, d, w, b in (("y1", x0, e0, w1a, b1a), ("y2", h1, e1, w1b, b1b), ("y3", xb, eb, w2a, b2a),
                                ("y4", h3, e3, w2b, b2b)):
            y = conv(v, w, b)
            out[key] = (y, _out_round(y, _conv_err(v, d, w, b, 9 * 32, mode), mode))
        x1 = relu(xb + g4)
        out["x1"] = (x1, eb + e4 + U * (xb + g4).abs())
    return {k: (w, torch.nan_to_num(b, nan=float("inf"))) for k, (w, b) in out.items()}
