"""Independent fp64 torch restatement of the regressor's decoder1 (TEST INFRASTRUCTURE ONLY), a CPU emulation of the
TF32 arithmetic of csrc/decoder1.cu, and per-element error bounds for it.

Maths (reference lib/gs_parm_network.py, decoder1 = two core/extractor.py ResidualBlocks with GroupNorm(6, 48)), params
in gps_gaussian_b200.decoder.params_of order:
  v   = cat(up(s), f_i, f_d), up the bilinear x2 of oracle/gs_head_torch64.py (align_corners=False)
  y1  = conv3x3(v) + b;  yd = conv1x1(v) + b;  y2 = conv3x3(relu(GN6(y1))) + b;  xb = relu(GN6(yd) + relu(GN6(y2)))
  y3  = conv3x3(xb) + b;  y4 = conv3x3(relu(GN6(y3))) + b;  out = relu(xb + relu(GN6(y4)))
The convolutions and GroupNorm are oracle/encoder_torch64.py's (im2col + matmul; GroupNorm from its definition).

`forward64` evaluates this in fp64.  `emulate` runs the kernels' arithmetic on the CPU in fp32: the upsample evaluated in
fp32 with torch's formula, every convolution operand rounded to TF32, exact products, fp32 sums in a random order, the
bias after the sum, GroupNorm as the kernels evaluate it (fp64 statistics, A and C rounded to fp32, one fmaf).  Its
`mutant` argument swaps in one deliberate error (MUTANTS) so the tests can show that each breaks a check.

Bounds: encoder_torch64's convolution, GroupNorm, ReLU and residual terms (TF32 mode), and for the upsampled channels of
v an input error of gamma(6) up(|s|), as oracle/gs_head_torch64.py bounds its fp32 interpolation (weights 0, 1/4, 3/4
or 1, two products and a sum per direction).  `bounds` chains them from the inputs to `out`; `stage_checks` bounds each
stage from the kernels' stored input to that stage, which pins the chain to fp64 step by step (see encoder_torch64).
"""
import torch

from oracle.encoder_torch64 import _conv32, _conv_err, _gn32, _gn_arith, _gn_err, conv, group_norm, relu
from oracle.gs_head_torch64 import gamma, ratio, upsample2  # noqa: F401  (ratio is part of this module's interface)

F64 = torch.float64
U = 2.0 ** -24
G = 6
KEYS = ("y1", "yd", "y2", "y3", "y4", "out")
MUTANTS = ("upsample_phase", "concat_order", "downsample_relu", "unbiased_var", "residual_dropped", "relu_drops_nan")


def _split(ps):
    """(block 0: conv1 w, b, norm1 w, b, conv2 w, b, norm2 w, b, down w, b, norm3 w, b), (block 1: 8 tensors)"""
    return ps[:12], ps[12:]


def forward64(s, f_i, f_d, params):
    """dict(y1, yd, y2, y3, y4, xb, out) in fp64: the five convolution outputs, block 0's output and decoder1's."""
    s, f_i, f_d = (t.to(F64) for t in (s, f_i, f_d))
    ps = [p.to(F64) for p in params]
    (w1, b1, g1, be1, w2, b2, g2, be2, wd, bd, gd, bed), (w3, b3, g3, be3, w4, b4, g4, be4) = _split(ps)
    v = torch.cat([upsample2(s), f_i, f_d], 1)
    y1, yd = conv(v, w1, b1), conv(v, wd, bd)
    y2 = conv(relu(group_norm(y1, G, g1, be1)), w2, b2)
    xb = relu(group_norm(yd, G, gd, bed) + relu(group_norm(y2, G, g2, be2)))
    y3 = conv(xb, w3, b3)
    y4 = conv(relu(group_norm(y3, G, g3, be3)), w4, b4)
    return dict(y1=y1, yd=yd, y2=y2, y3=y3, y4=y4, xb=xb, out=relu(xb + relu(group_norm(y4, G, g4, be4))))


def emulate(s, f_i, f_d, params, seed=0, mutant=None):
    """The kernels' result on the CPU in fp32 (see the module docstring): the same keys as forward64; `mutant` in
    MUTANTS injects one error."""
    assert mutant is None or mutant in MUTANTS, mutant
    gen = torch.Generator().manual_seed(seed)
    s, f_i, f_d = (t.to(torch.float32).cpu() for t in (s, f_i, f_d))
    ps = [p.to(torch.float32).cpu() for p in params]
    (w1, b1, g1, be1, w2, b2, g2, be2, wd, bd, gd, bed), (w3, b3, g3, be3, w4, b4, g4, be4) = _split(ps)
    act = (lambda t: torch.fmax(t, torch.zeros_like(t))) if mutant == "relu_drops_nan" else relu
    up = upsample2(s, align_corners=mutant == "upsample_phase")
    v = torch.cat([up, f_d, f_i] if mutant == "concat_order" else [up, f_i, f_d], 1)
    gn = lambda y, g, b: _gn32(y, G, g, b, mutant)
    y1, yd = _conv32(v, w1, b1, gen, "tf32"), _conv32(v, wd, bd, gen, "tf32")
    y2 = _conv32(act(gn(y1, g1, be1)), w2, b2, gen, "tf32")
    nd = gn(yd, gd, bed)
    if mutant == "downsample_relu":
        nd = act(nd)
    xb = act(nd + act(gn(y2, g2, be2)))
    y3 = _conv32(xb, w3, b3, gen, "tf32")
    y4 = _conv32(act(gn(y3, g3, be3)), w4, b4, gen, "tf32")
    g = act(gn(y4, g4, be4))
    out = act(g) if mutant == "residual_dropped" else act(xb + g)
    return dict(y1=y1, yd=yd, y2=y2, y3=y3, y4=y4, xb=xb, out=out)


def _input_err(s, f_i, f_d):
    """v and the bound on the kernels' fp32 v: the upsample's interpolation on its 64 channels, exact elsewhere."""
    v = torch.cat([upsample2(s), f_i, f_d], 1)
    d = torch.cat([gamma(6) * upsample2(s.abs()), torch.zeros_like(f_i), torch.zeros_like(f_d)], 1)
    return v, d


def bounds(s, f_i, f_d, params):
    """Per-element bounds dict(y1, yd, y2, y3, y4, out) on the kernels' results, chained from the inputs, fp64 on the
    inputs' device."""
    s, f_i, f_d = (t.to(F64) for t in (s, f_i, f_d))
    ps = [p.to(F64) for p in params]
    (w1, b1, g1, be1, w2, b2, g2, be2, wd, bd, gd, bed), (w3, b3, g3, be3, w4, b4, g4, be4) = _split(ps)
    cin = w1.shape[1]
    with torch.no_grad():
        v, d = _input_err(s, f_i, f_d)
        y1, yd = conv(v, w1, b1), conv(v, wd, bd)
        e1, ed = _conv_err(v, d, w1, b1, 9 * cin, "tf32"), _conv_err(v, d, wd, bd, cin, "tf32")
        h1, eh1 = relu(group_norm(y1, G, g1, be1)), _gn_err(y1, e1, G, g1, be1, None)
        y2 = conv(h1, w2, b2)
        e2 = _conv_err(h1, eh1, w2, b2, 9 * 48, "tf32")
        n2, en2 = relu(group_norm(y2, G, g2, be2)), _gn_err(y2, e2, G, g2, be2, None)
        nd, end = group_norm(yd, G, gd, bed), _gn_err(yd, ed, G, gd, bed, None)
        xb, exb = relu(nd + n2), end + en2 + U * (nd + n2).abs()
        y3 = conv(xb, w3, b3)
        e3 = _conv_err(xb, exb, w3, b3, 9 * 48, "tf32")
        h3, eh3 = relu(group_norm(y3, G, g3, be3)), _gn_err(y3, e3, G, g3, be3, None)
        y4 = conv(h3, w4, b4)
        e4 = _conv_err(h3, eh3, w4, b4, 9 * 48, "tf32")
        n4, en4 = relu(group_norm(y4, G, g4, be4)), _gn_err(y4, e4, G, g4, be4, None)
        out = dict(y1=e1, yd=ed, y2=e2, y3=e3, y4=e4, out=exb + en4 + U * (xb + n4).abs())
    return {k: torch.nan_to_num(t, nan=float("inf")) for k, t in out.items()}


def stage_checks(s, f_i, f_d, params, raws):
    """{stage: (want, bound)} for the kernels' stored convolution outputs raws = (y1, yd, y2, y3, y4) (fp32 or fp64 NCHW)
    and their out: y1 and yd from the inputs; y2 from relu(GN(y1)); y3 from relu(GN(yd) + relu(GN(y2))); y4 from
    relu(GN(y3)); out from yd, y2 and y4.  Each want is fp64 on the stored input, each bound covers that stage's own
    evaluation (the interpolation, operand rounding, fp32 sums, the GroupNorm / ReLU / residual arithmetic)."""
    s, f_i, f_d = (t.to(F64) for t in (s, f_i, f_d))
    ps = [p.to(F64) for p in params]
    y1s, yds, y2s, y3s, y4s = (r.to(F64).to(s.device) for r in raws)
    (w1, b1, g1, be1, w2, b2, g2, be2, wd, bd, gd, bed), (w3, b3, g3, be3, w4, b4, g4, be4) = _split(ps)
    cin = w1.shape[1]
    with torch.no_grad():
        v, d = _input_err(s, f_i, f_d)
        out = {}
        y = conv(v, w1, b1)
        out["y1"] = (y, _conv_err(v, d, w1, b1, 9 * cin, "tf32"))
        y = conv(v, wd, bd)
        out["yd"] = (y, _conv_err(v, d, wd, bd, cin, "tf32"))
        h1, e1 = _gn_arith(y1s, G, g1, be1)
        n2, e2 = _gn_arith(y2s, G, g2, be2)
        _, ed = _gn_arith(yds, G, gd, bed)                   # the same arithmetic without the ReLU (1-Lipschitz)
        nd = group_norm(yds, G, gd, bed)
        xb, exb = relu(nd + n2), ed + e2 + U * (nd + n2).abs()
        h3, e3 = _gn_arith(y3s, G, g3, be3)
        n4, e4 = _gn_arith(y4s, G, g4, be4)
        for key, a, da, w, b in (("y2", h1, e1, w2, b2), ("y3", xb, exb, w3, b3), ("y4", h3, e3, w4, b4)):
            y = conv(a, w, b)
            out[key] = (y, _conv_err(a, da, w, b, 9 * 48, "tf32"))
        out["out"] = (relu(xb + n4), exb + e4 + U * (xb + n4).abs())
    return {k: (w, torch.nan_to_num(b, nan=float("inf"))) for k, (w, b) in out.items()}
