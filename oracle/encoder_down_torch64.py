"""Independent fp64 torch restatement of the UnetExtractor's stride-2 residual stages res2 / res3 (TEST INFRASTRUCTURE
ONLY), a CPU emulation of the arithmetic of csrc/encoder_down.cu in both precisions, and per-element error bounds for it.
The machinery (im2col convolution, GroupNorm, the operand rounding, the bound terms) is oracle/encoder_torch64.py's.

Maths (reference core/extractor.py: two ResidualBlocks, the first with stride 2), params in
gps_gaussian_b200.encoder.down_params_of order, G = C / 8 groups:
  ya = conv3x3(v, stride 2, padding 1) + b     yd = conv1x1(v, stride 2) + b
  yb = conv3x3(relu(GN1(ya))) + b              xb = relu(GN3(yd) + relu(GN2(yb)))
  yc = conv3x3(xb) + b                         ye = conv3x3(relu(GN1'(yc))) + b
  out = relu(xb + relu(GN2'(ye)))

`forward64` evaluates this in fp64.  `emulate(x, params, mode)` runs the kernels' arithmetic on the CPU in fp32 as
encoder_torch64.emulate does (TF32 or fp16 operands, exact products, fp32 sums in a random order, fp16 output rounding,
GroupNorm statistics in fp64 with A and C rounded to fp32).  Its `mutant` argument swaps in one deliberate error
(MUTANTS) so the tests can show that each breaks a check.  `bounds` chains worst-case errors end to end;
`stage_checks` checks each stage from the kernels' stored input to it.
"""
import torch

from oracle.encoder_torch64 import (F64, U, _conv32, _conv_err, _gn32, _gn_arith, _gn_err, _out_round, conv,
                                    group_norm, ratio, relu)  # noqa: F401  (ratio is part of this module's interface)

KEYS = ("ya", "yd", "yb", "yc", "ye", "out")
MUTANTS = ("stride_phase", "downsample_no_norm3", "downsample_relu", "groups_other_stage", "unbiased_var",
           "eps_outside_sqrt", "residual_dropped", "relu_drops_nan")


def _unpack(params):
    ps = list(params)
    return ps[0:4], ps[4:8], ps[8:12], ps[12:16], ps[16:20]


def forward64(x, params):
    """dict(ya, yd, yb, yc, ye, xb, out) in fp64."""
    x = x.to(F64)
    ps = [p.to(F64) for p in params]
    (w1, b1, g1, e1), (w2, b2, g2, e2), (wd, bd, g3, e3), (w4, b4, g4, e4), (w5, b5, g5, e5) = _unpack(ps)
    G = w1.shape[0] // 8
    ya = conv(x, w1, b1, stride=2, pad=1)
    yd = conv(x, wd, bd, stride=2, pad=0)
    yb = conv(relu(group_norm(ya, G, g1, e1)), w2, b2)
    xb = relu(group_norm(yd, G, g3, e3) + relu(group_norm(yb, G, g2, e2)))
    yc = conv(xb, w4, b4)
    ye = conv(relu(group_norm(yc, G, g4, e4)), w5, b5)
    out = relu(xb + relu(group_norm(ye, G, g5, e5)))
    return dict(ya=ya, yd=yd, yb=yb, yc=yc, ye=ye, xb=xb, out=out)


def emulate(x, params, mode="tf32", seed=0, mutant=None):
    """The kernels' result on the CPU in fp32: dict(ya, yd, yb, yc, ye, out); `mutant` in MUTANTS injects one error."""
    assert mode in ("tf32", "fp16") and (mutant is None or mutant in MUTANTS), (mode, mutant)
    gen = torch.Generator().manual_seed(seed)
    x = x.to(torch.float32).cpu()
    ps = [p.to(torch.float32).cpu() for p in params]
    (w1, b1, g1, e1), (w2, b2, g2, e2), (wd, bd, g3, e3), (w4, b4, g4, e4), (w5, b5, g5, e5) = _unpack(ps)
    C = w1.shape[0]
    G = (12 if C == 48 else 6) if mutant == "groups_other_stage" else C // 8
    act = (lambda t: torch.fmax(t, torch.zeros_like(t))) if mutant == "relu_drops_nan" else relu
    gn = lambda y, g, b: _gn32(y, G, g, b, mutant)
    if mutant == "stride_phase":                         # the stride-2 window one input pixel off
        ya = _conv32(x, w1, b1, gen, mode, stride=2, pads=(0, 2, 0, 2))
    else:
        ya = _conv32(x, w1, b1, gen, mode, stride=2, pad=1)
    yd = _conv32(x, wd, bd, gen, mode, stride=2, pad=0)
    yb = _conv32(act(gn(ya, g1, e1)), w2, b2, gen, mode)
    d = yd if mutant == "downsample_no_norm3" else gn(yd, g3, e3)
    if mutant == "downsample_relu":
        d = act(d)
    xb = act(d + act(gn(yb, g2, e2)))
    yc = _conv32(xb, w4, b4, gen, mode)
    ye = _conv32(act(gn(yc, g4, e4)), w5, b5, gen, mode)
    g = act(gn(ye, g5, e5))
    out = act(g) if mutant == "residual_dropped" else act(xb + g)
    return dict(ya=ya, yd=yd, yb=yb, yc=yc, ye=ye, out=out)


def bounds(x, params, mode="tf32"):
    """Per-element bounds dict(ya, yd, yb, yc, ye, out) on the kernels' results in `mode`, chained end to end."""
    x = x.to(F64)
    ps = [p.to(F64) for p in params]
    (w1, b1, g1, e1), (w2, b2, g2, e2), (wd, bd, g3, e3), (w4, b4, g4, e4), (w5, b5, g5, e5) = _unpack(ps)
    cin, C = x.shape[1], w1.shape[0]
    G = C // 8
    z = torch.zeros_like(x)
    with torch.no_grad():
        ya = conv(x, w1, b1, stride=2, pad=1)
        ea = _out_round(ya, _conv_err(x, z, w1, b1, 9 * cin, mode, stride=2, pad=1), mode)
        yd = conv(x, wd, bd, stride=2, pad=0)
        ed = _out_round(yd, _conv_err(x, z, wd, bd, cin, mode, stride=2, pad=0), mode)
        n1 = group_norm(ya, G, g1, e1)
        h1, eh1 = relu(n1), _gn_err(ya, ea, G, g1, e1, n1)
        yb = conv(h1, w2, b2)
        eb = _out_round(yb, _conv_err(h1, eh1, w2, b2, 9 * C, mode), mode)
        n3, n2 = group_norm(yd, G, g3, e3), group_norm(yb, G, g2, e2)
        e3n, e2n = _gn_err(yd, ed, G, g3, e3, n3), _gn_err(yb, eb, G, g2, e2, n2)
        s = n3 + relu(n2)
        xb, exb = relu(s), e3n + e2n + U * s.abs()
        yc = conv(xb, w4, b4)
        ec = _out_round(yc, _conv_err(xb, exb, w4, b4, 9 * C, mode), mode)
        n4 = group_norm(yc, G, g4, e4)
        h4, eh4 = relu(n4), _gn_err(yc, ec, G, g4, e4, n4)
        ye = conv(h4, w5, b5)
        ee = _out_round(ye, _conv_err(h4, eh4, w5, b5, 9 * C, mode), mode)
        n5 = group_norm(ye, G, g5, e5)
        g, eg = relu(n5), _gn_err(ye, ee, G, g5, e5, n5)
        eo = exb + eg + U * (xb + g).abs()
    out = dict(ya=ea, yd=ed, yb=eb, yc=ec, ye=ee, out=eo)
    return {k: torch.nan_to_num(t, nan=float("inf")) for k, t in out.items()}


def stage_checks(x, params, raws, mode="tf32"):
    """{stage: (want, bound)} for the kernels' stored convolution outputs raws = (ya, yd, yb, yc, ye) (fp32 or fp64
    NCHW) and their out: ya, yd from x; yb from relu(GN(ya)); yc from xb = relu(GN(yd) + relu(GN(yb))); ye from
    relu(GN(yc)); out from yd, yb and ye.  Each want is fp64 on the stored input; each bound covers the stage's own
    evaluation (operand rounding, fp32 sums, output rounding, the GroupNorm / ReLU / residual arithmetic)."""
    x = x.to(F64)
    ps = [p.to(F64) for p in params]
    ys = [r.to(F64).to(x.device) for r in raws]
    (w1, b1, g1, e1), (w2, b2, g2, e2), (wd, bd, g3, e3), (w4, b4, g4, e4), (w5, b5, g5, e5) = _unpack(ps)
    cin, C = x.shape[1], w1.shape[0]
    G = C // 8
    z = torch.zeros_like(x)
    with torch.no_grad():
        out = {}
        ya = conv(x, w1, b1, stride=2, pad=1)
        out["ya"] = (ya, _out_round(ya, _conv_err(x, z, w1, b1, 9 * cin, mode, stride=2, pad=1), mode))
        yd = conv(x, wd, bd, stride=2, pad=0)
        out["yd"] = (yd, _out_round(yd, _conv_err(x, z, wd, bd, cin, mode, stride=2, pad=0), mode))
        h1, eh1 = _gn_arith(ys[0], G, g1, e1)
        # GN3 without the ReLU: _gn_arith's relu is 1-Lipschitz, so its bound also covers the value before the ReLU
        n3 = group_norm(ys[1], G, g3, e3)
        _, e3n = _gn_arith(ys[1], G, g3, e3)
        h2, eh2 = _gn_arith(ys[2], G, g2, e2)
        s = n3 + h2
        xb, exb = relu(s), e3n + eh2 + U * s.abs()
        h4, eh4 = _gn_arith(ys[3], G, g4, e4)
        g5, eg5 = _gn_arith(ys[4], G, g5, e5)
        for key, v, d, w, b in (("yb", h1, eh1, w2, b2), ("yc", xb, exb, w4, b4), ("ye", h4, eh4, w5, b5)):
            y = conv(v, w, b)
            out[key] = (y, _out_round(y, _conv_err(v, d, w, b, 9 * C, mode), mode))
        o = relu(xb + g5)
        out["out"] = (o, exb + eg5 + U * (xb + g5).abs())
    return {k: (w, torch.nan_to_num(b, nan=float("inf"))) for k, (w, b) in out.items()}
