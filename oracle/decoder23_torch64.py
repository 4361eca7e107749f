"""Independent fp64 torch restatement of the regressor's decoder3 and decoder2 (TEST INFRASTRUCTURE ONLY), a CPU
emulation of the TF32 arithmetic of csrc/decoder23.cu, and per-element error bounds for it.

Maths (reference lib/gs_parm_network.py with the stage-2 config; two core/extractor.py ResidualBlocks per stage), params
in gps_gaussian_b200.decoder.deep_params_of order.  A stage is named by STAGES:
  "d3": v = cat(f_i, f_d) from img_feat3, depth_feat3 [B,96,H,W]; GroupNorm(12, 96)
  "d2": v = cat(up(s), f_i, f_d) from s [B,96,Hs,Ws] and img_feat2, depth_feat2 [B,48,2Hs,2Ws]; GroupNorm(8, 64);
        up the bilinear x2 of oracle/gs_head_torch64.py (align_corners=False)
and then, with GN the stage's GroupNorm:
  ya = conv3x3(v) + b;  yd = conv1x1(v) + b;  yb = conv3x3(relu(GN(ya))) + b;  xb = relu(GN(yd) + relu(GN(yb)))
  yc = conv3x3(xb) + b;  ye = conv3x3(relu(GN(yc))) + b;  out = relu(xb + relu(GN(ye)))
The terms are oracle/decoder1_torch64.py's with the group count as a parameter: encoder_torch64's convolution and
GroupNorm (im2col + matmul; GroupNorm from its definition) and error terms, gs_head_torch64's upsample and its bound.

`forward64` evaluates a stage in fp64.  `emulate` runs the kernels' arithmetic on the CPU in fp32 (the upsample in fp32
with torch's formula, every convolution operand rounded to TF32, exact products, fp32 sums in a random order, the bias
after the sum, GroupNorm with fp64 statistics, A and C rounded to fp32 and one fmaf); its `mutant` argument swaps in one
deliberate error (MUTANTS) so the tests can show that each breaks a check.  `bounds` chains the error terms from the
inputs to `out`; `stage_checks` bounds each stage from the kernels' stored input to that stage.
"""
import torch

from oracle.encoder_torch64 import _conv32, _conv_err, _gn32, _gn_arith, _gn_err, conv, group_norm, relu
from oracle.gs_head_torch64 import gamma, ratio, upsample2  # noqa: F401  (ratio is part of this module's interface)

F64 = torch.float64
U = 2.0 ** -24
STAGES = ("d3", "d2")
GROUPS = {"d3": 12, "d2": 8}
CHANNELS = {"d3": 96, "d2": 64}
RAW_KEYS = ("ya", "yd", "yb", "yc", "ye")
KEYS = RAW_KEYS + ("out",)
MUTANTS = ("upsample_phase", "concat_order", "downsample_relu", "unbiased_var", "residual_dropped", "relu_drops_nan",
           "wrong_groups")
# the group count a "wrong_groups" mutant uses: decoder3 with decoder2's GroupNorm(8) and decoder2 with 16 groups of 4
WRONG_GROUPS = {"d3": 8, "d2": 16}


def _split(ps):
    """(block 0: conv1 w, b, norm1 w, b, conv2 w, b, norm2 w, b, down w, b, norm3 w, b), (block 1: 8 tensors)"""
    return ps[:12], ps[12:]


def _v(stage, srcs, up=upsample2):
    if stage == "d3":
        return torch.cat(list(srcs), 1)
    s, f_i, f_d = srcs
    return torch.cat([up(s), f_i, f_d], 1)


def forward64(stage, srcs, params):
    """dict(ya, yd, yb, yc, ye, xb, out) in fp64: the five convolution outputs, block 0's output and the stage's.  srcs
    is (f_i, f_d) for "d3", (s, f_i, f_d) for "d2"."""
    G = GROUPS[stage]
    srcs = [t.to(F64) for t in srcs]
    ps = [p.to(F64) for p in params]
    (w1, b1, g1, be1, w2, b2, g2, be2, wd, bd, gd, bed), (w3, b3, g3, be3, w4, b4, g4, be4) = _split(ps)
    v = _v(stage, srcs)
    ya, yd = conv(v, w1, b1), conv(v, wd, bd)
    yb = conv(relu(group_norm(ya, G, g1, be1)), w2, b2)
    xb = relu(group_norm(yd, G, gd, bed) + relu(group_norm(yb, G, g2, be2)))
    yc = conv(xb, w3, b3)
    ye = conv(relu(group_norm(yc, G, g3, be3)), w4, b4)
    return dict(ya=ya, yd=yd, yb=yb, yc=yc, ye=ye, xb=xb, out=relu(xb + relu(group_norm(ye, G, g4, be4))))


def emulate(stage, srcs, params, seed=0, mutant=None):
    """The kernels' result on the CPU in fp32 (see the module docstring): the same keys as forward64; `mutant` in
    MUTANTS injects one error."""
    assert stage in STAGES and (mutant is None or mutant in MUTANTS), (stage, mutant)
    gen = torch.Generator().manual_seed(seed)
    srcs = [t.to(torch.float32).cpu() for t in srcs]
    ps = [p.to(torch.float32).cpu() for p in params]
    (w1, b1, g1, be1, w2, b2, g2, be2, wd, bd, gd, bed), (w3, b3, g3, be3, w4, b4, g4, be4) = _split(ps)
    G = WRONG_GROUPS[stage] if mutant == "wrong_groups" else GROUPS[stage]
    act = (lambda t: torch.fmax(t, torch.zeros_like(t))) if mutant == "relu_drops_nan" else relu
    if mutant == "concat_order":
        srcs = srcs[::-1] if stage == "d3" else [srcs[0], srcs[2], srcs[1]]
    v = _v(stage, srcs, up=lambda s: upsample2(s, align_corners=mutant == "upsample_phase"))
    gn = lambda y, g, b: _gn32(y, G, g, b, mutant)
    ya, yd = _conv32(v, w1, b1, gen, "tf32"), _conv32(v, wd, bd, gen, "tf32")
    yb = _conv32(act(gn(ya, g1, be1)), w2, b2, gen, "tf32")
    nd = gn(yd, gd, bed)
    if mutant == "downsample_relu":
        nd = act(nd)
    xb = act(nd + act(gn(yb, g2, be2)))
    yc = _conv32(xb, w3, b3, gen, "tf32")
    ye = _conv32(act(gn(yc, g3, be3)), w4, b4, gen, "tf32")
    g = act(gn(ye, g4, be4))
    out = act(g) if mutant == "residual_dropped" else act(xb + g)
    return dict(ya=ya, yd=yd, yb=yb, yc=yc, ye=ye, xb=xb, out=out)


def _input_err(stage, srcs):
    """v and the bound on the kernels' fp32 v: decoder2's upsample interpolation on its first 96 channels, exact
    elsewhere."""
    v = _v(stage, srcs)
    if stage == "d3":
        return v, torch.zeros_like(v)
    s, f_i, f_d = srcs
    return v, torch.cat([gamma(6) * upsample2(s.abs()), torch.zeros_like(f_i), torch.zeros_like(f_d)], 1)


def bounds(stage, srcs, params):
    """Per-element bounds dict(ya, yd, yb, yc, ye, out) on the kernels' results, chained from the inputs, fp64 on the
    inputs' device."""
    G, C = GROUPS[stage], CHANNELS[stage]
    srcs = [t.to(F64) for t in srcs]
    ps = [p.to(F64) for p in params]
    (w1, b1, g1, be1, w2, b2, g2, be2, wd, bd, gd, bed), (w3, b3, g3, be3, w4, b4, g4, be4) = _split(ps)
    cin = w1.shape[1]
    with torch.no_grad():
        v, d = _input_err(stage, srcs)
        ya, yd = conv(v, w1, b1), conv(v, wd, bd)
        ea, ed = _conv_err(v, d, w1, b1, 9 * cin, "tf32"), _conv_err(v, d, wd, bd, cin, "tf32")
        h1, eh1 = relu(group_norm(ya, G, g1, be1)), _gn_err(ya, ea, G, g1, be1, None)
        yb = conv(h1, w2, b2)
        eb = _conv_err(h1, eh1, w2, b2, 9 * C, "tf32")
        n2, en2 = relu(group_norm(yb, G, g2, be2)), _gn_err(yb, eb, G, g2, be2, None)
        nd, end = group_norm(yd, G, gd, bed), _gn_err(yd, ed, G, gd, bed, None)
        xb, exb = relu(nd + n2), end + en2 + U * (nd + n2).abs()
        yc = conv(xb, w3, b3)
        ec = _conv_err(xb, exb, w3, b3, 9 * C, "tf32")
        h3, eh3 = relu(group_norm(yc, G, g3, be3)), _gn_err(yc, ec, G, g3, be3, None)
        ye = conv(h3, w4, b4)
        ee = _conv_err(h3, eh3, w4, b4, 9 * C, "tf32")
        n4, en4 = relu(group_norm(ye, G, g4, be4)), _gn_err(ye, ee, G, g4, be4, None)
        out = dict(ya=ea, yd=ed, yb=eb, yc=ec, ye=ee, out=exb + en4 + U * (xb + n4).abs())
    return {k: torch.nan_to_num(t, nan=float("inf")) for k, t in out.items()}


def stage_checks(stage, srcs, params, raws):
    """{stage key: (want, bound)} for the kernels' stored convolution outputs raws = (ya, yd, yb, yc, ye) (fp32 or fp64
    NCHW) and their out: ya and yd from the inputs; yb from relu(GN(ya)); yc from relu(GN(yd) + relu(GN(yb))); ye from
    relu(GN(yc)); out from yd, yb and ye.  Each want is fp64 on the stored input, each bound covers that stage's own
    evaluation (the interpolation, operand rounding, fp32 sums, the GroupNorm / ReLU / residual arithmetic)."""
    G, C = GROUPS[stage], CHANNELS[stage]
    srcs = [t.to(F64) for t in srcs]
    ps = [p.to(F64) for p in params]
    yas, yds, ybs, ycs, yes = (r.to(F64).to(srcs[0].device) for r in raws)
    (w1, b1, g1, be1, w2, b2, g2, be2, wd, bd, gd, bed), (w3, b3, g3, be3, w4, b4, g4, be4) = _split(ps)
    cin = w1.shape[1]
    with torch.no_grad():
        v, d = _input_err(stage, srcs)
        out = {"ya": (conv(v, w1, b1), _conv_err(v, d, w1, b1, 9 * cin, "tf32")),
               "yd": (conv(v, wd, bd), _conv_err(v, d, wd, bd, cin, "tf32"))}
        h1, e1 = _gn_arith(yas, G, g1, be1)
        n2, e2 = _gn_arith(ybs, G, g2, be2)
        _, ed = _gn_arith(yds, G, gd, bed)                   # the same arithmetic without the ReLU (1-Lipschitz)
        nd = group_norm(yds, G, gd, bed)
        xb, exb = relu(nd + n2), ed + e2 + U * (nd + n2).abs()
        h3, e3 = _gn_arith(ycs, G, g3, be3)
        n4, e4 = _gn_arith(yes, G, g4, be4)
        for key, a, da, w, b in (("yb", h1, e1, w2, b2), ("yc", xb, exb, w3, b3), ("ye", h3, e3, w4, b4)):
            out[key] = (conv(a, w, b), _conv_err(a, da, w, b, 9 * C, "tf32"))
        out["out"] = (relu(xb + n4), exb + e4 + U * (xb + n4).abs())
    return {k: (w, torch.nan_to_num(b, nan=float("inf"))) for k, (w, b) in out.items()}
