"""Independent fp64 torch restatement of the RAFT update block (reference core/update.py, BasicMultiUpdateBlock with one
GRU layer, and the iteration loop of core/raft_stereo_human.py's FlowUpdateModule.forward), a CPU emulation of the fp16
autocast route of csrc/update_block.cu, and per-element bounds for it (TEST INFRASTRUCTURE ONLY).

Params are in gps_gaussian_b200.update.params_of order.  One iteration, flow = coords1 - coords0:
  cor = relu(convc2(relu(convc1(corr))))   flo = relu(convf2(relu(convf1(flow))))
  x = [relu(conv([cor, flo])), flow]       z = sigmoid(convz([h, x]) + cz)   r = sigmoid(convr([h, x]) + cr)
  q = tanh(convq([r h, x]) + cq)           h' = (1 - z) h + z q
  delta = conv2(relu(conv1(h')))           mask = .25 mask2(relu(mask0(h')))   coords1' = coords1 + [delta_x, 0]

`iteration64` / `loop64` evaluate this in fp64 (`loop64` with the CorrBlock1D lookup and the convex upsampling restated;
the lookup's result is rounded to fp32 as CorrBlock1D's `.float()` does).

The fp16 route rounds at fixed points (include/gpsg.h): operands, weights and biases to fp16, each convolution's fp32
sum to fp16 and then the bias add to fp16, every elementwise op's result to fp16.  Given a stage's fp16 inputs, its
result is therefore a monotone function f of the exact fp64 convolution sums v, and the only freedom the kernels have
is the fp32 accumulation error e of v.  `stage_checks` gives, per element, want = f(v) and the bound
max |f(v +- e) - f(v)|: zero wherever e cannot move a rounding, one fp16 step where it can.  `emulate` chains the same
stages on the CPU; its `mutant` argument swaps in one deliberate error so the tests can show that each breaks a check.
MUTANTS are rounding and formula mistakes.  INDEX_MUTANTS have the shape of the bugs a persistent tiled GEMM tends to
have (tiles of 2 rows x 64 columns of one sample, csrc/update_block.cu): a halo line of every tile read as zero
(`seam_column_zero`: the column left and right of each 64-column tile, `halo_row_below_zero`: the row below each 2-row
tile, both in every 3x3 GEMM convolution), convf1's 7x7 window clipped to 5x5, cz / cr / cq of sample b read at the
packed stride 288 H W from the start of a wider context (`czrq_packed_stride`), two carried-state mistakes that need
the previous iteration (`emulate(..., prev=)`): the GRU reading that iteration's hidden state (`h_stale`) and x's flow
channels from its coords (`x_flow_stale`), and mask[2]'s N-block nb written at channel offset ((nb + 1) mod 3) 192
(`mask_nblock_offset`).  Each moves some element by far more than the ACC K sum|a w| envelope at B = 2, H = 5,
W = 130 (tests/test_update_cpu.py); none slips under it.
"""
import torch
import torch.nn.functional as F

from oracle.encoder_torch64 import F64, conv, ratio, relu  # noqa: F401  (ratio is part of this module's interface)

HID = 96
KEYS = ("cf1", "cf2", "x", "z", "rh", "h", "fh1", "m1", "delta", "mask", "coords1")
MUTANTS = ("flow_unrounded", "bias_fp32", "sigmoid_unrounded_sum", "delta_y_kept", "mask_unscaled", "z_r_swapped")
INDEX_MUTANTS = ("seam_column_zero", "halo_row_below_zero", "convf1_5x5", "czrq_packed_stride", "h_stale",
                 "x_flow_stale", "mask_nblock_offset")
TILE_H, TILE_W = 2, 64
MASK_NB = 192         # mask[2]'s N-block: 576 channels in three
# fp32 accumulation of K products on the tensor cores: 4 K units of 2^-24 of sum |a w| (room for the truncating adds)
ACC = 2.0 ** -22
# expf / tanhf in fp32 before the fp16 rounding: a few fp32 ulps
SFU = 2.0 ** -20


def r16(x):
    """x rounded to fp16 (to nearest even), in fp64."""
    return x.to(torch.float32).to(torch.float16).to(F64)


def grid(B, H, W, device="cpu"):
    """coords0 [B,2,H,W]: x then y, as the reference's coords_grid."""
    ys, xs = torch.meshgrid(torch.arange(H, dtype=F64, device=device), torch.arange(W, dtype=F64, device=device),
                            indexing="ij")
    return torch.stack([xs, ys])[None].repeat(B, 1, 1, 1)


def _split(ps):
    ps = [p.to(F64) for p in ps]
    return [(ps[2 * i], ps[2 * i + 1]) for i in range(12)]


# ---- fp64 restatement ----------------------------------------------------------------------------------------------

def iteration64(params, corr, flow, h, cz, cr, cq):
    """One update-block iteration in fp64: dict(x, z, r, h, delta, mask)."""
    (c1, c2, f1, f2, cv, cwz, cwr, cwq, fh1, fh2, m0, m2) = _split(params)
    corr, flow, h, cz, cr, cq = (t.to(F64) for t in (corr, flow, h, cz, cr, cq))
    cor = relu(conv(relu(conv(corr, *c1)), *c2))
    flo = relu(conv(relu(conv(flow, *f1)), *f2))
    x = torch.cat([relu(conv(torch.cat([cor, flo], 1), *cv)), flow], 1)
    hx = torch.cat([h, x], 1)
    z = torch.sigmoid(conv(hx, *cwz) + cz)
    r = torch.sigmoid(conv(hx, *cwr) + cr)
    q = torch.tanh(conv(torch.cat([r * h, x], 1), *cwq) + cq)
    h = (1 - z) * h + z * q
    delta = conv(relu(conv(h, *fh1)), *fh2)
    mask = .25 * conv(relu(conv(h, *m0)), *m2)
    return dict(x=x, z=z, r=r, h=h, delta=delta, mask=mask)


def corr_pyramid64(fmap1, fmap2, levels=4):
    """CorrBlock1D's volume and pyramid in fp64: level i [B*H*W1, W2 / 2^i]."""
    B, D, H, W1 = fmap1.shape
    vol = torch.einsum("bdhw,bdhv->bhwv", fmap1.to(F64), fmap2.to(F64)) / D ** 0.5
    pyr = [vol.reshape(B * H * W1, -1)]
    for _ in range(levels - 1):
        v = pyr[-1]
        pyr.append(0.5 * (v[:, 0:(v.shape[1] // 2) * 2:2] + v[:, 1:(v.shape[1] // 2) * 2:2]))
    return pyr


def lookup64(pyr, coords1, radius=4):
    """CorrBlock1D.__call__ in fp64: linear interpolation in x at coords_x / 2^i + d, d = -r .. r, zero outside."""
    B, _, H, W = coords1.shape
    x = coords1[:, 0].to(F64).reshape(-1, 1)
    out = []
    for i, v in enumerate(pyr):
        n = v.shape[1]
        pos = x / 2 ** i + torch.arange(-radius, radius + 1, dtype=F64, device=x.device).view(1, -1)
        x0 = torch.floor(pos)
        a = pos - x0
        def tap(ix):
            ok = (ix >= 0) & (ix <= n - 1)
            return torch.where(ok, torch.gather(v, 1, ix.clamp(0, n - 1).long()), torch.zeros_like(pos))
        out.append((1 - a) * tap(x0) + a * tap(x0 + 1))
    return torch.cat(out, 1).view(B, H, W, -1).permute(0, 3, 1, 2)


def upsample64(flow, mask, factor=8):
    """FlowUpdateModule.upsample_flow in fp64."""
    N, D, H, W = flow.shape
    m = torch.softmax(mask.to(F64).view(N, 1, 9, factor, factor, H, W), dim=2)
    up = F.unfold(factor * flow.to(F64), [3, 3], padding=1).view(N, D, 9, 1, 1, H, W)
    up = torch.sum(m * up, dim=2).permute(0, 1, 4, 2, 5, 3)
    return up.reshape(N, D, factor * H, factor * W)


def loop64(params, fmap1, fmap2, net, czrq, iters, flow_init=None, test_mode=True):
    """FlowUpdateModule.forward in fp64 with the "reg" corr block: flow_up [B,1,8H,8W] in test mode, else the list."""
    B, _, H, W = net.shape
    pyr = corr_pyramid64(fmap1, fmap2)
    coords0 = grid(B, H, W, net.device)
    coords1 = coords0.clone() if flow_init is None else coords0 + flow_init.to(F64)
    h = net.to(F64)
    cz, cr, cq = czrq.to(F64).split(HID, 1)
    preds = []
    for itr in range(iters):
        corr = lookup64(pyr, coords1).to(torch.float32).to(F64)     # CorrBlock1D returns its lookup as fp32
        o = iteration64(params, corr, coords1 - coords0, h, cz, cr, cq)
        h = o["h"]
        d = o["delta"].clone()
        d[:, 1] = 0
        coords1 = coords1 + d
        if test_mode and itr < iters - 1:
            continue
        preds.append(upsample64(coords1 - coords0, o["mask"])[:, :1])
    return preds[-1] if test_mode else preds


# ---- the fp16 route: stages as monotone functions of the exact sums ----------------------------------------------------

def _sum(a, w, pad=None, mutant=None):
    """(v, e): the exact fp64 sum conv(a, w) of fp16-exact operands and the kernels' accumulation error bound.  The tile
    mutants replace v of a 3x3 convolution by `_halo_dropped`'s."""
    K = w[0].numel()
    v = conv(a, w, pad=pad)
    if mutant in ("seam_column_zero", "halo_row_below_zero") and w.shape[-1] == 3:
        v = _halo_dropped(a, w, mutant)
    return v, ACC * K * conv(a.abs(), w.abs(), pad=pad)


def _halo_dropped(a, w, mutant):
    """The 3x3 zero-padded conv(a, w) computed tile by tile with one halo line of each tile read as zero: the columns
    left and right of every TILE_W-column tile, or the row below every TILE_H-row tile."""
    B, _, H, W = a.shape
    ap = F.pad(a, (1, 1, 1, 1))
    out = torch.empty(B, w.shape[0], H, W, dtype=a.dtype, device=a.device)
    if mutant == "seam_column_zero":
        for x0 in range(0, W, TILE_W):
            s = ap[..., x0:x0 + TILE_W + 2].clone()
            s[..., 0] = 0
            s[..., -1] = 0
            out[..., x0:x0 + TILE_W] = conv(s, w, pad=0)
    else:
        for y0 in range(0, H, TILE_H):
            s = ap[:, :, y0:y0 + TILE_H + 2].clone()
            if s.shape[2] == TILE_H + 2:
                s[:, :, -1] = 0
            out[:, :, y0:y0 + TILE_H] = conv(s, w, pad=0)
    return out


def _envelope(f, v, e):
    """want = f(v) and the bound max |f(v +- e) - f(v)| of a monotone f."""
    want = f(v)
    hi, lo = f(v + e), f(v - e)
    bnd = torch.maximum((hi - want).abs(), (lo - want).abs())
    return want, torch.where(torch.isnan(bnd), torch.zeros_like(bnd), bnd)


def _conv_out(b, bias_fp32=False):
    """the convolution output after cuDNN's rounding and the bias add: r16(r16(v) + b16)."""
    bb = b.view(1, -1, 1, 1) if bias_fp32 else r16(b).view(1, -1, 1, 1)
    return lambda v: r16(r16(v) + bb)


def _sig(x, s):
    return r16(torch.sigmoid(x) * (1 + s))


def _tanh(x, s):
    return r16(torch.tanh(x) * (1 + s))


def _sfu(fn, v, e):
    """want and bound of fn(v, s) with fn monotone in v and in the fp32-evaluation slack s."""
    want = fn(v, 0.0)
    hi, lo = fn(v + e, SFU), fn(v - e, -SFU)
    hi2, lo2 = fn(v + e, -SFU), fn(v - e, SFU)
    bnd = torch.stack([(t - want).abs() for t in (hi, lo, hi2, lo2)]).amax(0)
    return want, torch.where(torch.isnan(bnd), torch.zeros_like(bnd), bnd)


def stages(params, inp, mutant=None):
    """Every stage of one iteration from its own fp16 inputs in `inp` (h_in, corr, coords1_in, czrq and the stored
    cf1, cf2, x, z, rh, h, fh1, m1, delta): {key: (want, bound)}.  `mutant` in MUTANTS or INDEX_MUTANTS injects one
    error; h_stale and x_flow_stale read inp's h_stale / coords1_stale."""
    assert mutant is None or mutant in MUTANTS + INDEX_MUTANTS, mutant
    W = [(r16(w.to(inp["h_in"].device)), b.to(inp["h_in"].device)) for w, b in _split(params)]
    (c1, c2, f1, f2, cv, cwz, cwr, cwq, fh1, fh2, m0, m2) = W
    B, _, H, Wd = inp["coords1_in"].shape
    if mutant == "czrq_packed_stride":
        c = inp["czrq"]
        inp = {**inp, "czrq": torch.as_strided(c, c.shape, (3 * HID * H * Wd, H * Wd, Wd, 1), c.storage_offset())}
    if mutant == "convf1_5x5":
        f1 = (f1[0].clone(), f1[1])
        f1[0][..., (0, 6), :] = 0
        f1[0][..., :, (0, 6)] = 0
    g = {k: v.to(F64) if torch.is_tensor(v) else v for k, v in inp.items()}
    S = lambda a, w, pad=None: _sum(a, w, pad, mutant)
    bf = mutant == "bias_fp32"
    out = {}
    # motion encoder: convc1 on the fp16 corr, convf1 on the fp16 flow
    dev = g["coords1_in"].device
    flow32 = (g["coords1_in"].to(torch.float32) - grid(B, H, Wd, dev).to(torch.float32)).to(F64)
    flow = flow32 if mutant == "flow_unrounded" else r16(flow32)
    relu_out = lambda b: (lambda v: relu(_conv_out(b, bf)(v)))
    a = _envelope(relu_out(c1[1]), *S(r16(g["corr"]), c1[0]))
    b = _envelope(relu_out(f1[1]), *S(flow, f1[0]))
    out["cf1"] = (torch.cat([a[0], b[0]], 1), torch.cat([a[1], b[1]], 1))
    cf1 = g["cf1"]
    a = _envelope(relu_out(c2[1]), *S(cf1[:, :64], c2[0]))
    b = _envelope(relu_out(f2[1]), *S(cf1[:, 64:], f2[0]))
    out["cf2"] = (torch.cat([a[0], b[0]], 1), torch.cat([a[1], b[1]], 1))
    a = _envelope(relu_out(cv[1]), *S(g["cf2"], cv[0]))
    xf = flow
    if mutant == "x_flow_stale":
        xf = r16((g["coords1_stale"].to(torch.float32) - grid(B, H, Wd, dev).to(torch.float32)).to(F64))
    out["x"] = (torch.cat([a[0], xf], 1), torch.cat([a[1], torch.zeros_like(flow)], 1))
    # GRU
    h, x = g["h_stale" if mutant == "h_stale" else "h_in"], g["x"]
    cz, cr, cq = g["czrq"].split(HID, 1)
    hx = torch.cat([h, x], 1)
    if mutant == "z_r_swapped":
        cwz, cwr = cwr, cwz
    pre = lambda b, c: (lambda v: r16(_conv_out(b, bf)(v) + c))
    if mutant == "sigmoid_unrounded_sum":
        pre = lambda b, c: (lambda v: _conv_out(b, bf)(v) + c)
    vz, ez = S(hx, cwz[0])
    vr, er = S(hx, cwr[0])
    out["z"] = _sfu(lambda v, s: _sig(pre(cwz[1], cz)(v), s), vz, ez)
    out["rh"] = _sfu(lambda v, s: r16(_sig(pre(cwr[1], cr)(v), s) * h), vr, er)
    # rh is monotone in v with the sign of h: the envelope's max over both ends holds either way
    vq, eq = S(torch.cat([g["rh"], x], 1), cwq[0])
    z = g["z"]
    upd = lambda v, s: r16(r16(r16(1 - z) * h) + r16(z * _tanh(pre(cwq[1], cq)(v), s)))
    out["h"] = _sfu(upd, vq, eq)
    # heads from the new h
    out["fh1"] = _envelope(relu_out(fh1[1]), *S(g["h"], fh1[0]))
    out["m1"] = _envelope(relu_out(m0[1]), *S(g["h"], m0[0]))
    out["delta"] = _envelope(_conv_out(fh2[1], bf), *S(g["fh1"], fh2[0]))
    scale = 1.0 if mutant == "mask_unscaled" else .25
    out["mask"] = _envelope(lambda v: r16(scale * _conv_out(m2[1], bf)(v)), *S(g["m1"], m2[0], pad=0))
    if mutant == "mask_nblock_offset":
        out["mask"] = tuple(t.roll(MASK_NB, 1) for t in out["mask"])
    d = g["delta"].clone()
    if mutant != "delta_y_kept":
        d[:, 1] = 0
    c = (g["coords1_in"].to(torch.float32) + d.to(torch.float32)).to(F64)
    out["coords1"] = (c, torch.zeros_like(c))
    return out


def emulate(params, corr, coords1, net, czrq, mutant=None, prev=None):
    """One iteration of the fp16 route on the CPU, each stage from the previous stages' emulated outputs: a dict with
    the inputs (h_in, corr, coords1_in, czrq) and every key of KEYS.  `mutant` in MUTANTS or INDEX_MUTANTS injects one
    error; prev, the previous iteration's emulate() dict, holds the stale state h_stale and x_flow_stale read."""
    g = dict(h_in=net.to(F64), corr=corr.to(F64), coords1_in=coords1.to(F64), czrq=czrq.to(F64))
    if prev is not None:
        g.update(h_stale=prev["h_in"], coords1_stale=prev["coords1_in"])
    order = ("cf1", "cf2", "x", "z", "rh", "h", "fh1", "m1", "delta", "mask", "coords1")
    for k in order:
        g[k] = _stage(params, g, k, mutant)
    return g


def _stage(params, g, key, mutant):
    """`stages(...)[key][0]` for the inputs present in g: the others are never read by that key."""
    fill = {}
    B, _, H, W = g["coords1_in"].shape
    shapes = dict(cf1=128, cf2=128, x=128, z=HID, rh=HID, h=HID, fh1=256, m1=256, delta=2)
    for k, c in shapes.items():
        if k not in g:
            fill[k] = torch.zeros(B, c, H, W, dtype=F64, device=g["coords1_in"].device)
    return stages(params, {**g, **fill}, mutant)[key][0]


def stage_checks(params, got):
    """{key: (want, bound)} of every stage from the kernels' own inputs to it (`got`: update.step_with_workspace's
    dict plus czrq); without the mask head's m1 in `got`, m1 and mask are not checked."""
    if "m1" in got:
        return stages(params, got)
    B, _, H, W = got["coords1_in"].shape
    m1 = torch.zeros(B, 256, H, W, dtype=F64, device=got["coords1_in"].device)
    out = stages(params, {**got, "m1": m1})
    return {k: v for k, v in out.items() if k not in ("m1", "mask")}
