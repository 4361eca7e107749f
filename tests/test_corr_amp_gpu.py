"""GPU: the correlation kernels against the fp64 restatement (oracle/corr_torch64.py), in fp16 (stage-2 AMP) and fp32.

Every device result is compared with the restatement evaluated on the exact inputs the device saw: its own pyramid
levels for the lookups, its own incoming gradients for the backwards, the fp16-quantised feature maps for the build.
Bounds are per element and follow from rounding:

  * lookup forward, fused and per-level: out = prev (1-dx) + cur dx in fp32, rounded once to the volume dtype
    (DESIGN.md section 2).  The fp32 arithmetic (1-dx, two products, one add) is within 2^-22 (|prev| + |cur|) of the
    fp64 value v, so fp32: |got - v| <= 2^-22 (|prev| + |cur|); fp16 adds half an fp16 ulp of v, and got == fp16(v)
    except where v lies within that fp32 error of an fp16 rounding boundary.  Double rounding, fp16 arithmetic or a
    wrong dx each break one of the two.
  * lookup backward: each level-gradient element is a dx + b (1-dx) of two incoming gradients, rounded once: the same
    bound with |a| + |b|.
  * the whole block in fp16 (build, three lookups, their backward, the fold of the pooled levels, the build backward):
    see test_fp16_block_fmap_grads_vs_fp64.
"""
import numpy as np
import pytest
import torch

import corr_sampler
from gps_gaussian_b200 import _lib
from gps_gaussian_b200.corr import CorrBlockFast1D, _LookupPyramid
from oracle import corr_torch64 as ct

pytestmark = pytest.mark.gpu
F64 = torch.float64
E32 = 2.0 ** -22
MISMATCH_MAX = 1e-3          # share of a test's fp16 results that may differ from fp16(v) (see check_bound)


def ulp16(v):
    """fp16 ulp at v (fp64): 2^(e-10) for |v| in [2^e, 2^(e+1)), 2^-24 in the subnormal range."""
    _, e = torch.frexp(v)
    e = torch.where(v == 0, torch.full_like(e, -100), e) - 1
    return torch.exp2(e.clamp_min(-14).to(F64) - 10)


def fp16_rn(v):
    """v (fp64) rounded to the nearest fp16, ties to even, in one step (no detour through fp32)."""
    u = ulp16(v)
    return torch.round(v / u) * u


def same_bits(a, b):
    """Bit-for-bit equality (NaN rows included)."""
    it = {torch.float16: torch.int16, torch.float32: torch.int32}[a.dtype]
    return a.dtype == b.dtype and a.shape == b.shape and torch.equal(a.contiguous().view(it), b.contiguous().view(it))


def check_bound(name, got, v, mag, half, keep=None, tally=None):
    """|got - v| <= [1/2 ulp16(v)] + 2^-22 mag per element (rows outside `keep` excluded).  fp16: got == fp16(v) except
    where v lies within 2^-22 mag of a midpoint between two fp16 values, where the fp32 result may round either way;
    such elements are counted in `tally` [mismatches, elements], whose share the caller bounds over a whole test.
    Returns the worst ratio of error to bound."""
    got = got.detach().cpu().to(F64)
    assert got.shape == v.shape, (name, got.shape, v.shape)
    if keep is not None:
        got, v, mag = got[keep], v[keep], mag[keep]
    if got.numel() == 0:
        return 0.0
    err = (got - v).abs()
    bound = E32 * mag + (0.5 * ulp16(v) if half else 0.0)
    ratio = torch.where(err == 0, torch.zeros_like(err), err / bound)
    worst = float(ratio.max())
    msg = f"{name}: worst err/bound {worst:.3g}"
    if half:
        mis = got != fp16_rn(v)
        u = ulp16(v)
        to_mid = (0.5 - (v / u - torch.round(v / u)).abs()) * u            # distance from v to the nearest midpoint
        msg += f", {int(mis.sum())} of {mis.numel()} != fp16(v)"
        assert bool((to_mid[mis] <= E32 * mag[mis]).all()), msg + " away from a rounding midpoint"
        if tally is not None:
            tally[0] += int(mis.sum())
            tally[1] += mis.numel()
    print(msg)
    assert worst <= 1.0, msg
    return worst


# ------------------------------------------------------------------------------------------------------------------
# (a), (b): lookup forward and backward, fused and per level, over edge shapes and coordinates
# ------------------------------------------------------------------------------------------------------------------
def _edge_coords(W2, r, rng):
    """Level-0 x coordinates: for every level l, integers and .5 values of x / 2^l across [-r-1, W2_l + r] (windows
    cut off at either end), x / 2^l = W2_l - 1, -0.0, 1e6 and 1e10 either sign, and uniform values."""
    xs = []
    for l in range(4):
        w = W2 >> l
        u = np.arange(-r - 1, w + r + 0.5, 0.5)
        xs += list(u * 2 ** l) + [(w - 1) * 2 ** l]
    xs += [W2 - 1.0, -0.0, 1e6, -1e6, 1e10, -1e10, 3e9, -3e9]
    xs += list(rng.uniform(-2 * r - 4, W2 + 2 * r + 4, 64))
    return np.array(xs, np.float32)


def _layouts(cx, H, W1):
    """The same fp32 x values as [B,2,H,W1] (x channel passed as a view with its batch stride), channels-last, and
    fp64 (both copied to a contiguous fp32 plane before the launch)."""
    B = cx.shape[0]
    y = torch.arange(H, dtype=torch.float32).view(1, H, 1).expand(B, H, W1)
    c = torch.stack([cx, y], 1).cuda()
    return {"view": c, "channels_last": c.to(memory_format=torch.channels_last), "fp64": c.double()}


def _mags(levels, cx, r, g):
    """Per level, |prev| + |cur| of every lookup output and |a| + |b| of every level-gradient element: the forward and
    the backward (of |g|) at the integer coordinates floor(x / 2^l) and floor(x / 2^l) + 1, where dx = 0."""
    rd = 2 * r + 1
    fwd, bwd = [], []
    for l, v in enumerate(levels):
        fl = torch.floor(cx.to(F64) / 2 ** l)
        leaf = torch.zeros(v.shape, dtype=F64, requires_grad=True)
        gl = g[:, l * rd:(l + 1) * rd].abs()
        fwd.append(ct.sample(v.abs(), fl, r) + ct.sample(v.abs(), fl + 1, r))
        bwd.append(sum(torch.autograd.grad(ct.sample(leaf, x, r), leaf, gl)[0] for x in (fl, fl + 1)))
    return torch.cat(fwd, 1), bwd


@pytest.mark.parametrize("dtype", [torch.float16, torch.float32], ids=["fp16", "fp32"])
@pytest.mark.parametrize("W2", [128, 150, 17, 8, 7])
@pytest.mark.parametrize("r", [0, 1, 4, 6])
def test_lookup_fwd_bwd_vs_fp64(dtype, W2, r):
    """Fused 1-4 level lookup and the per-level drop-in sampler, forward and backward, against the restatement on the
    device's own levels and incoming gradients.  NaN / inf coordinates in a few pixels: only their own rows are
    exempt."""
    half = dtype == torch.float16
    rng = np.random.default_rng(1000 * W2 + r)
    gen = torch.Generator("cuda").manual_seed(W2 + r)
    xs = _edge_coords(W2, r, rng)
    B, H = 2, 3
    W1 = -(-len(xs) // (B * H))
    W1 += W1 == W2
    cx = np.concatenate([xs, rng.uniform(-8, W2 + 8, B * H * W1 - len(xs)).astype(np.float32)])
    rng.shuffle(cx)
    bad = rng.choice(B * H * W1, 3, replace=False)
    cx[bad] = [np.nan, np.inf, -np.inf]
    keep = torch.from_numpy(np.isfinite(cx).reshape(B, H, W1))
    cx = torch.from_numpy(cx.reshape(B, H, W1))
    coords = _layouts(cx, H, W1)

    # the device's pyramid, built from fp16/fp32 feature maps
    f1 = torch.randn(B, 16, H, W1, device="cuda", generator=gen).to(dtype)
    f2 = torch.randn(B, 16, H, W2, device="cuda", generator=gen).to(dtype)
    lv = [v.detach().clone() for v in CorrBlockFast1D(f1, f2, num_levels=4, radius=r)._vols]
    lv64 = [v.cpu().to(F64) for v in lv]
    rd = 2 * r + 1
    gout = torch.randn(B, 4 * rd, H, W1, device="cuda", generator=gen).to(dtype)
    g64 = gout.cpu().to(F64)

    v_fwd = ct.lookup(lv64, cx, r)                                              # [B, 4 rd, H, W1]
    v_bwd = ct.level_grads([v.shape for v in lv64], cx, r, g64)
    m_fwd, m_bwd = _mags(lv64, cx, r, g64)
    keep_out = keep.unsqueeze(1).expand(B, rd, H, W1)
    tally = [0, 0]

    for L in range(1, 5):
        outs, grads = {}, {}
        for name, c in coords.items():
            leaves = [v.clone().requires_grad_(True) for v in lv[:L]]
            out = _LookupPyramid.apply(c[:, :1], r, *leaves)
            assert out.dtype == dtype and out.shape == (B, L * rd, H, W1)
            outs[name] = out.detach()
            grads[name] = torch.autograd.grad(out, leaves, gout[:, :L * rd].contiguous())
        for name in ("channels_last", "fp64"):                                # copy path == view path, bit for bit
            assert same_bits(outs[name], outs["view"]), (name, L)
            assert all(same_bits(a, b) for a, b in zip(grads[name], grads["view"])), (name, L)
        for l in range(L):
            sl = slice(l * rd, (l + 1) * rd)
            check_bound(f"fused fwd {dtype} W2={W2} r={r} L={L} l={l}", outs["view"][:, sl], v_fwd[:, sl], m_fwd[:, sl],
                        half, keep_out, tally)
            check_bound(f"fused bwd {dtype} W2={W2} r={r} L={L} l={l}", grads["view"][l], v_bwd[l], m_bwd[l], half, keep,
                        tally)

    # per-level drop-in sampler (coords / 2^l is exact in fp32), and a strided volume view (row stride != W2)
    for l in range(4):
        sl = slice(l * rd, (l + 1) * rd)
        c = coords["view"] / 2 ** l
        out, = corr_sampler.forward(lv[l], c, r)
        check_bound(f"sampler fwd {dtype} W2={W2} r={r} l={l}", out, v_fwd[:, sl], m_fwd[:, sl], half, keep_out, tally)
        wide = torch.randn(B, H, 2 * W1, W2 >> l, device="cuda", generator=gen).to(dtype)
        wide[:, :, ::2] = lv[l]
        view = wide[:, :, ::2]
        assert not view.is_contiguous() or view.numel() == 0
        out_s, = corr_sampler.forward(view, c, r)
        assert same_bits(out_s, out)
        gv, = corr_sampler.backward(lv[l], c, gout[:, sl].contiguous(), r)
        check_bound(f"sampler bwd {dtype} W2={W2} r={r} l={l}", gv, v_bwd[l], m_bwd[l], half, keep, tally)
    if half:
        print(f"W2={W2} r={r}: {tally[0]} of {tally[1]} fp16 results != fp16(v)")
        assert tally[0] < MISMATCH_MAX * tally[1], tally


@pytest.mark.parametrize("dtype", [torch.float16, torch.float32], ids=["fp16", "fp32"])
def test_lookup_empty_batch(dtype):
    lv = [torch.zeros(0, 3, 5, 7 >> l, device="cuda", dtype=dtype, requires_grad=True) for l in range(4)]
    c = torch.zeros(0, 2, 3, 5, device="cuda")
    out = _LookupPyramid.apply(c[:, :1], 4, *lv)
    assert out.shape == (0, 36, 3, 5)
    g = torch.autograd.grad(out, lv, torch.zeros_like(out))
    assert [tuple(t.shape) for t in g] == [tuple(v.shape) for v in lv]
    out, = corr_sampler.forward(lv[0].detach(), c, 4)
    assert out.shape == (0, 9, 3, 5)
    gv, = corr_sampler.backward(lv[0].detach(), c, torch.zeros(0, 9, 3, 5, device="cuda", dtype=dtype), 4)
    assert gv.shape == (0, 3, 5, 7)


# ------------------------------------------------------------------------------------------------------------------
# (d): the whole block as stage 2 uses it, in fp16
# ------------------------------------------------------------------------------------------------------------------
# Per element, |got - ref| <= C_BLOCK (2^-11 A + 2^-25 (1 + Z)), A the contraction over absolute values:
# sum_y U |F2| / sqrt(D) for dF1, sum_x U |F1| / sqrt(D) for dF2, with U the level-0 gradient folded from unsigned terms
# (see _block_reference), and Z the same contraction with U = 1.  An fp16 rounding errs by at most 2^-11 relative, or
# 2^-25 absolute in the subnormal range (small pooled-level gradients, halved by the fold, can land there).  The
# fp16 roundings between the incoming gradients and dF: each lookup's backward rounds its level gradient once (1);
# autograd sums the three lookups' fp16 gradients (2 more); the fold adds each pooled level's gradient into the level
# below in fp16 (3 more for level 0; the halving is exact); the build backward accumulates in fp32 (error near
# 2^-24 sqrt(K), negligible) and rounds once (1).  Each rounding is at most 2^-11 relative to what it rounds, so
# C_BLOCK = 7.  On an H100 the worst measured error is 0.2 of this bound (dF2, W2=160), 0.13 at the stage-2 shape.
C_BLOCK = 7


def _block_case(shape, n_lookups, seed, only_level=None):
    B, D, H, W1, W2 = shape
    gen = torch.Generator("cuda").manual_seed(seed)
    f1 = torch.randn(B, D, H, W1, device="cuda", generator=gen).half().requires_grad_(True)
    f2 = torch.randn(B, D, H, W2, device="cuda", generator=gen).half().requires_grad_(True)
    blk = CorrBlockFast1D(f1, f2, num_levels=4, radius=4)
    grid = torch.arange(W1, device="cuda", dtype=torch.float32).view(1, 1, W1).expand(B, H, W1)
    ys = torch.arange(H, device="cuda", dtype=torch.float32).view(1, H, 1).expand(B, H, W1)
    coords, gs = [], []
    loss = 0
    if only_level is None:
        for k in range(n_lookups):                                  # grid + N(0, 6^2): some windows leave the row
            cx = grid + 6.0 * torch.randn(B, H, W1, device="cuda", generator=gen)
            c = torch.stack([cx, ys], 1).contiguous()
            out = blk(c)
            g = torch.randn(out.shape, device="cuda", generator=gen).half()
            loss = loss + (out.float() * g.float()).sum()          # d loss / d out = g exactly, no fp16 overflow
            coords.append(cx.cpu())
            gs.append(g.cpu().to(F64))
    else:
        lvl = blk.corr_pyramid[only_level]
        g = torch.randn(lvl.shape, device="cuda", generator=gen).half()
        loss = (lvl.float() * g.float()).sum()
        gs.append(g.cpu().to(F64).squeeze(3))
    loss.backward()
    torch.cuda.synchronize()
    return f1, f2, coords, gs


def _block_reference(f1, f2, coords, gs, only_level=None):
    """fp64 autograd through the restatement on the quantised fmaps, and the contractions A over the unsigned level-0
    gradient U: the fold of every lookup's level gradients taken with |G_k| and the weights dx, 1-dx.  U bounds every
    partial sum the fp16 chain rounds; |G| does not where the lookups' or levels' terms cancel."""
    a1 = f1.detach().cpu().to(F64).requires_grad_(True)
    a2 = f2.detach().cpu().to(F64).requires_grad_(True)
    lv = ct.pyramid(a1, a2, 4)
    if only_level is None:
        loss = sum((ct.lookup(lv, c, 4) * g).sum() for c, g in zip(coords, gs))
        grads = [0] * 4
        for c, g in zip(coords, gs):
            gl = ct.level_grads([v.shape for v in lv], c, 4, g.abs())
            grads = [x + y for x, y in zip(grads, gl)]
    else:
        loss = (lv[only_level] * gs[0]).sum()
        grads = [gs[0].abs() if l == only_level else None for l in range(4)]
    d1, d2 = torch.autograd.grad(loss, (a1, a2))
    G = ct.fold(grads, a2.shape[3])
    div = ct.sqrt_d(a1.shape[1])
    A1 = torch.einsum("bhxy,bdhy->bdhx", G, a2.detach().abs()) / div
    A2 = torch.einsum("bhxy,bdhx->bdhy", G, a1.detach().abs()) / div
    Z1 = a2.detach().abs().sum(3, keepdim=True) / div                   # the same contractions with every |U| = 1
    Z2 = a1.detach().abs().sum(3, keepdim=True) / div
    return (d1, A1, Z1), (d2, A2, Z2)


def _check_block(name, f1, f2, refs):
    worst = 0.0
    for which, got, (ref, A, Z) in (("dF1", f1.grad, refs[0]), ("dF2", f2.grad, refs[1])):
        assert got is not None and got.dtype == torch.float16
        got = got.cpu().to(F64)
        assert bool(torch.isfinite(got).all())
        err = (got - ref).abs()
        bound = C_BLOCK * (2.0 ** -11 * A + 2.0 ** -25 * (1.0 + Z))
        r = err / bound
        i = int(r.argmax())
        ratio = float(r.flatten()[i])
        maxn = float(err.max()) / max(1.0, float(ref.abs().max()))
        print(f"{name} {which}: worst err/bound {ratio:.3g} (c = {C_BLOCK}; there got {float(got.flatten()[i]):.4g}, "
              f"ref {float(ref.flatten()[i]):.4g}, A {float(A.flatten()[i]):.3g}), max-normalised error {maxn:.3g}")
        assert ratio <= 1.0, (name, which, ratio)
        assert maxn < 4e-3, (name, which, maxn)
        worst = max(worst, ratio)
    return worst


@pytest.mark.parametrize("mode", ["wgmma", "ffma"])
@pytest.mark.parametrize("shape", [(4, 192, 128, 128, 128), (1, 48, 3, 72, 112), (2, 64, 4, 96, 160)],
                         ids=["stage2", "ragged", "W2=160"])
def test_fp16_block_fmap_grads_vs_fp64(mode, shape):
    """fp16 fmaps -> CorrBlockFast1D(4 levels, r=4) -> three lookups -> sum out_k G_k -> backward, against fp64
    autograd through the restatement.  stage2 is the training shape; W2=160 leaves the tensor-core build and its
    backward; ragged has W1 != W2 and partial tiles."""
    _lib.set_corr_build(mode)
    try:
        f1, f2, coords, gs = _block_case(shape, 3, seed=sum(shape))
    finally:
        _lib.set_corr_build("wgmma")
    _check_block(f"block {mode} {shape}", f1, f2, _block_reference(f1, f2, coords, gs))


@pytest.mark.parametrize("mode", ["wgmma", "ffma"])
def test_fp16_block_grad_on_one_level(mode):
    """A loss on corr_pyramid[2] alone: levels 0, 1 and 3 get no gradient (the None branches of the fold)."""
    shape = (1, 64, 4, 96, 128)
    _lib.set_corr_build(mode)
    try:
        f1, f2, coords, gs = _block_case(shape, 0, seed=77, only_level=2)
    finally:
        _lib.set_corr_build("wgmma")
    _check_block(f"level-2 loss {mode}", f1, f2, _block_reference(f1, f2, coords, gs, only_level=2))
