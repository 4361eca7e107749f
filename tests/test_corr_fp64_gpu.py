"""GPU: the correlation volume build (forward and backward, both dtypes, every kernel) and stage 1's fp32 correlation
block against the fp64 restatement, per element, with the bounds derived in oracle/corr_bounds.py:

  * level 0 lies in [R(S - E), R(S + E)], R the dtype's rounding chain and E the accumulation bound of the kernel that
    ran (bit-exact where both ends round alike); every pooled level equals avg_pool2d of the device's own level below;
  * the build backward (C ABI) lies in the same kind of interval;
  * the fp32 block as stage 1 runs it (fp32 fmaps, 4 levels, r = 4, lookups at grid + N(0, 6^2)): every lookup output
    and dF1, dF2 within the derived bounds of fp64 autograd through the restatement (evaluated in fp64 on the device).

Every buffer corr.py allocates is filled with NaN before each launch, so an element no kernel writes shows.  Each case's
worst ratio (interval: |got - centre| / half-width; bound: err / bound) goes to $GPSG_PARITY_LOG."""
import ctypes as C
import types

import pytest
import torch

from helpers import record
from gps_gaussian_b200 import _lib, corr
from gps_gaussian_b200.corr import CorrBlockFast1D
from oracle import corr_bounds as cb

pytestmark = pytest.mark.gpu
R = 4


@pytest.fixture(autouse=True)
def poisoned_buffers(monkeypatch):
    """torch.empty / empty_like inside corr.py return NaN-filled tensors: the pyramid, the lookup output, the level
    gradients and the build backward's d1, d2."""
    def nan(fn):
        def make(*a, **k):
            t = fn(*a, **k)
            if t.is_floating_point():
                t.fill_(float("nan"))
            return t
        return make
    fake = types.SimpleNamespace(**{n: getattr(torch, n) for n in dir(torch) if not n.startswith("__")})
    fake.empty, fake.empty_like = nan(torch.empty), nan(torch.empty_like)
    monkeypatch.setattr(corr, "torch", fake)
    assert bool(corr.torch.empty(2, device="cuda").isnan().all())
    yield
    _lib.set_corr_build("wgmma")


def _tc_fwd(D, W1, W2):
    """corr_build_tc_supported for fresh (aligned) tensors: the wgmma build runs."""
    return (D >= 16 and D % 16 == 0 and W1 >= 8 and W1 % 8 == 0 and 16 <= W2 <= 128 and W2 % 16 == 0
            and max(D * 256 + D * W2 * 2, 128 * (W2 + 8) * 2) <= 200 * 1024)


def _tc_bwd(D, W1, W2):
    """corr_build_bwd_tc_supported for fresh tensors: the wgmma build backward runs."""
    def smem(K):
        kc = ((K + 15) & ~15) >> 3
        return max(kc * (2048 + D * 16), D * (128 + 8) * 2)
    return (16 <= D <= 256 and D % 16 == 0 and W1 >= 8 and W1 % 8 == 0 and 16 <= W2 <= 128 and W2 % 16 == 0
            and max(smem(W1), smem(W2)) <= 200 * 1024)


MODES = {"fp32": (torch.float32, "ffma"), "fp16-wgmma": (torch.float16, "wgmma"), "fp16-ffma": (torch.float16, "ffma")}
STAGE1, STAGE2 = (6, 96, 128, 128, 128), (2, 96, 128, 128, 128)
TC_SHAPES = [(1, 48, 3, 152, 112), (1, 16, 1, 8, 16), (1, 256, 1, 264, 64)]
SHAPES = [STAGE1, STAGE2, (1, 70, 3, 33, 150), (1, 40, 2, 300, 264), (1, 5, 1, 1, 7), (1, 1, 1, 1, 1)] + TC_SHAPES


def _cases():
    for mode in MODES:
        for s in SHAPES:
            if (s == STAGE1 and mode != "fp32") or (s == STAGE2 and mode == "fp32"):
                continue
            yield pytest.param(mode, s, id=f"{mode}-{'x'.join(map(str, s))}")


def _summary(tag, checks):
    for c in checks:
        print(f"{tag} {c.name}: worst {c.worst:.3g} {c.info}")
    worst = {c.name: c.worst for c in checks}
    shares = {c.name + " " + k: c.info[k] for c in checks for k in ("wide", "off") if k in c.info}
    record("corr_fp64:" + tag, **worst, **shares)
    for c in checks:
        c.require()


@pytest.mark.parametrize("mode,shape", list(_cases()))
def test_build_levels_vs_fp64(mode, shape):
    """Every level of 1-4 level pyramids: level 0 in its rounding interval, pooled levels bit-exact; one all-zero row
    of F2 gives exactly 0 in level 0."""
    dtype, kernel = MODES[mode]
    B, D, H, W1, W2 = shape
    wgmma = kernel == "wgmma" and _tc_fwd(D, W1, W2)
    if mode == "fp16-wgmma" and shape in TC_SHAPES + [STAGE2]:
        assert wgmma, shape
    gen = torch.Generator("cuda").manual_seed(sum(shape))
    f1 = torch.randn(B, D, H, W1, device="cuda", generator=gen).to(dtype)
    f2 = torch.randn(B, D, H, W2, device="cuda", generator=gen).to(dtype)
    yz = min(3, W2 - 1)
    f2[0, :, 0, yz] = 0
    _lib.set_corr_build(kernel)
    checks = []
    l0 = None
    for L in range(1, 5):
        lv = [v.detach().clone() for v in CorrBlockFast1D(f1, f2, num_levels=L, radius=R)._vols]
        torch.cuda.synchronize()
        assert [tuple(v.shape) for v in lv] == [(B, H, W1, W2 >> l) for l in range(L)]
        assert all(v.dtype == dtype for v in lv)
        assert bool((lv[0][0, 0, :, yz] == 0).all())
        if l0 is None:
            checks.append(cb.check_level0("level 0", lv[0], f1, f2, dtype, wgmma))
            l0 = lv[0]
        else:
            assert torch.equal(lv[0].view(-1).view(torch.int16 if dtype == torch.float16 else torch.int32),
                               l0.view(-1).view(torch.int16 if dtype == torch.float16 else torch.int32)), L
        checks.append(cb.check_pooled(f"L={L} pooled", lv))
    _summary(f"build:{mode}:{shape}", checks)


BWD_SHAPES = SHAPES + [(1, 130, 2, 150, 70)]


def _bwd_cases():
    for mode in MODES:
        for s in BWD_SHAPES:
            if (s == STAGE1 and mode != "fp32") or (s == STAGE2 and mode == "fp32"):
                continue
            yield pytest.param(mode, s, id=f"{mode}-{'x'.join(map(str, s))}")


@pytest.mark.parametrize("mode,shape", list(_bwd_cases()))
def test_build_backward_vs_fp64(mode, shape):
    """gpsg_corr_build_backward: dF1 = F2 g^T / sqrt(D), dF2 = F1 g / sqrt(D) in their rounding intervals (W1 != W2,
    D > 64 with a partial 64-row tile, W1 > 128, K padded to 16 on the tensor cores)."""
    dtype, kernel = MODES[mode]
    B, D, H, W1, W2 = shape
    wgmma = kernel == "wgmma" and _tc_bwd(D, W1, W2)
    if mode == "fp16-wgmma" and shape in [STAGE2, (1, 48, 3, 152, 112), (1, 16, 1, 8, 16)]:
        assert wgmma, shape
    gen = torch.Generator("cuda").manual_seed(sum(shape) + 1)
    f1 = torch.randn(B, D, H, W1, device="cuda", generator=gen).to(dtype)
    f2 = torch.randn(B, D, H, W2, device="cuda", generator=gen).to(dtype)
    g = torch.randn(B, H, W1, W2, device="cuda", generator=gen).to(dtype)
    d1, d2 = torch.full_like(f1, float("nan")), torch.full_like(f2, float("nan"))
    p = lambda t: C.c_void_p(t.data_ptr())
    _lib.set_corr_build(kernel)
    rc = _lib.lib.gpsg_corr_build_backward(*_lib.device_stream(f1.device), 0 if dtype == torch.float32 else 1,
                                           B, D, H, W1, W2, p(f1), p(f2), p(g), p(d1), p(d2))
    _lib.check(rc, "gpsg_corr_build_backward")
    torch.cuda.synchronize()
    _summary(f"build_backward:{mode}:{shape}", cb.check_build_backward("", d1, d2, f1, f2, g, dtype, wgmma))


# ---------------------------------------------------------------------------------------------------------------------
# the fp32 block as stage 1 runs it
# ---------------------------------------------------------------------------------------------------------------------
def _block_run(shape, n_lookups, seed, levels=4, only_level=None):
    """fp32 fmaps -> CorrBlockFast1D(levels, r=4) -> lookups at grid + N(0, 6^2) -> sum <out_k, G_k> -> backward."""
    B, D, H, W1, W2 = shape
    gen = torch.Generator("cuda").manual_seed(seed)
    f1 = torch.randn(B, D, H, W1, device="cuda", generator=gen).requires_grad_(True)
    f2 = torch.randn(B, D, H, W2, device="cuda", generator=gen).requires_grad_(True)
    blk = CorrBlockFast1D(f1, f2, num_levels=levels, radius=R)
    lv = [v.detach().clone() for v in blk._vols]
    grid = torch.arange(W1, device="cuda", dtype=torch.float32).view(1, 1, W1).expand(B, H, W1)
    ys = torch.arange(H, device="cuda", dtype=torch.float32).view(1, H, 1).expand(B, H, W1)
    outs, coords, gs = [], [], []
    if only_level is None:
        for _ in range(n_lookups):
            cx = grid + 6.0 * torch.randn(B, H, W1, device="cuda", generator=gen)
            outs.append(blk(torch.stack([cx, ys], 1).contiguous()))
            gs.append(torch.randn(outs[-1].shape, device="cuda", generator=gen))
            coords.append(cx)
        torch.autograd.backward(outs, gs)                   # d loss / d out_k = G_k exactly
    else:
        lvl = blk.corr_pyramid[only_level]
        g = torch.randn(lvl.shape, device="cuda", generator=gen)
        torch.autograd.backward([lvl], [g])
        gs.append(g.squeeze(3))
    torch.cuda.synchronize()
    return f1, f2, lv, [o.detach() for o in outs], coords, gs


BLOCKS = {
    "stage1": dict(shape=STAGE1, n_lookups=3),
    "ragged-N12": dict(shape=(2, 70, 3, 150, 97), n_lookups=12),
    "level2-only": dict(shape=(1, 64, 4, 96, 128), n_lookups=0, only_level=2),
    "levels2": dict(shape=(1, 48, 3, 72, 100), n_lookups=3, levels=2),
}


@pytest.mark.parametrize("case", list(BLOCKS))
def test_fp32_block_vs_fp64(case):
    kw = dict(BLOCKS[case])
    shape = kw.pop("shape")
    levels = kw.get("levels", 4)
    f1, f2, lv, outs, coords, gs = _block_run(shape, seed=sum(shape), **kw)
    checks = [cb.check_level0("level 0", lv[0], f1, f2, torch.float32), cb.check_pooled("pooled", lv)]
    lv64, E = cb.level_errors(f1.detach().double(), f2.detach().double(), levels)
    checks += [cb.check_block_forward(f"out {k}", o, lv, lv64, E, c, R) for k, (o, c) in enumerate(zip(outs, coords))]
    del lv64, E
    (r1, b1), (r2, b2) = cb.block_grad_reference(f1, f2, coords, gs, levels, R, kw.get("only_level"))
    checks += [cb.check_bound("dF1", f1.grad, r1, b1), cb.check_bound("dF2", f2.grad, r2, b2)]
    _summary(f"block:{case}", checks)


def test_fp32_block_is_reproducible():
    """Two runs of the stage-1 block: the same bits in every level, output and feature-map gradient."""
    runs = []
    for _ in range(2):
        f1, f2, lv, outs, _, _ = _block_run(STAGE1, 3, seed=5)
        runs.append(lv + outs + [f1.grad, f2.grad])
    for a, b in zip(*runs):
        assert torch.equal(a.view(torch.int32), b.view(torch.int32))
