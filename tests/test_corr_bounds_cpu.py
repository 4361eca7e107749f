"""CPU: the per-element correlation checks of oracle/corr_bounds.py pass on an fp32/fp16 emulation of the kernels' chain
and fail for each named defect (corr_bounds.MUTANTS) that a kernel or corr.py could have."""
import pytest
import torch

from oracle import corr_bounds as cb

R = 4
SHAPES = [(1, 24, 2, 20, 23), (2, 13, 1, 21, 21), (1, 40, 2, 9, 34)]      # (B, D, H, W1, W2): odd level widths, W1 = W2


def _inputs(shape, n_lookups, seed):
    B, D, H, W1, W2 = shape
    gen = torch.Generator().manual_seed(seed)
    f1 = torch.randn(B, D, H, W1, generator=gen)
    f2 = torch.randn(B, D, H, W2, generator=gen)
    grid = torch.arange(W1, dtype=torch.float32).view(1, 1, W1).expand(B, H, W1)
    coords = [grid + 6.0 * torch.randn(B, H, W1, generator=gen) for _ in range(n_lookups)]
    gs = [torch.randn(B, 4 * (2 * R + 1), H, W1, generator=gen) for _ in range(n_lookups)]
    g = torch.randn(B, H, W1, W2, generator=gen)
    return f1, f2, coords, gs, g


def _all_checks(shape, mutant, seed=0):
    """Every check of corr_bounds on the emulation of `shape` with `mutant` (None: the kernels' chain)."""
    f1, f2, coords, gs, g = _inputs(shape, 3, seed)
    lv, outs, d1, d2 = cb.emulate_block(f1, f2, coords, gs, 4, R, mutant)
    res = [cb.check_level0("fp32 level 0", lv[0], f1, f2, torch.float32), cb.check_pooled("fp32 pooled", lv)]
    lv64, E = cb.level_errors(f1.double(), f2.double(), 4)
    res += [cb.check_block_forward(f"block out {k}", o, lv, lv64, E, c, R) for k, (o, c) in enumerate(zip(outs, coords))]
    (r1, b1), (r2, b2) = cb.block_grad_reference(f1, f2, coords, gs, 4, R)
    res += [cb.check_bound("block dF1", d1, r1, b1), cb.check_bound("block dF2", d2, r2, b2)]
    for dt in (torch.float32, torch.float16):
        a1, a2, gg = f1.to(dt), f2.to(dt), g.to(dt)
        e1, e2 = cb.emulate_build_backward(a1, a2, gg, dt, mutant)
        res += list(cb.check_build_backward(f"build backward {dt}", e1, e2, a1, a2, gg, dt))
    h1, h2 = f1.half(), f2.half()
    lvh = cb.emulate_pyramid(h1, h2, 4, torch.float16, mutant)
    res += [cb.check_level0("fp16 level 0", lvh[0], h1, h2, torch.float16), cb.check_pooled("fp16 pooled", lvh)]
    return res


@pytest.mark.parametrize("shape", SHAPES, ids=str)
def test_emulation_passes_every_check(shape):
    res = _all_checks(shape, None)
    for c in res:
        print(c.name, c.worst, c.info)
        c.require()
    # fp16 intervals are mostly a single value, so the check is bit-exact there
    assert all(c.info["wide"] < 0.2 for c in res if c.name.startswith(("fp16 level 0", "build backward torch.float16")))


def test_emulation_one_level_loss_and_two_levels():
    f1, f2, coords, gs, _ = _inputs((1, 24, 2, 20, 23), 3, 1)
    g2 = torch.randn(1, 2, 20, 23 >> 2, generator=torch.Generator().manual_seed(2))
    _, _, d1, d2 = cb.emulate_block(f1, f2, [], [g2], 4, R, only_level=2)
    (r1, b1), (r2, b2) = cb.block_grad_reference(f1, f2, [], [g2], 4, R, only_level=2)
    cb.check_bound("dF1", d1, r1, b1).require()
    cb.check_bound("dF2", d2, r2, b2).require()
    gs2 = [g[:, :2 * (2 * R + 1)] for g in gs]
    lv, outs, d1, d2 = cb.emulate_block(f1, f2, coords, gs2, 2, R)
    lv64, E = cb.level_errors(f1.double(), f2.double(), 2)
    for o, c in zip(outs, coords):
        cb.check_block_forward("out", o, lv, lv64, E, c, R).require()
    (r1, b1), (r2, b2) = cb.block_grad_reference(f1, f2, coords, gs2, 2, R)
    cb.check_bound("dF1", d1, r1, b1).require()
    cb.check_bound("dF2", d2, r2, b2).require()


def test_zero_row_is_exactly_zero():
    f1, f2, *_ = _inputs((1, 24, 2, 20, 23), 0, 3)
    f2[:, :, 1, 5] = 0
    lv = cb.emulate_pyramid(f1, f2, 1, torch.float32)
    assert bool((lv[0][:, 1, :, 5] == 0).all())
    cb.check_level0("level 0", lv[0], f1, f2, torch.float32).require()


@pytest.mark.parametrize("mutant", sorted(cb.MUTANTS))
def test_every_mutant_fails_a_check(mutant):
    shapes = [s for s in SHAPES if mutant != "g_transposed" or s[3] == s[4]]
    for shape in shapes:
        failed = [c.name for c in _all_checks(shape, mutant) if not c.ok]
        print(mutant, shape, failed)
        assert failed, (mutant, shape)
