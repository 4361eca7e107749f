"""CPU: the fp64 backward of the regressor's full-resolution tail (oracle/gs_head_grad_torch64.backward64) against the
reference module's own autograd (tests/golden/gs_head_grad_golden.npz), the fp32 emulation of the backward kernels
against `grad_bounds`, and each mutant of the emulation against those bounds: every mutant must break a check that the
emulation passes."""
import pytest
import torch

import gs_head_cases as gc
import gs_head_grad_cases as gg
from oracle import gs_head_grad_torch64 as gt


def _same(got, want):
    """Equal to fp64 rounding where finite; NaN and inf exactly where the reference has them."""
    got = got.to(torch.float64).reshape(want.shape)
    if not torch.equal(torch.isnan(got), torch.isnan(want)):
        return False
    inf = torch.isinf(want)
    if not torch.equal(got[inf], want[inf]) or torch.isinf(got[~inf]).any():
        return False
    fin = torch.isfinite(want)
    scale = want[fin].abs().max() if fin.any() else torch.tensor(0.0, dtype=torch.float64)
    return bool(((got[fin] - want[fin]).abs() <= 1e-11 * want[fin].abs() + 1e-13 * scale).all())


@pytest.mark.parametrize("name", gg.GOLDEN_CASES)
def test_backward64_matches_golden(name):
    src, img, depth, ps, grads, want, finite, stride = gg.golden(name)
    got = gt.backward64(src, img, depth, ps, grads)
    for k in gg.GRAD_KEYS:
        assert torch.equal(torch.isfinite(got[k]), finite[k]), k
        assert _same(gg.pick(k, got[k], stride), want[k]), k
    if name == "nan_depth":
        assert torch.isnan(want["d_depth"]).any() and not finite["out_w"].any()
    if name == "inf_g_scale":
        assert not finite["scale_w2"].all() and not finite["scale_w1"].all()


def _all_cases():
    """Every case twice: as given, and with g_rot = 0.  normalize's gradient amplifies the forward error by 1 / ||pre||
    and the default init's rot pre-activations are small, so with g_rot the bounds of everything downstream are loose;
    without it they are tight enough for the mutants."""
    def both(cid, src, img, depth, ps, grads):
        yield cid, (src, img, depth, ps, grads)
        yield cid + "_no_rot", (src, img, depth, ps, [grads[0] * 0] + list(grads[1:]))
    for name in gg.GOLDEN_CASES:
        src, img, depth, ps, grads = gg.golden(name)[:5]
        yield from both("golden_" + name, src, img, depth, ps, grads)
    for case in gc.SWEEP:
        src, img, depth, ps = gc.inputs(case)
        yield from both(case.id, src, img, depth, ps, gg.upstream(case.B, case.H, case.W, case.seed))


CASES = dict(_all_cases())


def _worst(args, got):
    """Worst ratio per gradient end to end (fp64 on the emulation's mid), and of d_src against the fp64 adjoint of the
    emulation's own dcat (`d_src_stage`)."""
    want = gt.backward64(*args, mid=got["mid"])
    b = gt.grad_bounds(*args, got["mid"])
    worst = {k: gt.ratio(got[k], want[k], b[k]) for k in gg.GRAD_KEYS}
    worst["d_src_stage"] = gt.ratio(got["d_src"], *gt.src_stage(got["dcat"]))
    return worst


@pytest.mark.parametrize("cid", list(CASES))
def test_emulation_within_grad_bounds(cid):
    args = CASES[cid]
    for seed in (0, 1):                                         # two accumulation orders
        worst = _worst(args, gt.emulate_backward(*args, seed=seed))
        print(cid, seed, {k: round(v, 4) for k, v in worst.items()})
        assert max(worst.values()) <= 1.0, worst


def test_emulation_nonfinite_where_fp64_is():
    for cid in ("golden_nan_depth", "golden_inf_g_scale", "nan_depth_14x36"):
        args = CASES[cid]
        got = gt.emulate_backward(*args)
        want = gt.backward64(*args, mid=got["mid"])
        for k in gg.GRAD_KEYS:
            assert torch.equal(torch.isfinite(got[k]), torch.isfinite(want[k])), (cid, k)


@pytest.mark.parametrize("mutant", gt.GRAD_MUTANTS)
def test_grad_mutant_breaks_a_check(mutant):
    broken = {}
    for cid, args in CASES.items():
        worst = _worst(args, gt.emulate_backward(*args, mutant=mutant))
        bad = {k: v for k, v in worst.items() if v > 1.0}
        if bad:
            broken[cid] = bad
    print(mutant, broken)
    assert broken, f"mutant {mutant} passes every check"
