"""CPU: the fp64 restatement of the UnetExtractor's half-resolution stem (oracle/encoder_torch64.py) against the
reference's own module (tests/golden/encoder_golden.npz), the emulation of both kernel precisions against the
per-element bounds, and each mutant of the emulation against those bounds: every mutant must break a check that the
emulation passes."""
import pytest
import torch

import encoder_cases as ec
from oracle import encoder_torch64 as et

MODES = ("tf32", "fp16")


@pytest.mark.parametrize("name", ec.GOLDEN_CASES)
def test_restatement_matches_golden(name):
    x, ps, want = ec.golden(name)
    got = et.forward64(x, ps)["x1"]
    assert got.shape == want.shape
    assert torch.allclose(got, want, rtol=1e-10, atol=1e-12), float((got - want).abs().max())


def test_zero_variance_group_is_its_bias():
    x, ps, want = ec.golden("zero_var_group")
    x0 = et.forward64(x, ps)["x0"]
    beta = ps[3][:4].to(torch.float64).view(1, 4, 1, 1)
    assert torch.equal(x0[:, :4], torch.where(beta < 0, torch.zeros_like(beta), beta).expand_as(x0[:, :4]))


def _all_cases():
    for name in ec.GOLDEN_CASES:
        x, ps, _ = ec.golden(name)
        yield "golden_" + name, (x, ps)
    for case in ec.SWEEP:
        yield case.id, ec.inputs(case)


CASES = dict(_all_cases())


def _worst(args, got, mode):
    """Worst error-to-bound ratios: end to end against fp64 (KEYS) and per stage on the emulation's own stored
    convolution outputs (stage_<key>)."""
    want = et.forward64(*args)
    b = et.bounds(*args, mode=mode)
    out = {k: et.ratio(got[k], want[k], b[k]) for k in et.KEYS}
    stages = et.stage_checks(*args, [got[f"y{i}"] for i in range(5)], mode=mode)
    out.update({"stage_" + k: et.ratio(got[k], w, bd) for k, (w, bd) in stages.items()})
    return out


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("cid", list(CASES))
def test_emulation_within_bounds(cid, mode):
    args = CASES[cid]
    for seed in (0, 1):                                         # two accumulation orders
        worst = _worst(args, et.emulate(*args, mode=mode, seed=seed), mode)
        print(cid, mode, seed, worst)
        assert max(worst.values()) <= 1.0, worst


@pytest.mark.parametrize("mode", MODES)
def test_emulation_nan_where_fp64_nan(mode):
    for cid in ("depth_nan_14x12", "rgb_inf_9x11"):
        args = CASES[cid]
        want, got = et.forward64(*args)["x1"], et.emulate(*args, mode=mode)["x1"]
        assert torch.isnan(want[0]).all() and not torch.isnan(want[1:]).any()       # the whole sample, only it
        assert torch.equal(torch.isnan(got), torch.isnan(want))


@pytest.mark.parametrize("mutant", et.MUTANTS)
def test_mutant_breaks_a_check(mutant):
    broken = {}
    for mode in MODES:
        for cid, args in CASES.items():
            worst = _worst(args, et.emulate(*args, mode=mode, mutant=mutant), mode)
            bad = {k: v for k, v in worst.items() if v > 1.0}
            if bad:
                broken[(mode, cid)] = bad
    print(mutant, broken)
    assert broken, f"mutant {mutant} passes every check"
