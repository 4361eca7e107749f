"""CPU: the fp64 restatement of the regressor's full-resolution tail (oracle/gs_head_torch64.py) against the reference's
own module (tests/golden/gs_head_golden.npz), its TF32 emulation against the per-element bounds, and each mutant of the
emulation against those bounds: every mutant must break a check that the emulation passes."""
import pytest
import torch

import gs_head_cases as gc
from oracle import gs_head_torch64 as gt

OUTS = ("rot", "scale", "opacity")
CHECKED = OUTS + ("scale_pre", "pre", "mid")


@pytest.mark.parametrize("name", gc.GOLDEN_CASES)
def test_restatement_matches_golden(name):
    src, img, depth, ps, want = gc.golden(name)
    got = gt.forward64(src, img, depth, ps)
    for k in OUTS:
        assert torch.allclose(got[k], want[k], rtol=1e-12, atol=1e-15), (k, float((got[k] - want[k]).abs().max()))


def _all_cases():
    for name in gc.GOLDEN_CASES:
        src, img, depth, ps, _ = gc.golden(name)
        yield "golden_" + name, (src, img, depth, ps)
    for case in gc.SWEEP:
        yield case.id, gc.inputs(case)


CASES = dict(_all_cases())


def _worst(args, got):
    want = gt.forward64(*args)
    b = gt.bounds(*args)
    return {k: gt.ratio(got[k], want[k], b[k]) for k in CHECKED}


@pytest.mark.parametrize("cid", list(CASES))
def test_emulation_within_bounds(cid):
    args = CASES[cid]
    for seed in (0, 1):                                         # two accumulation orders
        worst = _worst(args, gt.emulate(*args, seed=seed))
        print(cid, seed, worst)
        assert max(worst.values()) <= 1.0, worst


def test_emulation_nan_where_fp64_nan():
    args = CASES["nan_depth_14x36"]
    want, got = gt.forward64(*args), gt.emulate(*args)
    for k in OUTS:
        assert torch.isnan(want[k]).any() and torch.equal(torch.isnan(got[k]), torch.isnan(want[k])), k


@pytest.mark.parametrize("mutant", gt.MUTANTS)
def test_mutant_breaks_a_check(mutant):
    broken = {}
    for cid, args in CASES.items():
        worst = _worst(args, gt.emulate(*args, mutant=mutant))
        bad = {k: v for k, v in worst.items() if v > 1.0}
        if bad:
            broken[cid] = bad
    print(mutant, broken)
    assert broken, f"mutant {mutant} passes every check"
