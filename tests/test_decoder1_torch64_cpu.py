"""CPU: the fp64 restatement of the regressor's decoder1 (oracle/decoder1_torch64.py) against the reference's own
ResidualBlocks and nn.Upsample (tests/golden/decoder1_golden.npz), the TF32 emulation of the kernels against the
per-element bounds, and each mutant of the emulation against those bounds: every mutant must break a check that the
emulation passes."""
import pytest
import torch

import decoder1_cases as dc
from oracle import decoder1_torch64 as dt


@pytest.mark.parametrize("name", dc.GOLDEN_CASES)
def test_restatement_matches_golden(name):
    s, fi, fd, ps, want = dc.golden(name)
    got = dt.forward64(s, fi, fd, ps)["out"]
    assert got.shape == want.shape
    assert torch.allclose(got, want, rtol=1e-10, atol=1e-12), float((got - want).abs().max())


def test_zero_variance_group_is_its_bias():
    s, fi, fd, ps, _ = dc.golden("zero_var_group")
    y1 = dt.forward64(s, fi, fd, ps)["y1"]
    assert torch.equal(y1[:, :8], ps[1][:8].to(torch.float64).view(1, 8, 1, 1).expand_as(y1[:, :8]))
    h = dt.group_norm(y1, 6, ps[2], ps[3])                      # a zero-variance group normalizes to its bias
    assert torch.equal(h[:, :8], ps[3][:8].to(torch.float64).view(1, 8, 1, 1).expand_as(h[:, :8]))


def _all_cases():
    for name in dc.GOLDEN_CASES:
        s, fi, fd, ps, _ = dc.golden(name)
        yield "golden_" + name, (s, fi, fd, ps)
    for case in dc.SWEEP:
        yield case.id, dc.inputs(case)


CASES = dict(_all_cases())


def _worst(args, got):
    """Worst error-to-bound ratios: end to end against fp64 (KEYS) and per stage on the emulation's own stored
    convolution outputs (stage_<key>)."""
    want = dt.forward64(*args)
    b = dt.bounds(*args)
    out = {k: dt.ratio(got[k], want[k], b[k]) for k in dt.KEYS}
    stages = dt.stage_checks(*args, [got[k] for k in ("y1", "yd", "y2", "y3", "y4")])
    out.update({"stage_" + k: dt.ratio(got[k], w, bd) for k, (w, bd) in stages.items()})
    return out


@pytest.mark.parametrize("cid", list(CASES))
def test_emulation_within_bounds(cid):
    args = CASES[cid]
    for seed in (0, 1):                                         # two accumulation orders
        worst = _worst(args, dt.emulate(*args, seed=seed))
        print(cid, seed, worst)
        assert max(worst.values()) <= 1.0, worst


def test_emulation_nan_where_fp64_nan():
    for cid in ("nan_4x6", "inf_3x5"):
        args = CASES[cid]
        want, got = dt.forward64(*args)["out"], dt.emulate(*args)["out"]
        assert torch.isnan(want[0]).all() and not torch.isnan(want[1:]).any()       # the whole sample, only it
        assert torch.equal(torch.isnan(got), torch.isnan(want))


@pytest.mark.parametrize("mutant", dt.MUTANTS)
def test_mutant_breaks_a_check(mutant):
    broken = {}
    for cid, args in CASES.items():
        worst = _worst(args, dt.emulate(*args, mutant=mutant))
        bad = {k: v for k, v in worst.items() if v > 1.0}
        if bad:
            broken[cid] = bad
    print(mutant, broken)
    assert broken, f"mutant {mutant} passes every check"
