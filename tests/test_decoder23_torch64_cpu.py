"""CPU: the fp64 restatement of the regressor's decoder3 and decoder2 (oracle/decoder23_torch64.py) against the
reference's own ResidualBlocks and nn.Upsample (tests/golden/decoder23_golden.npz), the TF32 emulation of the kernels
against the per-element bounds, and each mutant of the emulation against those bounds: every mutant must break a check
that the emulation passes."""
import pytest
import torch

import decoder23_cases as dc
from oracle import decoder23_torch64 as dt


@pytest.mark.parametrize("name", dc.GOLDEN_CASES)
def test_restatement_matches_golden(name):
    d = dc.golden(name)
    out3 = dt.forward64("d3", *dc.stage_args(d, "d3"))["out"]
    assert out3.shape == d["out3"].shape
    assert torch.allclose(out3, d["out3"], rtol=1e-10, atol=1e-12), float((out3 - d["out3"]).abs().max())
    out2 = dt.forward64("d2", *dc.stage_args(d, "d2", s=d["out3"]))["out"]
    assert out2.shape == d["out2"].shape
    assert torch.allclose(out2, d["out2"], rtol=1e-10, atol=1e-12), float((out2 - d["out2"]).abs().max())


def test_zero_variance_group_is_its_bias():
    d = dc.golden("zero_var_group")
    for st in dt.STAGES:                                        # decoder2 on a zero s: its whole input is zero
        srcs, ps = dc.stage_args(d, st, s=torch.zeros_like(d["f3i"]))
        ya = dt.forward64(st, srcs, ps)["ya"]
        assert torch.equal(ya[:, :8], ps[1][:8].to(torch.float64).view(1, 8, 1, 1).expand_as(ya[:, :8]))
        h = dt.group_norm(ya, dt.GROUPS[st], ps[2], ps[3])      # a zero-variance group normalizes to its bias
        assert torch.equal(h[:, :8], ps[3][:8].to(torch.float64).view(1, 8, 1, 1).expand_as(h[:, :8]))


def _all_cases():
    for name in dc.GOLDEN_CASES:
        d = dc.golden(name)
        d["s"] = d["out3"].float()
        for st in dt.STAGES:
            yield f"golden_{name}_{st}", (st,) + dc.stage_args(d, st)
    for case in dc.SWEEP:
        d = dc.inputs(case)
        for st in dt.STAGES:
            yield f"{case.id}_{st}", (st,) + dc.stage_args(d, st)


CASES = dict(_all_cases())


def _worst(args, got):
    """Worst error-to-bound ratios: end to end against fp64 (KEYS) and per stage on the emulation's own stored
    convolution outputs (stage_<key>)."""
    want = dt.forward64(*args)
    b = dt.bounds(*args)
    out = {k: dt.ratio(got[k], want[k], b[k]) for k in dt.KEYS}
    stages = dt.stage_checks(*args, [got[k] for k in dt.RAW_KEYS])
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
    for cid in ("nan_3x4_d3", "nan_3x4_d2", "inf_2x3_d3", "inf_2x3_d2"):
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
