"""CPU: the fp64 restatement of the update block (oracle/update_torch64.py) against the reference's own
BasicMultiUpdateBlock and FlowUpdateModule run in fp64 (tests/golden/update_golden.npz, tests/golden/make_update_golden.py):
single iterations at 1 x 1, 3 x 5 and 9 x 7 with B = 1 and 2, and a three-iteration loop in test mode and not."""
import os

import numpy as np
import pytest
import torch

import update_cases as uc
from oracle import update_torch64 as ut

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "update_golden.npz")


@pytest.fixture(scope="module")
def golden():
    return np.load(GOLDEN)


def _close(got, want):
    want = torch.from_numpy(want).to(torch.float64)
    tol = 1e-6 * float(want.abs().max()) + 1e-12
    err = float((got.to(torch.float64) - want).abs().max())
    assert err <= tol, (err, tol)


@pytest.mark.parametrize("case", uc.STEP_CASES, ids=lambda c: "x".join(map(str, c)))
def test_iteration(golden, case):
    B, H, W = case
    inp = uc.inputs(B, H, W)
    cz, cr, cq = inp["czrq"].split(uc.HID, 1)
    o = ut.iteration64(uc.params(0), inp["corr"], inp["coords1"] - ut.grid(B, H, W), inp["net"], cz, cr, cq)
    tag = f"step_{B}x{H}x{W}_"
    for k in ("h", "delta", "mask"):
        _close(o[k], golden[tag + k])


@pytest.mark.parametrize("test_mode", [True, False], ids=["test", "train"])
def test_loop(golden, test_mode):
    B, H, W, iters = uc.LOOP_CASE
    f1, f2 = uc.fmaps(B, H, W)
    inp = uc.inputs(B, H, W)
    got = ut.loop64(uc.params(0), f1, f2, inp["net"], inp["czrq"], iters, None, test_mode)
    if test_mode:
        _close(got, golden["loop_flow_up"])
    else:
        assert len(got) == iters
        for i, p in enumerate(got):
            _close(p, golden[f"loop_pred{i}"])
