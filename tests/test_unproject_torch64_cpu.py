"""CPU: pins oracle/unproject_torch64.py (the fp64 autograd restatement of flow2depth + depth2pc) against the golden
vectors produced by the reference's own functions (tests/golden/make_unproject_golden.py), checks that its fp32 form
(the reference's op order) meets the bounds the kernel is held to, and shows that every mutant of it breaks a check on
a case of the GPU sweep.  No CUDA library is imported here."""
import os

import numpy as np
import pytest
import torch

import unproject_cases as uc
from oracle import unproject_torch64 as ut

G = np.load(os.path.join(os.path.dirname(__file__), "golden", "unproject_golden.npz"))
T = lambda k: torch.from_numpy(G[k])
CPU_SWEEP = [c for c in uc.SWEEP if c[1] <= 257]


def _rel(a, b):
    return float((a - b).abs().max()) / max(float(b.abs().max()), 1e-300)


def test_restatement_matches_reference_golden():
    args = [T(k) for k in ("flow", "mask", "intr", "extr", "ref_intr", "tf_x")]
    depth, xyz, valid, g = ut.forward_and_grad(*args, T("g_xyz"), T("g_depth"))
    assert _rel(depth, T("depth")) <= 1e-12
    assert torch.equal(valid, T("valid"))
    v = T("valid")
    assert _rel(xyz[v], T("xyz")[v]) <= 1e-12
    assert _rel(xyz, T("xyz")) <= 1e-12                                  # the 1e8-scaled invalid pixels as well
    assert _rel(g, T("d_flow")) <= 1e-12


def test_pixel_centres_are_exact_in_fp32():
    """linspace(0.5, S - 0.5, S) in fp32 is u + 0.5 exactly, so the fp32 restatement sees the kernel's centres."""
    for S in uc.SIZES:
        assert torch.equal(ut.pixel_centres(S, torch.float32), torch.arange(S, dtype=torch.float32) + 0.5)


def test_case_inputs_have_the_edges():
    """flow == offset at mask 1 gives depth 0 and pts_valid False; cx != cy; mask channel 1 != channel 0."""
    inp = uc.make_case(*uc.SWEEP[3])
    d, _, valid = ut.unproject(inp["flow"], inp["mask"], inp["intr"], inp["extr"], inp["ref_intr"], inp["tf_x"],
                               dtype=torch.float32)
    zero_at_mask1 = (d[:, 0] == 0) & (inp["mask"][:, 0] == 1)
    assert int(zero_at_mask1.sum()) >= 1 and not bool(valid.reshape(d[:, 0].shape)[zero_at_mask1].any())
    assert bool((inp["intr"][:, 0, 2] != inp["intr"][:, 1, 2]).all())
    assert set(np.sign(np.concatenate([uc.make_case(*c)["tf_x"].numpy() for c in uc.SWEEP[:3]]))) == {-1.0, 1.0}


@pytest.mark.parametrize("case", CPU_SWEEP[::3], ids=uc.case_id)
def test_fp32_restatement_within_every_bound(case):
    """The reference's own fp32 chain (autograd included) meets every check the kernel is held to."""
    inp = uc.make_case(*case)
    r = uc.ratios(uc.reference(inp), uc.stand_in(inp))
    print(uc.case_id(case), r)
    assert max(r.values()) <= 0.25, r


@pytest.mark.parametrize("mutant", ut.MUTANTS)
def test_mutant_breaks_a_check_on_the_gpu_sweep(mutant):
    for case in CPU_SWEEP:
        inp = uc.make_case(*case)
        r = uc.ratios(uc.reference(inp), uc.stand_in(inp, mutant))
        if max(r.values()) > 1.0:
            print(mutant, "caught by", uc.case_id(case), {k: v for k, v in r.items() if v > 1.0})
            return
    pytest.fail(f"mutant {mutant} passes every check on the whole sweep")
