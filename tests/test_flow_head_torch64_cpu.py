"""CPU: pins oracle/flow_head_torch64.py (the fp64 autograd restatement of the disparity head) against the goldens
produced by the reference's own functions (tests/golden/make_flow_head_golden.py), checks that the fp32 emulation of the
kernels (oracle/flow_head_oracle.py with their dtype boundaries) stays within the per-element bounds on the sweep of
tests/flow_head_cases.py, and shows that every mutant of that emulation breaks a bound on a case of the GPU sweep.
No CUDA library is imported here."""
import functools
import os

import numpy as np
import pytest
import torch

import flow_head_cases as fc
from oracle import flow_head_oracle as fo
from oracle import flow_head_torch64 as ft

GOLDEN = np.load(os.path.join(os.path.dirname(__file__), "golden", "flow_head_golden.npz"))
UP = sorted({k[3:-len("_factor")] for k in GOLDEN.files if k.startswith("up_") and k.endswith("_factor")})
SL = sorted({k[3:-len("_raises")] for k in GOLDEN.files if k.startswith("sl_") and k.endswith("_raises")})
NP_DT = {"f32": np.float32, "f16": np.float16}
TENSORS = ("out", "dmask", "dflow")


def _rel(a, b):
    a, b = torch.as_tensor(a, dtype=torch.float64), torch.as_tensor(b, dtype=torch.float64)
    fin = ~torch.isnan(b)
    assert torch.equal(torch.isnan(a), ~fin)
    return float((a[fin] - b[fin]).abs().max()) / max(float(b[fin].abs().max()), 1e-300)


def _up(name, key):
    return GOLDEN[f"up_{name}_{key}"]


@pytest.mark.parametrize("name", UP)
def test_restatement_matches_reference_golden(name):
    """fp64 goldens to ~1e-12.  The fp32 goldens are the reference's own fp32 op chain on the CPU: each of its elements
    lies within the kernels' bounds, which shows they hold an independent fp32 evaluation.  (The CPU's fp16 softmax
    does not round the weights once from fp32, so the fp16 goldens are held to test_flow_head_cpu.py's bounds only.)"""
    f = int(_up(name, "factor"))
    flow, mask, g = (torch.from_numpy(_up(name, k)) for k in ("flow", "mask", "g"))
    out, dflow, dmask = ft.forward_and_grads(flow, mask, f, g)
    got = {"out": _up(name, "out"), "dflow": _up(name, "d_flow"), "dmask": _up(name, "d_mask")}
    if name.endswith("_f64"):
        for k, want in (("out", out), ("dflow", dflow), ("dmask", dmask)):
            assert _rel(got[k], want) <= 1e-12, k
        return
    if name.endswith("_f16"):
        pytest.skip("the CPU's fp16 softmax rounds the weights in its own places; held to test_flow_head_cpu.py's bounds")
    b = ft.bounds(flow, mask, f, g)
    r = {k: ft.ratio(got[k], want, b[k]) for k, want in (("out", out), ("dflow", dflow), ("dmask", dmask))}
    print(f"{name}: reference fp32 chain at {r} of the bounds")
    assert max(r.values()) <= 1.0, r


@pytest.mark.parametrize("name", SL)
def test_sequence_loss64_matches_reference_golden(name):
    sl = lambda k: GOLDEN[f"sl_{name}_{k}"]
    if str(sl("raises")):
        return
    preds, gt, valid = [torch.from_numpy(p) for p in sl("preds")], torch.from_numpy(sl("gt")), torch.from_numpy(sl("valid"))
    r = ft.sequence_loss64(preds, gt, valid, fp32_diff=False)
    want_loss, (epe, px1, px3) = float(sl("loss_f64")), sl("metrics_f64")
    if np.isnan(want_loss):
        assert r["count"] == 0
        return
    assert abs(float(r["loss"]) - want_loss) <= 1e-12 * abs(want_loss)
    assert abs(float(r["epe"]) - epe) <= 1e-12 * abs(epe)
    # the golden takes (epe < t).float().mean(): an fp32 fraction even in the fp64 run
    assert abs(r["c1"] / r["count"] - px1) <= 2.0 ** -24 and abs(r["c3"] / r["count"] - px3) <= 2.0 ** -24
    # on the fp32 differences the loss moves by at most the fp32 rounding of each |p - gt| and of the weights
    r32 = ft.sequence_loss64(preds, gt, valid)
    assert abs(float(r32["loss"]) - want_loss) <= 2 * 2.0 ** -24 * abs(want_loss)


@functools.lru_cache(maxsize=4)
def _truth(case):
    flow, mask, g = fc.inputs(case, n=1)
    out, dflow, dmask = ft.forward_and_grads(flow, mask, case.f, g)
    return (flow, mask, g), {"out": out, "dflow": dflow, "dmask": dmask}, ft.bounds(flow, mask, case.f, g)


def _emulate(case, mutant=None):
    (flow, mask, g), _, _ = _truth(case)
    fl, m, gg = flow.numpy(), mask.numpy(), g.numpy()
    dt = NP_DT[case.dtype]
    out = fo.convex_upsample(fl, m, case.f, dt, mutant)
    dflow, dmask = fo.convex_upsample_backward(fl, m, case.f, gg, dt, mutant)
    return {"out": out, "dflow": dflow, "dmask": dmask}


def _ratios(case, got):
    _, want, b = _truth(case)
    return {k: ft.ratio(got[k], want[k], b[k]) for k in TENSORS}


@pytest.mark.parametrize("dtype", ["f32", "f16"])
def test_emulation_within_the_bounds_on_the_sweep(dtype):
    """The kernels' op order and dtype boundaries in numpy stay within every bound, on every element of every sweep case
    at N = 1 and at the training shapes; the printed worst utilisation per tensor shows how much room is left.  With an
    fp16 mask it is close to 1 by construction: a weight that rounds by nearly half an fp16 ulp uses up its bound."""
    worst = dict.fromkeys(TENSORS, 0.0)
    for case in [c for c in fc.SWEEP + fc.STAGES if c.dtype == dtype]:
        r = _ratios(case, _emulate(case))
        assert max(r.values()) <= 1.0, (case.id, r)
        worst = {k: max(worst[k], r[k]) for k in TENSORS}
    print(f"{dtype} mask: worst utilisation of the emulation {worst}")


@pytest.mark.parametrize("mutant", fo.UPSAMPLE_MUTANTS)
def test_upsample_mutant_breaks_a_bound_on_the_gpu_sweep(mutant):
    """A kernel with this bug would fail tests/test_flow_head_fp64_gpu.py: some element leaves its bound on some case."""
    for case in fc.SWEEP:
        r = _ratios(case, _emulate(case, mutant))
        if max(r.values()) > 1.0:
            print(mutant, "caught by", case.id, {k: v for k, v in r.items() if v > 1.0})
            return
    pytest.fail(f"mutant {mutant} stays within every bound on the whole sweep")


def _loss_check(case, mutant=None, n=None):
    """Worst |kernel emulation - fp64| / bound of the loss and the EPE, and whether the fractions are exact."""
    preds, gt, valid = fc.loss_inputs(case, n=n)
    want = ft.sequence_loss64(preds, gt, valid)
    loss, epe, px1, px3 = fo.sequence_loss_kernel([p.numpy() for p in preds], gt.numpy(), valid.numpy(), mutant=mutant)
    tol = ft.loss_bound(case.P)
    r = {"loss": abs(float(loss) - float(want["loss"])) / (tol * float(want["loss"])),
         "epe": abs(float(epe) - float(want["epe"])) / (tol * float(want["epe"]))}
    exact = float(px1) == ft.fraction32(want["c1"], want["count"]) and float(px3) == ft.fraction32(want["c3"], want["count"])
    return r, exact


def test_loss_emulation_within_the_bounds():
    """Every loss case at full size, among them 17 * 1024^2 pixels with an odd valid count above 2^24, where the
    forward's float(count) rounds and (P + 4) has to cover that rounding too."""
    most = next(c for c in fc.LOSS if c.valid == "most")
    count = int((fc.loss_inputs(most)[2] >= 0.5).sum())
    assert count > 2 ** 24 and float(np.float32(count)) != count
    worst = {"loss": 0.0, "epe": 0.0}
    for case in fc.LOSS:
        r, exact = _loss_check(case)
        assert exact and max(r.values()) <= 1.0, (case.id, r)
        worst = {k: max(worst[k], r[k]) for k in worst}
    print(f"sequence loss: worst utilisation of the emulation {worst}")


def test_loss_bound_constant_covers_the_count_rounding():
    """Above 2^24 float(count) rounds: one more rounding than below, and (P + 4) counts it.  The count 2^24 + 1 rounds
    to 2^24, a relative change of 2^-24 / (1 + 2^-24), within one u."""
    c = 2 ** 24 + 1
    assert float(np.float32(c)) == 2.0 ** 24
    assert abs(float(np.float32(c)) - c) / c <= ft.U


@pytest.mark.parametrize("mutant", fo.LOSS_MUTANTS)
def test_loss_mutant_breaks_a_bound(mutant):
    for case in fc.LOSS:
        r, exact = _loss_check(case, mutant, n=1)
        if max(r.values()) > 1.0 or not exact:
            print(mutant, "caught by", case.id, r, "fractions exact" if exact else "fractions differ")
            return
    pytest.fail(f"mutant {mutant} stays within every bound on every loss case")
