"""CPU: pins oracle/loss_torch64.py (the fp64 autograd restatement of the photometric loss) against the golden vectors
produced by the reference's own lib/loss.py (tests/golden/make_loss_golden.py), checks its per-element bounds against the
reference's own fp32 chain, and shows that every mutant of it breaks a bound on a case of the GPU sweep.
No CUDA library is imported here."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import loss_cases as lc
from oracle import loss_torch64 as lt

G = np.load(os.path.join(os.path.dirname(__file__), "golden", "loss_golden.npz"))
GOLDEN = ("noise", "smooth", "tiny")
T = lambda a: torch.from_numpy(np.ascontiguousarray(a))


def _rel(a, b):
    return float((a - b).abs().max()) / max(float(b.abs().max()), 1e-300)


def test_window_is_the_reference_window():
    """The fp32 outer product of the stored 1-D window, applied to fp64 precision (vs a plain fp64 11x11 conv2d)."""
    assert np.array_equal(lt.window_2d(torch.float32).numpy(), np.outer(G["window"], G["window"]).astype(np.float32))
    a = torch.from_numpy(np.random.default_rng(0).uniform(-1, 1, (2, 23, 40)))
    want = F.conv2d(a[:, None], lt.window_2d()[None, None], padding=5)[:, 0]
    assert _rel(lt.Window()(a), want) < 1e-14


@pytest.mark.parametrize("name", GOLDEN)
def test_restatement_matches_reference_golden(name):
    x, y = T(G[f"{name}_img"]), T(G[f"{name}_gt"])
    out, gx, _ = lt.forward_and_grads(x, y)
    for k in ("loss", "l1", "ssim"):
        assert abs(float(out[k]) - float(G[f"{name}_f64_{k}"])) <= 1e-14, k
    if f"{name}_f64_ssim_per_image" in G:
        assert _rel(out["ssim_per_image"], T(G[f"{name}_f64_ssim_per_image"])) <= 1e-14
    assert _rel(gx, T(G[f"{name}_f64_grad"])) <= 1e-12


@pytest.mark.parametrize("case", [lc.SWEEP[i] for i in (0, 13, 40, 62, 80, 83, 85)] + [("signed", (2, 3, 20, 9), 7)],
                         ids=lc.case_id)
def test_closed_form_backward_matches_autograd(case):
    """The backward the kernel evaluates (window sum of the three partials + the L1 sign) == autograd, for img and gt;
    the gt partials are the img partials of the swapped call (the binding's d/d gt)."""
    x, y = map(T, lc.image_pair(*case))
    out, gx, gy = lt.forward_and_grads(x, y, 0.3, 0.7)
    di, dg = lt.dmaps(out["moments"])
    assert _rel(lt.grad_from_dmaps(x, y, di, 0.3, 0.7), gx) <= 1e-12
    assert _rel(lt.grad_from_dmaps(y, x, dg, 0.3, 0.7), gy) <= 1e-12
    assert _rel(lt.dmaps(lt.forward(y, x)["moments"])[0], dg) <= 1e-14


def _fp32_chain_utilisation(x, y):
    out, gx, gy = lt.forward_and_grads(x, y)
    b = lt.bounds(x, y, out["moments"])
    loss, fx, fy = lt.reference_fp32(x, y)
    worst = 0.0
    for got, ref, bnd in ((fx, gx, b["grad_img"]), (fy, gy, b["grad_gt"])):
        err = (got.to(torch.float64) - ref).abs()
        worst = max(worst, float(torch.where(err == 0, torch.zeros_like(err), err / bnd).max()))
    assert abs(float(loss) - float(out["loss"])) <= b["loss"]
    return worst


@pytest.mark.parametrize("name", GOLDEN + ("flat_bright_256", "noisy_256"))
def test_reference_fp32_chain_within_a_quarter_of_the_bound(name):
    """The reference's fp32 autograd chain (121-tap conv2d, its op order) stays within C_BOUND / 4 on every element of
    both gradients: the bound leaves room for an fp32 kernel and is no looser than fp32 needs."""
    if name in GOLDEN:
        x, y = T(G[f"{name}_img"]), T(G[f"{name}_gt"])
        assert _rel(lt.reference_fp32(x, y)[1], T(G[f"{name}_f32_grad"])) < 1e-5      # it is the reference's chain
    else:
        rng = np.random.default_rng(11)
        gt = np.full((1, 3, 256, 256), 0.95) if name == "flat_bright_256" else rng.uniform(0, 1, (1, 3, 256, 256))
        img = np.clip(gt + rng.normal(0, 0.05, gt.shape), 0, 1)
        x, y = T(img.astype(np.float32)), T(gt.astype(np.float32))
    worst = _fp32_chain_utilisation(x, y)
    print(f"{name}: fp32 chain at {worst:.3f} of the bound")
    assert worst <= 0.25


def test_reference_fp32_chain_within_the_bound_on_the_sweep():
    worst = max(_fp32_chain_utilisation(*map(T, lc.image_pair(*c))) for c in lc.SWEEP)
    print(f"sweep: fp32 chain at {worst:.3f} of the bound")
    assert worst <= 0.25


def test_unmutated_closed_form_is_within_every_bound():
    for case in lc.SWEEP[::7]:
        x, y = map(T, lc.image_pair(*case))
        r = lc.ratios(lc.reference(x, y), lc.outputs_of(lt.mutant_outputs(x, y, 0.8, 0.2, None)))
        assert max(r.values()) <= 1e-3, (lc.case_id(case), r)


@pytest.mark.parametrize("mutant", lt.MUTANTS)
def test_mutant_breaks_a_bound_on_the_gpu_sweep(mutant):
    """A kernel with this bug would fail tests/test_loss_fp64_gpu.py: some quantity leaves its bound on some case."""
    for case in lc.SWEEP:
        x, y = map(T, lc.image_pair(*case))
        r = lc.ratios(lc.reference(x, y), lc.outputs_of(lt.mutant_outputs(x, y, 0.8, 0.2, mutant)))
        if max(r.values()) > 1.0:
            print(mutant, "caught by", lc.case_id(case), {k: v for k, v in r.items() if v > 1.0})
            return
    pytest.fail(f"mutant {mutant} stays within every bound on the whole sweep")


def test_fp32_partials_within_the_bound_on_the_sweep():
    """The three partials evaluated in fp32 from fp32 121-tap conv2d moments (the reference's forward) stay within
    half of their per-pixel bound: C_DMAPS leaves room for an fp32 kernel."""
    worst = 0.0
    for case in lc.SWEEP:
        x, y = map(T, lc.image_pair(*case))
        xp, yp = lt.planes_of(x), lt.planes_of(y)
        w = lt.window_2d(torch.float32)[None, None]
        conv = lambda t: F.conv2d(t[:, None], w, padding=5)[:, 0]
        m32 = [t.requires_grad_(True) for t in (conv(xp), conv(yp), conv(xp * xp), conv(yp * yp), conv(xp * yp))]
        g = torch.autograd.grad(lt.ssim_from_moments(*m32).sum(), m32)
        got = torch.stack([g[0], g[2], g[4]]).to(torch.float64)
        mom = lt.forward(x, y)["moments"]
        err = (got - lt.dmaps(mom)[0]).abs()
        r = torch.where(err == 0, torch.zeros_like(err), err / lt.bounds(x, y, mom)["dmaps_img"])
        worst = max(worst, float(r.max()))
    print(f"sweep: fp32 partials at {worst:.3f} of the bound")
    assert worst <= 0.5
