"""CPU: pins oracle/corr_torch64.py (the fp64 autograd restatement of the correlation block) against the golden vectors
produced by the reference's own CorrBlock1D (tests/golden/make_corr_golden.py), and against its own closed forms.
No CUDA library is imported here."""
import os

import numpy as np
import torch

from oracle import corr_torch64 as ct

G = np.load(os.path.join(os.path.dirname(__file__), "golden", "corr_golden.npz"))
T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(torch.float64)


def test_pyramid_matches_reference():
    pyr = ct.pyramid(T(G["fmap1"]), T(G["fmap2"]), 4)
    for i in range(4):
        assert tuple(pyr[i].shape) == G[f"level{i}"].shape
        assert float((pyr[i] - T(G[f"level{i}"])).abs().max()) <= 1e-12


def test_lookup_matches_reference():
    out = ct.lookup([T(G[f"level{i}"]) for i in range(4)], T(G["coords"]), 4)
    assert tuple(out.shape) == G["out"].shape
    assert float((out - T(G["out"])).abs().max()) <= 2e-6                    # the reference returns .float()


def test_level_grads_match_reference_autograd():
    shapes = [G[f"level{i}"].shape for i in range(4)]
    gl = ct.level_grads(shapes, T(G["coords"]), 4, T(G["grad_out"]))
    for i in range(4):
        assert float((gl[i] - T(G[f"grad_level{i}"])).abs().max()) <= 1e-6  # grad passes the reference's .float() cast


def test_fmap_grads_match_closed_form():
    """Autograd through volume, pyramid and lookup == dF1 = sum_y G F2 / sqrt(D), dF2 = sum_x G F1 / sqrt(D) with G the
    fold of its own per-level gradients; also with only some levels receiving a gradient."""
    f1 = T(G["fmap1"]).requires_grad_(True)
    f2 = T(G["fmap2"]).requires_grad_(True)
    coords, go = T(G["coords"]), T(G["grad_out"])
    for used in ((0, 1, 2, 3), (2,), (1, 3)):
        lv = ct.pyramid(f1, f2, 4)
        gout = go.clone()
        for l in range(4):
            if l not in used:
                gout[:, 9 * l:9 * l + 9] = 0
        d1, d2 = torch.autograd.grad(ct.lookup(lv, coords, 4), (f1, f2), gout)
        gl = ct.level_grads([v.shape for v in lv], coords, 4, gout)
        r1, r2 = ct.fmap_grads_from_levels(f1.detach(), f2.detach(), [g if l in used else None for l, g in enumerate(gl)])
        for got, ref in ((d1, r1), (d2, r2)):
            assert float(ref.abs().max()) > 0.1
            assert float((got - ref).abs().max()) <= 1e-12 * max(1.0, float(ref.abs().max()))


def _sample_loops(vol, x, r):
    """One output element at a time, straight from the definition (python ints)."""
    B, H, W1, W2 = vol.shape
    out = np.zeros((B, 2 * r + 1, H, W1))
    for b in range(B):
        for h in range(H):
            for w in range(W1):
                xv = float(x[b, h, w])
                xf = int(np.floor(xv))
                dx = xv - xf
                tap = lambda k: float(vol[b, h, w, k]) if 0 <= k < W2 else 0.0
                for i in range(2 * r + 1):
                    out[b, i, h, w] = tap(xf - r + i) * (1 - dx) + tap(xf - r + i + 1) * dx
    return out


def test_sample_matches_definition_at_edges():
    """Cut-off windows at both ends, W2 - 1, -0.0, integers, .5, widths 7, 1 and 0, radius 0 and 6."""
    rng = np.random.default_rng(3)
    for W2 in (7, 1, 0):
        for r in (0, 1, 6):
            vol = rng.standard_normal((1, 2, 9, W2))
            x = np.array([-r - 1.0, -r - 0.5, -0.0, 0.5, W2 - 1.0, W2 - 0.25, W2 + r, 3.0, -2.75] * 2,
                         np.float32).reshape(1, 2, 9)
            got = ct.sample(T(vol), torch.from_numpy(x), r).numpy()
            np.testing.assert_allclose(got, _sample_loops(vol, x, r), rtol=0, atol=1e-15)


def test_saturating_coordinates_give_zero_rows_and_zero_grads():
    """|x| past 2^31 (where a 32-bit (int)floorf saturates), and 1e6: the whole window is outside the row."""
    rng = np.random.default_rng(4)
    shapes = [(1, 1, 8, 17 >> l) for l in range(4)]
    lv = [T(rng.standard_normal(s)) for s in shapes]
    x = torch.tensor([[[1e10, -1e10, 3e9, -3e9, 2.0 ** 31, -2.0 ** 31, 1e6, -1e6]]], dtype=torch.float32)
    for r in (0, 4, 6):
        out = ct.lookup(lv, x, r)
        assert bool(torch.isfinite(out).all()) and float(out.abs().max()) == 0.0
        g = ct.level_grads(shapes, x, r, torch.from_numpy(rng.standard_normal(tuple(out.shape))))
        assert all(float(t.abs().max()) == 0.0 for t in g if t.numel())


def test_amp_pyramid_rounds_at_op_boundaries():
    """amp=True: every level holds fp16 values, each pooled level is the fp16 mean of the level above it, level 0 is the
    fp16 division of the fp16 einsum result, and gradients are those of the unrounded block."""
    rng = np.random.default_rng(5)
    f1 = T(rng.standard_normal((1, 48, 2, 24)).astype(np.float16))
    f2 = T(rng.standard_normal((1, 48, 2, 21)).astype(np.float16))
    lv = ct.pyramid(f1, f2, 4, amp=True)
    for v in lv:
        assert bool((v == v.half().double()).all())
    c = torch.einsum("bdhx,bdhy->bhxy", f1, f2).half().double()
    assert bool((lv[0] == (c / ct.sqrt_d(48)).half().double()).all())
    for l in range(1, 4):
        assert bool((lv[l] == ct.pool(lv[l - 1]).half().double()).all())
    a1, a2 = f1.clone().requires_grad_(True), f2.clone().requires_grad_(True)
    coords = torch.from_numpy(rng.uniform(-6, 27, (1, 2, 24)).astype(np.float32))
    go = torch.from_numpy(rng.standard_normal((1, 36, 2, 24)))
    ga = torch.autograd.grad(ct.lookup(ct.pyramid(a1, a2, 4, amp=True), coords, 4), (a1, a2), go)
    gb = torch.autograd.grad(ct.lookup(ct.pyramid(a1, a2, 4), coords, 4), (a1, a2), go)
    for a, b in zip(ga, gb):
        assert float((a - b).abs().max()) <= 1e-12 * float(b.abs().max())
