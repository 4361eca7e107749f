"""GPU: the disparity head (csrc/flow_head.cu through gps_gaussian_b200.flow_head) against the fp64 restatement
(oracle/flow_head_torch64.py), per element, over tests/flow_head_cases.py: every factor at widths on both sides of one,
two and three forward and backward segments, both mask dtypes, large, -inf and non-finite logits, dL/dout with channel 1
zero or not, one input without grad, the mask and the incoming gradient at element offsets 1 and 2, the training shapes
(every batch element), a mask of more than 2^31 elements, and the sequence loss at the training size, above 2^24 valid
pixels and at the edges of its partial grid.

Every output buffer is poisoned with NaN before each launch.  out, dL/dmask and dL/dflow must be NaN exactly where fp64
autograd is and within `flow_head_torch64.bounds` elsewhere; the worst error-to-bound ratio per tensor and case goes to
$GPSG_PARITY_LOG.  tests/test_flow_head_torch64_cpu.py shows that each mutant of the kernels' emulation breaks one of
these checks on this sweep."""
import types

import numpy as np
import pytest
import torch

import flow_head_cases as fc
from helpers import record
from gps_gaussian_b200 import flow_head, harness, patch
from oracle import flow_head_torch64 as ft

pytestmark = pytest.mark.gpu
needs_ref = pytest.mark.skipif(harness.staged_reference() is None, reason="oracle/_ref not staged")
TENSORS = ("out", "dflow", "dmask")


@pytest.fixture(autouse=True)
def poisoned_outputs(monkeypatch):
    """torch.empty / empty_like inside flow_head return NaN-filled buffers, so an output element the kernels skip shows."""
    def nan(fn):
        def make(*a, **k):
            t = fn(*a, **k)
            if t.is_floating_point():
                t.fill_(float("nan"))
            return t
        return make
    fake = types.SimpleNamespace(**{n: getattr(torch, n) for n in dir(torch) if not n.startswith("__")})
    fake.empty, fake.empty_like = nan(torch.empty), nan(torch.empty_like)
    monkeypatch.setattr(flow_head, "torch", fake)


def _at_offset(t, off):
    """t on the device as a view at element offset `off` of a larger buffer."""
    buf = torch.empty(t.numel() + off, dtype=t.dtype, device="cuda")
    v = buf[off:].view(t.shape)
    v.copy_(t)
    assert v.storage_offset() == off and v.is_contiguous()
    return v


def _device_run(case, flow, mask, g):
    fl = flow.cuda().requires_grad_(case.needs in ("both", "flow"))
    m = _at_offset(mask, case.mask_off).requires_grad_(case.needs in ("both", "mask"))
    gd = _at_offset(g, case.g_off)
    out = flow_head.convex_upsample(fl, m, case.f)
    out.backward(gd)
    assert out.dtype == torch.float32
    assert (fl.grad is None) == (case.needs == "mask") and (m.grad is None) == (case.needs == "flow")
    if m.grad is not None:
        assert m.grad.dtype == m.dtype
    return {"out": out.detach(), "dflow": fl.grad, "dmask": m.grad}


def _check(case, flow, mask, g, got):
    """Worst ratio per tensor, each batch element against its own fp64 truth on the device (pixels are independent
    across the batch)."""
    worst = {k: 0.0 for k in TENSORS if got[k] is not None}
    for n in range(case.N):
        sl = lambda t: t[n:n + 1].cuda()
        fl, m, gg = sl(flow), sl(mask), sl(g)
        out, dflow, dmask = ft.forward_and_grads(fl, m, case.f, gg, got["dflow"] is not None, got["dmask"] is not None)
        b = ft.bounds(fl, m, case.f, gg)
        want = {"out": out, "dflow": dflow, "dmask": dmask}
        for k in worst:
            worst[k] = max(worst[k], ft.ratio(got[k][n:n + 1], want[k], b[k]))
    record("flow_head_fp64:" + case.id, mask=case.dtype, **worst)
    print(f"{case.id}: utilisation {worst}")
    assert max(worst.values()) <= 1.0, worst


def _run_and_check(case):
    flow, mask, g = fc.inputs(case)
    _check(case, flow, mask, g, _device_run(case, flow, mask, g))


@pytest.mark.parametrize("case", fc.SWEEP, ids=lambda c: c.id)
def test_sweep_vs_fp64(case):
    _run_and_check(case)


@pytest.mark.parametrize("case", fc.ALIGN, ids=lambda c: c.id)
def test_offset_views_vs_fp64(case):
    _run_and_check(case)


@pytest.mark.parametrize("case", fc.STAGES, ids=lambda c: c.id)
def test_training_shapes_every_batch_element(case):
    _run_and_check(case)


def test_mask_past_2_31_elements():
    """N = 16, fp16, f = 8 at 512^2: 2.4e9 mask elements, so the whole last batch element sits past 2^31.  Every one
    of its coarse rows is checked, 64 at a time, against the fp64 truth of a band one row wider on each cut side (a
    row's results depend on its neighbours' flow and tap sums only)."""
    N, D, H, W, f = 16, 1, 512, 512, 8
    if torch.cuda.mem_get_info()[0] < 24 * 2 ** 30:
        pytest.skip("needs 24 GB of free device memory")
    gen = torch.Generator(device="cuda").manual_seed(7)
    flow = (torch.rand(N, D, H, W, device="cuda", generator=gen) * 25 - 20).requires_grad_()
    mask = torch.empty(N, 9 * f * f, H, W, dtype=torch.float16, device="cuda")
    mask.normal_(0.0, 4.0, generator=gen)
    assert mask.numel() > 2 ** 31 and (N - 1) * mask[0].numel() > 2 ** 31
    mask.requires_grad_()
    g = torch.randn(N, D, f * H, f * W, device="cuda", generator=gen)
    out = flow_head.convex_upsample(flow, mask, f)
    out.backward(g)
    got = {"out": out.detach()[-1:], "dflow": flow.grad[-1:], "dmask": mask.grad[-1:]}
    del out
    worst = dict.fromkeys(TENSORS, 0.0)
    for lo in range(0, H, 64):
        hi = min(H, lo + 64)
        r0, r1 = max(0, lo - 1), min(H, hi + 1)
        fl, m, gg = flow.detach()[-1:, :, r0:r1], mask.detach()[-1:, :, r0:r1], g[-1:, :, f * r0:f * r1]
        o, df, dm = ft.forward_and_grads(fl, m, f, gg)
        b = ft.bounds(fl, m, f, gg)
        a, z = lo - r0, hi - r0
        pairs = {"out": (got["out"][:, :, f * lo:f * hi], o[:, :, f * a:f * z], b["out"][:, :, f * a:f * z]),
                 "dflow": (got["dflow"][:, :, lo:hi], df[:, :, a:z], b["dflow"][:, :, a:z]),
                 "dmask": (got["dmask"][:, :, lo:hi], dm[:, :, a:z], b["dmask"][:, :, a:z])}
        for k, (x, want, bnd) in pairs.items():
            worst[k] = max(worst[k], ft.ratio(x, want, bnd))
    record("flow_head_fp64:f8-16x1x512x512-f16-int64", mask="f16", **worst)
    print(f"2^31+ mask elements, last batch element: utilisation {worst}")
    assert max(worst.values()) <= 1.0, worst


# ---- sequence loss ----------------------------------------------------------------------------------------------------

def _bits(t):
    return t.view(torch.int32)


@pytest.mark.parametrize("case", fc.LOSS, ids=lambda c: c.id)
def test_sequence_loss_vs_fp64(case):
    """The loss and the EPE mean within (P + 4) u relative of fp64 on the same fp32 differences; the 1px / 3px
    fractions exactly float(c) * (1 / float(count)), as torch's forward mean; the gradients exactly
    (w_i * fp32(1 / count)) * sign(p_i - gt) on the valid pixels and signed zeros elsewhere, as torch's CUDA mean
    backward (see test_cuda_mean_backward_scales_by_the_reciprocal_of_the_exact_count)."""
    preds, gt, valid = fc.loss_inputs(case, device="cuda")
    preds = [p.requires_grad_() for p in preds]
    loss, metrics = flow_head.sequence_loss(preds, gt, valid)
    loss.backward()
    want = ft.sequence_loss64([p.detach() for p in preds], gt, valid)
    tol = ft.loss_bound(case.P)
    r = {"loss": abs(float(loss.detach()) - float(want["loss"])) / (tol * float(want["loss"])),
         "epe": abs(metrics["train_epe"] - float(want["epe"])) / (tol * float(want["epe"]))}
    record("flow_head_fp64:loss-" + case.id, count=want["count"], **r)
    print(f"{case.id}: count {want['count']}, utilisation {r}")
    assert max(r.values()) <= 1.0, r
    assert metrics["train_1px"] == ft.fraction32(want["c1"], want["count"])
    assert metrics["train_3px"] == ft.fraction32(want["c3"], want["count"])
    inv = np.float32(1.0 / want["count"])
    v = valid >= 0.5
    for p, w in zip(preds, ft.weights32(case.P)):
        x = torch.where(v, torch.tensor(float(np.float32(w) * inv), device="cuda"), torch.zeros((), device="cuda"))
        sg = torch.sign(p.detach() - gt.float())
        assert torch.equal(_bits(p.grad), _bits(x * sg))


def _counts_where_reciprocals_differ(n=6, seed=0):
    """Odd valid counts in (2^24, 17 * 2^20) where fp32(1 / count) and 1 / fp32(count) are different fp32 values."""
    rng, out = np.random.default_rng(seed), []
    while len(out) < n:
        c = int(rng.integers(2 ** 24 + 1, 17 * 2 ** 20)) | 1
        if np.float32(1.0 / c) != np.float32(1) / np.float32(c):
            out.append(c)
    return out


COUNTS = _counts_where_reciprocals_differ()


def _count_inputs(count, P=3):
    """P predictions of [1, 1, 1, 17 * 2^20] with exactly `count` valid pixels."""
    M = 17 * 2 ** 20
    gen = torch.Generator(device="cuda").manual_seed(count)
    gt = torch.rand(1, 1, 1, M, device="cuda", generator=gen) * -40
    valid = torch.zeros(1, 1, 1, M, device="cuda")
    valid.view(-1)[:count] = 1.0
    gt[valid < 0.5] = float("inf")
    fin = gt.nan_to_num(posinf=0.0)
    preds = [(fin + torch.randn(gt.shape, device="cuda", generator=gen)).requires_grad_() for _ in range(P)]
    return preds, gt, valid


@pytest.mark.parametrize("count", COUNTS)
def test_cuda_mean_backward_scales_by_the_reciprocal_of_the_exact_count(count):
    """What the kernel's backward follows: torch's CUDA mean backward multiplies by fp32(1 / count), the reciprocal of
    the exact integer count, not by 1 / fp32(count) (the CPU's value; the two differ at these counts, all above 2^24).
    The kernel's gradients are (w_i * fp32(1 / count)) * sign(p_i - gt) at each of them."""
    x = torch.zeros(17 * 2 ** 20, device="cuda", requires_grad=True)
    v = torch.zeros_like(x, dtype=torch.bool)
    v[:count] = True
    x[v].mean().backward()
    assert float(x.grad[0]) == float(np.float32(1.0 / count)) != float(np.float32(1) / np.float32(count))
    preds, gt, valid = _count_inputs(count)
    loss, _ = flow_head.sequence_loss(preds, gt, valid)
    loss.backward()
    inv = np.float32(1.0 / count)
    for p, w in zip(preds, ft.weights32(len(preds))):
        x = torch.where(valid >= 0.5, torch.tensor(float(np.float32(w) * inv), device="cuda"),
                        torch.zeros((), device="cuda"))
        assert torch.equal(_bits(p.grad), _bits(x * torch.sign(p.detach() - gt)))


@needs_ref
@pytest.mark.parametrize("count", COUNTS)
def test_sequence_loss_grads_above_2_24_valid_pixels_match_the_reference(count):
    """At odd valid counts above 2^24 (a stage-1 batch of 8 at 1024^2 reaches them) the gradients stay bit-identical
    to the reference's own function on the device."""
    preds, gt, valid = _count_inputs(count)
    loss, _ = flow_head.sequence_loss(preds, gt, valid)
    loss.backward()
    ours = [p.grad.clone() for p in preds]
    for p in preds:
        p.grad = None
    harness.add_reference_to_path()
    import lib.loss
    ref_loss, _ = patch.original(lib.loss, "sequence_loss")(preds, gt, valid)
    ref_loss.backward()
    for a, p in zip(ours, preds):
        assert torch.equal(_bits(a), _bits(p.grad))
