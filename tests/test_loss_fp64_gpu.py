"""GPU: the fused L1 + SSIM loss (csrc/loss.cu through gps_gaussian_b200.loss) against the fp64 restatement
(oracle/loss_torch64.py) over tests/loss_cases.SWEEP: every (H, W) in {1, 5, 6, 11, 31, 32, 33, 37, 69}^2 (so every
combination of the 32-px tile and the 5-px halo), planes 1, 3, 6 and 96, flat, flat-bright, zero-variance, tied,
noisy, smooth and [-1, 1] content; and at 1024^2, 1024x512 and 512x1024.

Checked per element against the bounds of `loss_torch64.bounds` (constants fixed from the reference's fp32 chain on the
CPU): the loss, L1, SSIM and ssim(size_average=False); the three per-pixel partials the forward stores, read through
gpsg_l1_ssim_forward for (img, gt) and for (gt, img); and the gradients w.r.t. img and gt, both requiring grad.
tests/test_loss_torch64_cpu.py shows that each mutant of the restatement breaks one of these on this sweep."""
import ctypes as C
import functools

import pytest
import torch

import loss_cases as lc

pytestmark = pytest.mark.gpu


@functools.lru_cache(maxsize=8)
def _case(case):
    img, gt = map(torch.from_numpy, lc.image_pair(*case))
    return img, gt, lc.reference(img, gt)


def _dmaps(a, b):
    """[3,P,H,W] partials the forward stores for d/d a, through the C ABI."""
    from gps_gaussian_b200 import _lib
    H, W = a.shape[-2:]
    P = a.numel() // (H * W)
    maps = torch.full((3,) + tuple(a.shape), float("nan"), device="cuda")
    out = torch.empty(3, device="cuda")
    ws = torch.empty(int(_lib.lib.gpsg_l1_ssim_workspace_bytes(P, H, W)), dtype=torch.uint8, device="cuda")
    p = lambda t: C.c_void_p(t.data_ptr())
    rc = _lib.lib.gpsg_l1_ssim_forward(*_lib.device_stream(a.device), P, H, W, p(a), p(b), 0.8, 0.2, p(out), p(maps),
                                       p(ws))
    _lib.check(rc, "gpsg_l1_ssim_forward")
    return maps


def _device(img, gt):
    from gps_gaussian_b200.loss import fused_l1_ssim, ssim
    x, y = img.cuda().requires_grad_(True), gt.cuda().requires_grad_(True)
    loss = fused_l1_ssim(x, y)
    loss.backward()
    xd, yd = x.detach().contiguous(), y.detach().contiguous()
    return {"loss": loss.detach(), "l1": loss.l1, "ssim": loss.ssim, "ssim_per_image": ssim(xd, yd, size_average=False),
            "dmaps_img": _dmaps(xd, yd), "dmaps_gt": _dmaps(yd, xd), "grad_img": x.grad, "grad_gt": y.grad}


def _check(case):
    img, gt, ref = _case(case)
    got = _device(img, gt)
    for k in ("grad_img", "grad_gt"):
        assert got[k].dtype == torch.float32 and got[k].shape == img.shape
    r = lc.ratios(ref, got)
    print(f"{lc.case_id(case)}: utilisation {r}")
    assert max(r.values()) <= 1.0, r


@pytest.mark.parametrize("case", lc.SWEEP, ids=lc.case_id)
def test_sweep_vs_fp64(case):
    _check(case)


@pytest.mark.parametrize("case", lc.LARGE, ids=lc.case_id)
def test_full_size_vs_fp64(case):
    _check(case)


@pytest.mark.parametrize("dtype", (torch.float16, torch.bfloat16, torch.float64, "strided"))
def test_dtypes_and_layouts_match_the_fp32_contiguous_result(dtype):
    """fp16 / bf16 / fp64 inputs, and a channel slice of a [B,4,H,W] render buffer, give the loss and gradients of
    their contiguous fp32 copy, with the gradients in the input's dtype."""
    from gps_gaussian_b200.loss import fused_l1_ssim
    img, gt = map(torch.from_numpy, lc.image_pair("smooth", (2, 3, 37, 69), 9))
    if dtype == "strided":
        buf = torch.rand(2, 4, 37, 69, device="cuda")
        bg = torch.rand(2, 4, 37, 69, device="cuda")
        buf[:, 1:], bg[:, 1:] = img.cuda(), gt.cuda()
        x, y = buf[:, 1:], bg[:, 1:]
        assert not x.is_contiguous()
    else:
        x, y = img.cuda().to(dtype), gt.cuda().to(dtype)
    x, y = x.detach().requires_grad_(True), y.detach().requires_grad_(True)
    x32 = x.detach().float().contiguous().requires_grad_(True)
    y32 = y.detach().float().contiguous().requires_grad_(True)
    l, l32 = fused_l1_ssim(x, y), fused_l1_ssim(x32, y32)
    l.backward()
    l32.backward()
    assert torch.equal(l.detach(), l32.detach())
    want_dt = torch.float32 if dtype == "strided" else dtype
    for g, g32 in ((x.grad, x32.grad), (y.grad, y32.grad)):
        assert g.dtype == want_dt and g.shape == x.shape
        assert torch.equal(g, g32.to(want_dt))


def test_grid_limit_raises():
    """planes > 65535 does not fit the launch grid: refused with an error, not launched."""
    from gps_gaussian_b200.loss import fused_l1_ssim
    x = torch.rand(65536, 1, 1, device="cuda", requires_grad=True)
    with pytest.raises(RuntimeError):
        fused_l1_ssim(x, torch.rand(65536, 1, 1, device="cuda"))
    torch.cuda.synchronize()
