"""GPU: the fused unprojection (csrc/unproject.cu through gps_gaussian_b200.unproject) against the fp64 restatement
(oracle/unproject_torch64.py) over tests/unproject_cases.SWEEP: B in {1, 2, 4}, S in {1, 7, 24, 255, 256, 257, 1024},
masks with C in {1, 3} that are binary, soft or all zero, [B,3,4] and [B,4,4] extrinsics, both signs of Tf_x,
per-item ref_intr offsets and pixels with flow == offset exactly.

  * depth and pts_valid are bit-identical to the reference's fp32 op order (a subtraction, a negation, an IEEE
    division and a multiplication, none of them contractible into an FMA);
  * xyz, at valid and invalid (1e8-scaled) pixels alike, is within K_XYZ 2^-24 (|R^T| |p| + |R^T| |t|) of fp64;
  * d/d flow, for a loss on xyz only, on depth only and on both, is within K_GRAD 2^-24 of fp64 times the magnitude
    of its terms, and exactly 0 wherever the mask is 0.
tests/test_unproject_torch64_cpu.py shows that each mutant of the restatement breaks one of these on this sweep."""
import ctypes as C
import functools

import pytest
import torch

import unproject_cases as uc

pytestmark = pytest.mark.gpu


@functools.lru_cache(maxsize=None)
def _case(case):
    inp = uc.make_case(*case)
    return inp, uc.reference(inp)


def _view(inp, flow):
    d = lambda k: inp[k].cuda()
    return {"flow_pred": flow, "mask": d("mask"), "intr": d("intr"), "extr": d("extr"), "ref_intr": d("ref_intr"),
            "Tf_x": d("tf_x")}


def _device(inp, mode, flow=None):
    """(depth, xyz, valid, d/d flow) from the binding, with the loss on xyz, depth or both."""
    from gps_gaussian_b200.unproject import unproject_view
    flow = (inp["flow"].cuda() if flow is None else flow).detach().requires_grad_(True)
    depth, xyz, valid = unproject_view(_view(inp, flow))
    loss = 0.0
    if mode in ("xyz", "both"):
        loss = loss + (xyz * inp["g_xyz"].cuda()).sum()
    if mode in ("depth", "both"):
        loss = loss + (depth * inp["g_depth"].cuda()).sum()
    loss.backward()
    return depth.detach(), xyz.detach(), valid, flow.grad


def _check(case, got):
    r = uc.ratios(_case(case)[1], got)
    print(f"{uc.case_id(case)}: utilisation {r}")
    assert max(r.values()) <= 1.0, r
    return r


@pytest.mark.parametrize("case", uc.SWEEP, ids=uc.case_id)
def test_forward_bit_identical_depth_and_bounded_xyz(case):
    depth, xyz, valid, _ = _device(_case(case)[0], "both")
    assert bool(torch.isfinite(xyz).all())                        # invalid pixels carry finite 1e8-scaled points
    _check(case, {"depth": depth, "valid": valid, "xyz": xyz})


@pytest.mark.parametrize("case", uc.SWEEP, ids=uc.case_id)
def test_gradient_loss_on_xyz_only(case):
    _check(case, {"grad_xyz": _device(_case(case)[0], "xyz")[3]})


@pytest.mark.parametrize("case", uc.SWEEP, ids=uc.case_id)
def test_gradient_loss_on_depth_only(case):
    _check(case, {"grad_depth": _device(_case(case)[0], "depth")[3]})


@pytest.mark.parametrize("case", uc.SWEEP, ids=uc.case_id)
def test_gradient_loss_on_both(case):
    _check(case, {"grad_both": _device(_case(case)[0], "both")[3]})


@pytest.mark.parametrize("case", [c for c in uc.SWEEP if c[3] in ("binary", "zero")], ids=uc.case_id)
def test_zero_gradient_at_mask_zero(case):
    inp = _case(case)[0]
    m0 = (inp["mask"][:, :1] == 0).cuda()
    for mode in uc.GRAD_MODES:
        g = _device(inp, mode)[3]
        assert int((g[m0] != 0).sum()) == 0, mode


def test_noncontiguous_and_fp16_flow_match_their_fp32_copy():
    """A channel slice of a [B,3,S,S] buffer, and fp16 flow, give what their contiguous fp32 copy gives, bit for bit;
    the gradient comes back in the input's dtype."""
    inp = _case(uc.SWEEP[10])[0]
    B, _, S, _ = inp["flow"].shape
    want = _device(inp, "both")
    buf = torch.randn(B, 3, S, S, device="cuda")
    buf[:, 1:2] = inp["flow"].cuda()
    sl = buf[:, 1:2]
    assert not sl.is_contiguous()
    got = _device(inp, "both", sl)
    for a, b in zip(got, want):
        assert torch.equal(a, b)
    h = inp["flow"].cuda().half()
    want16 = _device(inp, "both", h.float())
    got16 = _device(inp, "both", h)
    assert got16[3].dtype == torch.float16
    for a, b in zip(got16[:3], want16[:3]):
        assert torch.equal(a, b)
    assert torch.equal(got16[3], want16[3].half())


@pytest.mark.parametrize("which", ("xyz", "depth"))
def test_c_abi_backward_takes_null_incoming_gradients(which):
    """gpsg_unproject_backward with dL_ddepth (or dL_dxyz) NULL == the fp64 gradient of the loss on the other output."""
    from gps_gaussian_b200 import _lib
    case = uc.SWEEP[11]
    inp = _case(case)[0]
    depth = _device(inp, "both")[0]
    d = {k: inp[k].cuda().contiguous() for k in inp}
    B, _, S, _ = d["mask"].shape
    out = torch.full((B, 1, S, S), float("nan"), device="cuda")
    p = lambda t: C.c_void_p(t.data_ptr()) if t is not None else None
    gx, gd = (d["g_xyz"], None) if which == "xyz" else (None, d["g_depth"])
    rc = _lib.lib.gpsg_unproject_backward(*_lib.device_stream(out.device), B, S, p(depth), p(d["mask"]),
                                          int(d["mask"].stride(0)), p(d["intr"]), p(d["extr"]), int(d["extr"].shape[1]),
                                          p(d["ref_intr"]), p(d["tf_x"]), p(gx), p(gd), p(out))
    _lib.check(rc, "gpsg_unproject_backward")
    _check(case, {"grad_" + which: out})
    rc = _lib.lib.gpsg_unproject_backward(*_lib.device_stream(out.device), B, S, p(depth), p(d["mask"]),
                                          int(d["mask"].stride(0)), p(d["intr"]), p(d["extr"]), int(d["extr"].shape[1]),
                                          p(d["ref_intr"]), p(d["tf_x"]), None, None, p(out))
    assert rc != 0                                                     # no incoming gradient at all is refused


@pytest.mark.parametrize("bad", ("intr", "ref_intr", "extr", "tf_x", "mask_rows", "mask_batch", "flow_channels"))
def test_misshaped_inputs_raise_before_any_launch(bad):
    from gps_gaussian_b200.unproject import unproject_view
    inp = _case(uc.SWEEP[7])[0]                                       # B = 2, S = 24
    view = _view(inp, inp["flow"].cuda())
    if bad in ("intr", "ref_intr", "extr"):
        view[bad] = view[bad][:1]
    elif bad == "tf_x":
        view["Tf_x"] = view["Tf_x"][:1]
    elif bad == "mask_rows":
        view["mask"] = view["mask"][:, :, :-1]
    elif bad == "mask_batch":
        view["mask"] = view["mask"][:1]
    else:
        view["flow_pred"] = view["flow_pred"].repeat(1, 2, 1, 1)
    torch.cuda.synchronize()
    with pytest.raises(RuntimeError):
        unproject_view(view)
    torch.cuda.synchronize()
