"""The disparity head without a GPU: the numpy oracle against the reference's own upsample_flow / sequence_loss
(tests/golden/flow_head_golden.npz), the exported ABI, and the GPSG_FLOW_HEAD switch of the patch."""
import os
import sys
import types

import numpy as np
import pytest
import torch

from gps_gaussian_b200 import harness, patch
from oracle import flow_head_oracle as fo

GOLDEN = np.load(os.path.join(os.path.dirname(__file__), "golden", "flow_head_golden.npz"))
UP = sorted({k[3:-len("_factor")] for k in GOLDEN.files if k.startswith("up_") and k.endswith("_factor")})
SL = sorted({k[3:-len("_raises")] for k in GOLDEN.files if k.startswith("sl_") and k.endswith("_raises")})
needs_ref = pytest.mark.skipif(harness.staged_reference() is None, reason="oracle/_ref not staged")

# Bounds relative to the largest |value| of each golden array.  fp64: the oracle restates the maths, so only rounding
# of fp64 re-association remains.  fp32: exp differs between numpy and torch's vectorised CPU kernel by a few ulps and
# the sums re-associate: 2^-17 (~8 ulps of the largest term) is far above that and far below any formula error.  fp16
# mask: a weight or dL/dweight within an ulp of an fp16 rounding boundary may round the other way, one fp16 ulp (2^-11),
# times the 9 taps: 9 * 2^-11.
BOUND = {"f64": 1e-12, "f32": 2.0 ** -17, "f16": 9 * 2.0 ** -11}


def up(name, key):
    return GOLDEN[f"up_{name}_{key}"]


def _kind(name):
    return name.rsplit("_", 1)[1]


def _close(got, want, rel, what):
    nan = np.isnan(want)
    assert np.array_equal(np.isnan(got), nan), (what, "NaN positions differ")
    scale = max(1.0, float(np.abs(want[~nan]).max())) if (~nan).any() else 1.0
    err = float(np.abs(got[~nan].astype(np.float64) - want[~nan]).max()) if (~nan).any() else 0.0
    assert err <= rel * scale, (what, err, rel * scale)


@pytest.mark.parametrize("name", UP)
def test_oracle_upsample_equals_golden(name):
    f = int(up(name, "factor"))
    kind = _kind(name)
    dtype = None if kind == "f64" else (np.float16 if kind == "f16" else np.float32)
    flow, mask = up(name, "flow"), up(name, "mask")
    _close(fo.convex_upsample(flow, mask, f, dtype), up(name, "out"), BOUND[kind], "out")
    dflow, dmask = fo.convex_upsample_backward(flow, mask, f, up(name, "g"), dtype)
    assert dmask.dtype == up(name, "d_mask").dtype
    _close(dflow, up(name, "d_flow"), BOUND[kind], "d_flow")
    _close(dmask.astype(np.float64), up(name, "d_mask").astype(np.float64), BOUND[kind], "d_mask")


def test_goldens_cover_the_issue_cases():
    assert {int(up(n, "factor")) for n in UP} == {2, 4, 8}
    assert {_kind(n) for n in UP} == {"f64", "f32", "f16"}
    assert any(up(n, "flow").shape[-1] == 1 for n in UP) and any(up(n, "flow").shape[1] == 1 for n in UP)
    assert any(np.abs(up(n, "flow")[:, 1:]).max() > 0 for n in UP if up(n, "flow").shape[1] == 2)
    assert any(np.isnan(up(n, "out")).any() for n in UP) and any(np.isneginf(up(n, "mask")).any() for n in UP)
    assert any(up(n, "mask").max() > 88 for n in UP)                  # exp overflows fp32 without the max subtraction
    assert {str(GOLDEN[f"sl_{n}_raises"]) for n in SL} == {"", "AssertionError", "ZeroDivisionError"}


@pytest.mark.parametrize("name", SL)
def test_oracle_sequence_loss_equals_golden(name):
    sl = lambda k: GOLDEN[f"sl_{name}_{k}"]
    preds = list(sl("preds"))
    raises = str(sl("raises"))
    if raises == "ZeroDivisionError":
        with pytest.raises(ZeroDivisionError):
            fo.sequence_loss(preds, sl("gt"), sl("valid"))
        return
    loss, metrics, grads, inf = fo.sequence_loss(preds, sl("gt"), sl("valid"))
    assert inf == (raises == "AssertionError")
    if inf:
        return
    m = np.array([metrics["train_epe"], metrics["train_1px"], metrics["train_3px"]])
    g = float(sl("g"))
    if np.isnan(sl("loss_f64")):
        assert np.isnan(loss) and np.isnan(m).all() and np.isnan(sl("metrics_f32")).all()
        assert not np.any(sl("grads_f64")) and not np.any(sl("grads_f32"))
        return
    assert abs(loss - sl("loss_f64")) <= 1e-12 * abs(sl("loss_f64"))
    # the reference takes (epe < t).float().mean(): an fp32 fraction even in the fp64 run
    assert np.allclose(m, sl("metrics_f64"), rtol=[1e-12, 2.0 ** -24, 2.0 ** -24], atol=0)
    assert np.allclose(np.stack(grads) * g, sl("grads_f64"), rtol=1e-12, atol=0)
    # the fp32 reference: the counts are exact, sums re-associate
    assert abs(loss - sl("loss_f32")) <= 1e-6 * abs(loss)
    assert np.allclose(m, sl("metrics_f32"), rtol=1e-6, atol=0)
    assert np.allclose(np.stack(grads) * g, sl("grads_f32"), rtol=1e-6, atol=0)


def test_abi_exports(built_lib):
    import ctypes as C
    from gps_gaussian_b200 import _lib
    for name in ("gpsg_convex_upsample_forward", "gpsg_convex_upsample_backward_workspace_bytes",
                 "gpsg_convex_upsample_backward", "gpsg_sequence_loss_workspace_bytes", "gpsg_sequence_loss_forward",
                 "gpsg_sequence_loss_backward"):
        assert name in _lib.EXPORTED and hasattr(C.CDLL(built_lib), name)
    assert _lib.lib.gpsg_convex_upsample_backward_workspace_bytes(2, 2, 3, 4) == 2 * 2 * 9 * 3 * 4 * 4
    assert C.sizeof(_lib.SeqLossArgs) == 32 * 8 * 2 + 32 * 4 + 8 * 3 + 8


def test_abi_refuses_bad_arguments():
    from gps_gaussian_b200 import _lib
    L = _lib.lib
    p = _lib.C.c_void_p(16)
    for dtype, f, D in ((2, 8, 2), (0, 3, 2), (0, 16, 2), (0, 8, 3), (0, 8, 0)):
        assert L.gpsg_convex_upsample_forward(0, None, dtype, f, 1, D, 4, 4, p, p, p) == -1
    assert L.gpsg_convex_upsample_forward(0, None, 0, 8, 1, 2, 4, 4, None, p, p) == -1
    assert L.gpsg_convex_upsample_backward(0, None, 0, 8, 1, 2, 4, 4, p, p, p, None, None, p) == -1
    assert L.gpsg_convex_upsample_backward(0, None, 0, 8, 1, 2, 4, 4, p, p, p, None, p, None) == -1
    a = _lib.SeqLossArgs()
    a.n_pred, a.numel = 0, 4
    assert L.gpsg_sequence_loss_forward(0, None, a, p, p) == -1
    a.n_pred = 33
    assert L.gpsg_sequence_loss_forward(0, None, a, p, p) == -1
    a.n_pred, a.gt, a.valid = 2, 16, 16
    a.pred[0] = 16
    assert L.gpsg_sequence_loss_forward(0, None, a, p, p) == -1           # pred[1] is NULL
    a.pred[1], a.gt_dtype = 16, 2
    assert L.gpsg_sequence_loss_forward(0, None, a, p, p) == -1           # gt_dtype neither fp32 nor fp16


def test_direct_api_refuses_what_it_does_not_cover():
    from gps_gaussian_b200 import flow_head
    flow, mask = torch.zeros(1, 2, 3, 4), torch.zeros(1, 576, 3, 4)
    with pytest.raises(RuntimeError, match="convex_upsample"):
        flow_head.convex_upsample(flow, mask, 8)                            # CPU tensors
    assert not flow_head.upsample_supported(flow, mask.to(torch.bfloat16), 8)
    assert not flow_head.upsample_supported(flow.half(), mask, 8)
    assert not flow_head.upsample_supported(flow, torch.zeros(1, 9 * 16 * 16, 3, 4), 16)
    gt = torch.zeros(2, 1, 3, 4)
    assert not flow_head.sequence_loss_supported([gt, gt], gt, gt)             # CPU tensors


# ---- the GPSG_FLOW_HEAD switch ---------------------------------------------------------------------------------------

@pytest.fixture
def clean_patch():
    patch.uninstall()
    yield
    patch.uninstall()


def _fake_modules(monkeypatch):
    raft = types.ModuleType("core.raft_stereo_human")

    class FlowUpdateModule:
        def upsample_flow(self, flow, mask):
            return "reference"
    raft.FlowUpdateModule = FlowUpdateModule
    loss = types.ModuleType("lib.loss")
    loss.sequence_loss = lambda *a, **k: "reference"
    net = types.ModuleType("lib.network")
    net.sequence_loss = loss.sequence_loss
    for name, mod in (("core.raft_stereo_human", raft), ("lib.loss", loss), ("lib.network", net)):
        monkeypatch.setitem(sys.modules, name, mod)
    return raft, loss, net


@pytest.mark.parametrize("value", [None, "0", "1"])
def test_switch_binds_only_when_set(monkeypatch, clean_patch, value):
    raft, loss, net = _fake_modules(monkeypatch)
    orig_up, orig_loss = raft.FlowUpdateModule.__dict__["upsample_flow"], loss.sequence_loss
    if value is None:
        monkeypatch.delenv("GPSG_FLOW_HEAD", raising=False)
    else:
        monkeypatch.setenv("GPSG_FLOW_HEAD", value)
    patch.install()
    bound = value == "1"
    assert patch.flow_head() is bound
    from gps_gaussian_b200 import flow_head
    assert (raft.FlowUpdateModule.__dict__["upsample_flow"] is not orig_up) is bound
    assert (loss.sequence_loss is flow_head.sequence_loss) is bound
    assert (net.sequence_loss is flow_head.sequence_loss) is bound
    patch.uninstall()
    assert raft.FlowUpdateModule.__dict__["upsample_flow"] is orig_up
    assert loss.sequence_loss is orig_loss and net.sequence_loss is orig_loss


def test_uninstall_restores_a_copy_made_after_install(monkeypatch, clean_patch):
    raft, loss, net = _fake_modules(monkeypatch)
    orig = loss.sequence_loss
    monkeypatch.delitem(sys.modules, "lib.network")
    monkeypatch.setenv("GPSG_FLOW_HEAD", "1")
    patch.install()
    from gps_gaussian_b200 import flow_head
    assert loss.sequence_loss is flow_head.sequence_loss
    net.sequence_loss = loss.sequence_loss                      # lib.network imported after install(): `from lib.loss import`
    monkeypatch.setitem(sys.modules, "lib.network", net)
    patch.uninstall()
    assert loss.sequence_loss is orig and net.sequence_loss is orig


def test_cpu_tensors_reach_the_reference_functions(monkeypatch, clean_patch):
    raft, loss, net = _fake_modules(monkeypatch)
    monkeypatch.setenv("GPSG_FLOW_HEAD", "1")
    patch.install()
    me = raft.FlowUpdateModule()
    me.args = types.SimpleNamespace(n_downsample=3)
    assert me.upsample_flow(torch.zeros(1, 2, 3, 4), torch.zeros(1, 576, 3, 4)) == "reference"
    assert net.sequence_loss([torch.zeros(1, 1, 2, 2)] * 2, torch.zeros(1, 1, 2, 2), torch.ones(1, 1, 2, 2)) == "reference"


_PROBE = ("import core.raft_stereo_human as r, lib.network as n, lib.loss as l\n"
          "print(r.FlowUpdateModule.upsample_flow.__module__, n.sequence_loss.__module__, l.sequence_loss.__module__)\n")


@needs_ref
@pytest.mark.parametrize("on", [False, True])
def test_unmodified_modules_with_patch(on):
    import subprocess
    env = harness.script_env(patch=True, extra={"GPSG_FLOW_HEAD": "1"} if on else None)
    if not on:
        env.pop("GPSG_FLOW_HEAD", None)
    p = subprocess.run([sys.executable, "-c", _PROBE], cwd=harness.staged_reference(), env=env, text=True,
                       capture_output=True, timeout=300)
    assert p.returncode == 0, p.stderr[-3000:]
    mods = p.stdout.split()
    want = "gps_gaussian_b200.flow_head" if on else None
    assert mods == ([want] * 3 if on else ["core.raft_stereo_human", "lib.loss", "lib.loss"]), mods
