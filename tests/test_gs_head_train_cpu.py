"""CPU: the GPSG_GS_HEAD_TRAIN switch rebinds GSRegresser.forward with the training route only when set to 1, alone or
with GPSG_GS_HEAD, and uninstall() restores it; the training route sends CPU inputs to the reference's own method."""
import sys
import types

import pytest
import torch

from gps_gaussian_b200 import gs_head, patch


@pytest.fixture
def clean_patch():
    patch.uninstall()
    yield
    patch.uninstall()


def _fake_module(monkeypatch):
    mod = types.ModuleType("lib.gs_parm_network")

    class GSRegresser:
        def forward(self, img, depth, img_feat):
            return "reference"
    mod.GSRegresser = GSRegresser
    monkeypatch.setitem(sys.modules, "lib.gs_parm_network", mod)
    return mod


@pytest.mark.parametrize("value", [None, "0", "true", "1"])
@pytest.mark.parametrize("forward_switch", [False, True])
def test_train_switch_binds_only_when_set(monkeypatch, clean_patch, value, forward_switch):
    mod = _fake_module(monkeypatch)
    orig = mod.GSRegresser.__dict__["forward"]
    if value is None:
        monkeypatch.delenv("GPSG_GS_HEAD_TRAIN", raising=False)
    else:
        monkeypatch.setenv("GPSG_GS_HEAD_TRAIN", value)
    if forward_switch:
        monkeypatch.setenv("GPSG_GS_HEAD", "1")
    else:
        monkeypatch.delenv("GPSG_GS_HEAD", raising=False)
    patch.install()
    train = value == "1"
    assert patch.gs_head_train() is train and patch.gs_head() is forward_switch
    assert (mod.GSRegresser.__dict__["forward"] is not orig) is (train or forward_switch)
    if train or forward_switch:
        assert mod.GSRegresser.forward.__module__ == gs_head.__name__
        for grad in (False, True):
            with torch.set_grad_enabled(grad):
                assert mod.GSRegresser().forward(torch.zeros(1, 3, 4, 4), torch.zeros(1, 1, 4, 4), [None] * 3) == "reference"
    patch.uninstall()
    assert mod.GSRegresser.__dict__["forward"] is orig


def test_gs_head_train_refuses_cpu_and_foreign_modules():
    img, depth = torch.zeros(1, 3, 8, 8), torch.zeros(1, 1, 8, 8)
    with pytest.raises(RuntimeError, match="gs_head"):
        gs_head.gs_head_train(torch.zeros(1, 48, 4, 4), img, depth, types.SimpleNamespace())
    with pytest.raises(RuntimeError, match="gs_head"):
        gs_head.backward(torch.zeros(1, 48, 4, 4), img, depth, [torch.zeros(s) for s in gs_head.PARAM_SHAPES],
                         torch.zeros(1), torch.zeros(1, 4, 8, 8), torch.zeros(1, 3, 8, 8), torch.zeros(1, 1, 8, 8))


def test_backward_argument_validation_without_gpu():
    """Error paths of gpsg_gs_head_backward return codes and messages and never touch the device."""
    from gps_gaussian_b200 import _lib
    w = _lib.GsHeadWeights(*([8] * 14))
    g = _lib.GsHeadGrads(*([16] * 14))
    call = lambda B, H, W, ptrs, gr=g, ws=16: _lib.lib.gpsg_gs_head_backward(0, None, B, H, W, *ptrs, w, gr, ws)
    ok = [16] * 7 + [None, None]
    assert call(1, 7, 8, ok) == -1 and b"even" in _lib.lib.gpsg_last_error()
    assert call(1, 8, 8, [16, 16, 16, None] + ok[4:]) == -1 and b"NULL" in _lib.lib.gpsg_last_error()
    assert call(1, 8, 8, ok, gr=_lib.GsHeadGrads(*([16] * 13 + [0]))) == -1
    assert b"gradient" in _lib.lib.gpsg_last_error()
    assert call(1, 8, 8, ok, ws=8) == -1 and b"aligned" in _lib.lib.gpsg_last_error()
    assert call(1, 8, 8, [16, 16, 16, 8] + ok[4:]) == -1 and b"aligned" in _lib.lib.gpsg_last_error()
    assert call(0, 8, 8, [None] * 9, ws=None) == 0
    assert _lib.lib.gpsg_gs_head_backward_workspace_bytes(0, 8, 8) == 0
    assert _lib.lib.gpsg_gs_head_backward_workspace_bytes(2, 8, 16) >= 2 * 8 * 16 * 128 * 4
