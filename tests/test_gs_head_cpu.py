"""CPU: the GPSG_GS_HEAD switch rebinds GSRegresser.forward only when set to 1 and uninstall() restores it; the rebound
forward and `supported` send CPU inputs to the reference's own method."""
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
def test_switch_binds_only_when_set(monkeypatch, clean_patch, value):
    mod = _fake_module(monkeypatch)
    orig = mod.GSRegresser.__dict__["forward"]
    if value is None:
        monkeypatch.delenv("GPSG_GS_HEAD", raising=False)
    else:
        monkeypatch.setenv("GPSG_GS_HEAD", value)
    patch.install()
    bound = value == "1"
    assert patch.gs_head() is bound
    assert (mod.GSRegresser.__dict__["forward"] is not orig) is bound
    if bound:
        assert mod.GSRegresser.forward.__module__ == gs_head.__name__
        # CPU inputs and a module without the expected layers: the reference's method answers
        assert mod.GSRegresser().forward(torch.zeros(1, 3, 4, 4), torch.zeros(1, 1, 4, 4), [None] * 3) == "reference"
    patch.uninstall()
    assert mod.GSRegresser.__dict__["forward"] is orig


def test_supported_refuses_cpu_and_foreign_modules():
    img, depth = torch.zeros(1, 3, 8, 8), torch.zeros(1, 1, 8, 8)
    assert not gs_head.supported(types.SimpleNamespace(), img, depth, None)
    with pytest.raises(RuntimeError, match="gs_head"):
        gs_head.run(torch.zeros(1, 48, 4, 4), img, depth, [torch.zeros(s) for s in gs_head.PARAM_SHAPES])
