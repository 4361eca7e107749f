"""CPU: the encoder-stem entry points are exported and declared, the GPSG_ENCODER switch hooks core.extractor only when
set to 1 and uninstall() restores UnetExtractor.forward, and the rebound forward sends what the kernels do not cover to
the reference's own method."""
import ctypes as C
import os
import re
import sys
import types

import pytest
import torch

from gps_gaussian_b200 import _lib, encoder, harness, patch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SYMBOLS = ("gpsg_encoder_stem_workspace_bytes", "gpsg_encoder_stem_forward")


def test_symbols_exported_and_declared():
    header = open(os.path.join(ROOT, "include", "gpsg.h")).read()
    for name in SYMBOLS:
        assert name in _lib.EXPORTED and hasattr(_lib.lib, name)
        assert re.search(r"GPSG_API\s+\w+\s+" + name + r"\(", header), name
    fields = re.search(r"typedef struct GpsgEncoderStemWeights \{(.*?)\}", header, re.S).group(1)
    assert re.findall(r"const float\* (\w+);", fields) == list(_lib.ENCODER_STEM_PARAMS)
    assert len(_lib.ENCODER_STEM_PARAMS) == 20


def test_workspace_bytes_and_refusals():
    f = _lib.lib.gpsg_encoder_stem_workspace_bytes
    assert f(2, 3, 1024, 1024, 0) >= 5 * 2 * 512 * 512 * 32 * 4
    assert f(2, 3, 1024, 1024, 1) >= 5 * 2 * 512 * 512 * 32 * 2
    assert f(2, 3, 1024, 1024, 1) < f(2, 3, 1024, 1024, 0)
    assert f(2, 2, 16, 16, 0) == 0 and f(2, 3, 0, 16, 0) == 0 and f(2, 3, 16, 16, 7) == 0
    w = _lib.EncoderStemWeights()
    assert _lib.lib.gpsg_encoder_stem_forward(0, None, 1, 2, 8, 8, 0, None, w, None, None) != 0   # Cin 2
    assert _lib.lib.gpsg_encoder_stem_forward(0, None, 0, 3, 8, 8, 0, None, w, None, None) == 0   # B = 0: nothing


@pytest.fixture
def clean_patch():
    patch.uninstall()
    yield
    patch.uninstall()


def _fake_module(monkeypatch):
    mod = types.ModuleType("core.extractor")

    class UnetExtractor:
        def forward(self, x):
            return "reference"
    mod.UnetExtractor = UnetExtractor
    monkeypatch.setitem(sys.modules, "core.extractor", mod)
    return mod


@pytest.mark.parametrize("value", [None, "0", "true", "1"])
def test_switch_binds_only_when_set(monkeypatch, clean_patch, value):
    mod = _fake_module(monkeypatch)
    orig = mod.UnetExtractor.__dict__["forward"]
    if value is None:
        monkeypatch.delenv("GPSG_ENCODER", raising=False)
    else:
        monkeypatch.setenv("GPSG_ENCODER", value)
    patch.install()
    bound = value == "1"
    assert patch.encoder() is bound
    assert ("core.extractor" in patch._targets()) is bound
    assert (mod.UnetExtractor.__dict__["forward"] is not orig) is bound
    if bound:
        assert mod.UnetExtractor.forward.__module__ == encoder.__name__
        with torch.no_grad():                       # a module without the stem's layers: the reference answers
            assert mod.UnetExtractor().forward(torch.zeros(1, 3, 4, 4)) == "reference"
    patch.uninstall()
    assert mod.UnetExtractor.__dict__["forward"] is orig


def _extractor(**kw):
    harness.add_reference_to_path()
    from core.extractor import UnetExtractor
    torch.manual_seed(0)
    return UnetExtractor, UnetExtractor(**kw).eval()


needs_ref = pytest.mark.skipif(harness.staged_reference() is None, reason="oracle/_ref not staged")


@needs_ref
@pytest.mark.parametrize("what", ["grad", "cpu", "allow_tf32_off", "bf16_autocast"])
def test_fallbacks_without_a_device(what, monkeypatch):
    cls, m = _extractor(in_channel=3, encoder_dim=[32, 48, 96])
    fwd = encoder.make_extractor_forward(cls.forward)
    monkeypatch.setattr(encoder, "run", lambda *a: pytest.fail("the kernels ran"))
    x = torch.rand(1, 3, 16, 12)
    if what == "allow_tf32_off":
        monkeypatch.setattr(torch.backends.cudnn, "allow_tf32", False)
        assert encoder.precision_now() is None
    if what == "bf16_autocast":                   # CUDA autocast in bf16, as the dispatcher reports it on a device
        monkeypatch.setattr(torch, "is_autocast_enabled", lambda *a: True)
        monkeypatch.setattr(torch, "get_autocast_dtype", lambda *a: torch.bfloat16)
        assert encoder.precision_now() is None
    ctx = torch.enable_grad() if what == "grad" else torch.no_grad()
    with ctx:
        got, want = fwd(m, x), cls.forward(m, x)
    for g, w in zip(got, want):
        assert torch.equal(g, w)


@needs_ref
def test_supported_rejects_foreign_configurations():
    x = torch.zeros(1, 3, 8, 8)
    assert not encoder.supported(types.SimpleNamespace(), x)
    _, m = _extractor(in_channel=3, encoder_dim=[32, 48, 96])
    assert encoder._module_supported(m, 3) and not encoder._module_supported(m, 1)
    assert not encoder.supported(m, x)                                     # CPU input
    for kw in (dict(encoder_dim=[64, 96, 128]), dict(encoder_dim=[32, 48, 96], norm_fn="batch"),
               dict(encoder_dim=[32, 48, 96], norm_fn="instance")):
        assert not encoder._module_supported(_extractor(in_channel=3, **kw)[1], 3), kw
    _, m = _extractor(in_channel=3, encoder_dim=[32, 48, 96])
    m.res1[0].norm1.eps = 1e-6
    assert not encoder._module_supported(m, 3)
    _, m = _extractor(in_channel=3, encoder_dim=[32, 48, 96])
    m.in_ds[1] = torch.nn.GroupNorm(8, 32, affine=False)
    assert not encoder._module_supported(m, 3)
    _, m = _extractor(in_channel=3, encoder_dim=[32, 48, 96])
    m.in_ds[0].padding = (1, 1)
    assert not encoder._module_supported(m, 3)


def test_run_refuses_cpu_tensors():
    with pytest.raises(RuntimeError, match="encoder_stem"):
        encoder.run(torch.zeros(1, 3, 8, 8), [torch.zeros(s) for s in encoder.param_shapes(3)], "tf32")
    with pytest.raises(ValueError):
        encoder.run(torch.zeros(1, 3, 8, 8), [], "bf16")
