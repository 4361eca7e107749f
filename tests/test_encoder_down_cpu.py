"""CPU: the res2 / res3 entry points are exported and declared, their workspace sizes and refusals, the parameter order
against the reference's own ResidualBlocks, `down_supported` and the deep route's res2 / res3 checks on foreign
modules, and the GPSG_ENCODER_DEEP switch: alone it does nothing, GPSG_ENCODER=1 alone binds the shallow forward as before."""
import os
import re
import sys
import types

import pytest
import torch

from gps_gaussian_b200 import _lib, encoder, harness, patch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SYMBOLS = ("gpsg_encoder_down_workspace_bytes", "gpsg_encoder_down_forward")
needs_ref = pytest.mark.skipif(harness.staged_reference() is None, reason="oracle/_ref not staged")


def test_symbols_exported_and_declared():
    header = open(os.path.join(ROOT, "include", "gpsg.h")).read()
    for name in SYMBOLS:
        assert name in _lib.EXPORTED and hasattr(_lib.lib, name)
        assert re.search(r"GPSG_API\s+\w+\s+" + name + r"\(", header), name
    fields = re.search(r"typedef struct GpsgEncoderDownWeights \{(.*?)\}", header, re.S).group(1)
    assert re.findall(r"const float\* (\w+);", fields) == list(_lib.DECODER1_PARAMS)
    assert [n for n, _ in _lib.EncoderDownWeights._fields_] == list(_lib.DECODER1_PARAMS)


def _tiles(B, Ho, Wo):
    return B * ((Ho + 1) // 2) * ((Wo + 63) // 64)


def _align(n):
    return (n + 255) // 256 * 256


@pytest.mark.parametrize("cin,c", encoder.DOWN_DIMS)
@pytest.mark.parametrize("prec,el", [(0, 4), (1, 2)])
@pytest.mark.parametrize("B,H,W", [(2, 512, 512), (1, 9, 5), (3, 1, 1), (2, 256, 255)])
def test_workspace_bytes(cin, c, prec, el, B, H, W):
    Ho, Wo = (H + 1) // 2, (W + 1) // 2
    want = (5 * _align(B * Ho * Wo * c * el) + 5 * _align(B * c * 8) + 2 * _align(_tiles(B, Ho, Wo) * (c // 8) * 24)
            + _align((10 * cin * c + 27 * c * c) * el))
    assert _lib.lib.gpsg_encoder_down_workspace_bytes(B, cin, c, H, W, prec) == want


def test_refusals():
    f = _lib.lib.gpsg_encoder_down_workspace_bytes
    for args in ((2, 32, 96, 16, 16, 0), (2, 48, 48, 16, 16, 0), (2, 64, 96, 16, 16, 0), (2, 32, 48, 0, 16, 0),
                 (2, 32, 48, 16, 16, 7), (0, 32, 48, 16, 16, 0)):
        assert f(*args) == 0, args
    w = _lib.EncoderDownWeights()
    assert _lib.lib.gpsg_encoder_down_forward(0, None, 1, 32, 96, 8, 8, 0, None, w, None, None) != 0
    assert b"encoder_down" in _lib.lib.gpsg_last_error()
    assert _lib.lib.gpsg_encoder_down_forward(0, None, 0, 48, 96, 8, 8, 1, None, w, None, None) == 0   # B = 0


def test_run_down_refuses_cpu_tensors_and_foreign_dims():
    with pytest.raises(RuntimeError, match="encoder_down"):
        encoder.run_down(torch.zeros(1, 32, 8, 8), [torch.zeros(s) for s in encoder.down_param_shapes(32, 48)], "tf32")
    with pytest.raises(RuntimeError, match="encoder_down"):
        encoder.run_down(torch.zeros(1, 64, 8, 8), [torch.zeros(s) for s in encoder.down_param_shapes(64, 96)], "tf32")
    with pytest.raises(ValueError):
        encoder.run_down(torch.zeros(1, 32, 8, 8), [], "bf16")


def _extractor(**kw):
    harness.add_reference_to_path()
    from core.extractor import UnetExtractor
    torch.manual_seed(0)
    return UnetExtractor, UnetExtractor(**{"in_channel": 3, "encoder_dim": [32, 48, 96], **kw}).eval()


@needs_ref
def test_param_order_and_shapes():
    _, m = _extractor()
    for name, (cin, c) in zip(("res2", "res3"), encoder.DOWN_DIMS):
        st = getattr(m, name)
        ps = encoder.down_params_of(st)
        assert [tuple(p.shape) for p in ps] == list(encoder.down_param_shapes(cin, c))
        named = dict(st.named_parameters())
        names = [next(k for k, v in named.items() if v is p) for p in ps]
        want = [f"{b}.{n}" for b, ns in (("0", ("conv1", "norm1", "conv2", "norm2", "downsample.0", "norm3")),
                                          ("1", ("conv1", "norm1", "conv2", "norm2"))) for n in ns
                for n in (f"{n}.weight", f"{n}.bias")]
        # downsample.1 is norm3 itself: named_parameters lists the shared tensors under the first name it meets
        assert [n.replace("downsample.1", "norm3") for n in names] == want


@needs_ref
def test_supported_rejects_foreign_modules():
    _, m = _extractor()
    x = torch.zeros(1, 32, 8, 8)
    assert not encoder.down_supported(m.res2, x)                        # CPU input
    blk = type(m.res2[0])
    assert encoder._stage_supported(m.res2, blk, 32, 48) and encoder._stage_supported(m.res3, blk, 48, 96)
    assert not encoder._stage_supported(m.res2, blk, 48, 96)
    assert not encoder.down_supported(types.SimpleNamespace(), x)
    assert not encoder.down_supported(torch.nn.Sequential(), x)
    for kw in (dict(encoder_dim=[64, 96, 128]), dict(norm_fn="batch"), dict(norm_fn="instance")):
        _, f = _extractor(**kw)
        assert not (encoder._stage_supported(f.res2, blk, 32, 48) and encoder._stage_supported(f.res3, blk, 48, 96)), kw
    for mutate in (lambda s: setattr(s[0].norm1, "eps", 1e-6),
                   lambda s: setattr(s[1], "norm2", torch.nn.GroupNorm(12, 48)),
                   lambda s: setattr(s[0].downsample, "1", torch.nn.Identity()),
                   lambda s: setattr(s[0].conv1, "stride", (1, 1)),
                   lambda s: setattr(s[0].norm3, "affine", False)):
        _, f = _extractor()
        mutate(f.res2)
        assert not encoder._stage_supported(f.res2, blk, 32, 48)


@needs_ref
def test_deep_route_checks_res2_and_res3(monkeypatch):
    # the structure alone: parameters count as supported where they are fp32 on the given device (CUDA in real use)
    monkeypatch.setattr(encoder, "_tensors_supported",
                        lambda dev, *ts: all(t.device == dev and t.dtype == torch.float32 for t in ts))
    _, m = _extractor()
    assert encoder._down_stages_supported(m, torch.device("cpu"))
    assert not encoder._down_stages_supported(m, torch.device("cuda", 0))          # parameters on another device
    m.res3[0].norm3.eps = 1e-6
    assert not encoder._down_stages_supported(m, torch.device("cpu"))
    _, m = _extractor()
    m.res2 = torch.nn.Sequential()
    assert not encoder._down_stages_supported(m, torch.device("cpu"))


@needs_ref
@pytest.mark.parametrize("what", ["grad", "cpu", "allow_tf32_off"])
def test_deep_fallbacks_without_a_device(what, monkeypatch):
    cls, m = _extractor()
    fwd = encoder.make_extractor_forward(cls.forward, deep=True)
    monkeypatch.setattr(encoder, "run", lambda *a: pytest.fail("the kernels ran"))
    monkeypatch.setattr(encoder, "run_down", lambda *a: pytest.fail("the kernels ran"))
    if what == "allow_tf32_off":
        monkeypatch.setattr(torch.backends.cudnn, "allow_tf32", False)
    x = torch.rand(1, 3, 16, 12)
    with torch.enable_grad() if what == "grad" else torch.no_grad():
        got, want = fwd(m, x), cls.forward(m, x)
    for g, w in zip(got, want):
        assert torch.equal(g, w)


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


@pytest.mark.parametrize("enc,deep", [(None, "1"), ("1", None), ("1", "0"), ("1", "1"), ("0", "1")])
def test_deep_switch_needs_the_encoder_switch(monkeypatch, clean_patch, enc, deep):
    mod = _fake_module(monkeypatch)
    orig = mod.UnetExtractor.__dict__["forward"]
    for k, v in (("GPSG_ENCODER", enc), ("GPSG_ENCODER_DEEP", deep)):
        if v is None:
            monkeypatch.delenv(k, raising=False)
        else:
            monkeypatch.setenv(k, v)
    seen = []
    real = encoder.make_extractor_forward
    monkeypatch.setattr(encoder, "make_extractor_forward", lambda o, deep=False: seen.append(deep) or real(o, deep))
    patch.install()
    bound = enc == "1"
    assert patch.encoder() is bound and patch.encoder_deep() is (bound and deep == "1")
    assert (mod.UnetExtractor.__dict__["forward"] is not orig) is bound
    assert seen == ([deep == "1"] if bound else [])
    patch.uninstall()
    assert mod.UnetExtractor.__dict__["forward"] is orig
