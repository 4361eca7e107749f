"""CPU: the decoder3 / decoder2 entry points are exported and declared with the struct in the header's field order, bad
arguments are refused, the GPSG_DECODER_DEEP switch takes effect only together with GPSG_DECODER=1 and uninstall()
restores GSRegresser.forward, it composes with GPSG_GS_HEAD / GPSG_GS_HEAD_TRAIN, `deep_supported` rejects foreign
configurations, and the restated regressor forward equals the original bit for bit on the CPU in every combination of
the deep, decoder and tail switches."""
import os
import re
import sys
import types

import pytest
import torch

from gps_gaussian_b200 import _lib, decoder, gs_head, harness, patch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SYMBOLS = ("gpsg_decoder3_workspace_bytes", "gpsg_decoder3_forward", "gpsg_decoder2_workspace_bytes",
           "gpsg_decoder2_forward")


def test_symbols_exported_and_declared():
    header = open(os.path.join(ROOT, "include", "gpsg.h")).read()
    for name in SYMBOLS:
        assert name in _lib.EXPORTED and hasattr(_lib.lib, name)
        assert re.search(r"GPSG_API\s+\w+\s+" + name + r"\(", header), name
    fields = re.search(r"typedef struct GpsgDecoder23Weights \{(.*?)\}", header, re.S).group(1)
    assert re.findall(r"const float\* (\w+);", fields) == list(_lib.DECODER1_PARAMS)
    assert [n for n, _ in _lib.Decoder23Weights._fields_] == list(_lib.DECODER1_PARAMS)
    assert len(decoder.D3_PARAM_SHAPES) == len(decoder.D2_PARAM_SHAPES) == 20


def test_workspace_bytes_and_refusals():
    f3, f2 = _lib.lib.gpsg_decoder3_workspace_bytes, _lib.lib.gpsg_decoder2_workspace_bytes
    assert f3(2, 128, 128) >= 5 * 2 * 128 * 128 * 96 * 4
    assert f2(2, 128, 128) >= 5 * 2 * 256 * 256 * 64 * 4
    for f in (f3, f2):
        assert f(4, 64, 64) > f(2, 64, 64) > 0 and f(1, 1, 1) > 0
        assert f(0, 8, 8) == 0 and f(2, 0, 8) == 0 and f(2, 8, 0) == 0 and f(-1, 8, 8) == 0
    w = _lib.Decoder23Weights()
    p = 256
    fwd3, fwd2 = _lib.lib.gpsg_decoder3_forward, _lib.lib.gpsg_decoder2_forward
    assert fwd3(0, None, 1, 0, 8, None, None, w, None, None) != 0                    # H < 1
    assert fwd3(0, None, 1, 8, 0, None, None, w, None, None) != 0                    # W < 1
    assert fwd3(0, None, -1, 8, 8, None, None, w, None, None) != 0                   # negative B
    assert fwd3(0, None, 1, 8, 8, None, None, w, None, None) != 0                    # null pointers
    assert fwd3(0, None, 1, 8, 8, p, p, w, p, p) != 0                                # null weight pointers
    assert fwd3(0, None, 0, 8, 8, None, None, w, None, None) == 0                    # B = 0: nothing
    assert fwd2(0, None, 1, 0, 8, None, None, None, w, None, None) != 0
    assert fwd2(0, None, 1, 8, 0, None, None, None, w, None, None) != 0
    assert fwd2(0, None, -1, 8, 8, None, None, None, w, None, None) != 0
    assert fwd2(0, None, 1, 8, 8, None, None, None, w, None, None) != 0
    assert fwd2(0, None, 1, 8, 8, p, p, p, w, p, p) != 0
    assert fwd2(0, None, 0, 8, 8, None, None, None, w, None, None) == 0


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


SWITCHES = ("GPSG_DECODER", "GPSG_DECODER_DEEP", "GPSG_GS_HEAD", "GPSG_GS_HEAD_TRAIN")


@pytest.mark.parametrize("dec,deep", [(None, "1"), ("1", None), ("1", "0"), ("1", "true"), ("0", "1"), ("1", "1")])
def test_switch_binds_only_with_both_set(monkeypatch, clean_patch, dec, deep):
    mod = _fake_module(monkeypatch)
    orig = mod.GSRegresser.__dict__["forward"]
    for k in SWITCHES:
        monkeypatch.delenv(k, raising=False)
    for k, v in (("GPSG_DECODER", dec), ("GPSG_DECODER_DEEP", deep)):
        if v is not None:
            monkeypatch.setenv(k, v)
    seen = {}
    real = gs_head.make_regresser_forward
    monkeypatch.setattr(gs_head, "make_regresser_forward",
                        lambda orig, train=False, tail=True, decoder=False, **kw: seen.setdefault(
                            "deep", kw.get("deep", False)) is not None and real(orig, train, tail, decoder, **kw))
    patch.install()
    on = dec == "1" and deep == "1"
    assert patch.decoder_deep() is on
    assert seen.get("deep", False) is on
    assert (mod.GSRegresser.__dict__["forward"] is not orig) is (dec == "1")
    if on:
        with torch.no_grad():                       # a module without the regressor's layers: the reference answers
            assert mod.GSRegresser().forward(torch.zeros(1, 3, 4, 4), torch.zeros(1, 1, 4, 4),
                                             [torch.zeros(1, 32, 2, 2)] * 3) == "reference"
    patch.uninstall()
    assert mod.GSRegresser.__dict__["forward"] is orig


@pytest.mark.parametrize("env,want", [({"GPSG_GS_HEAD": "1"}, (True, False, True, True)),
                                      ({"GPSG_GS_HEAD_TRAIN": "1"}, (True, True, True, True)),
                                      ({}, (False, False, True, True))])
def test_switch_composes_with_the_tail(monkeypatch, clean_patch, env, want):
    mod = _fake_module(monkeypatch)
    for k in SWITCHES:
        monkeypatch.delenv(k, raising=False)
    for k, v in dict(env, GPSG_DECODER="1", GPSG_DECODER_DEEP="1").items():
        monkeypatch.setenv(k, v)
    seen = {}
    real = gs_head.make_regresser_forward
    monkeypatch.setattr(gs_head, "make_regresser_forward",
                        lambda orig, train=False, tail=True, decoder=False, deep=False: seen.setdefault(
                            "parts", (tail, train, decoder, deep)) and real(orig, train, tail, decoder, deep))
    patch.install()
    assert seen["parts"] == want
    assert mod.GSRegresser.forward.__module__ == gs_head.__name__


needs_ref = pytest.mark.skipif(harness.staged_reference() is None, reason="oracle/_ref not staged")


def _regresser(decoder_dims=(48, 64, 96), norm_fn="group", dims=(32, 48, 96)):
    harness.add_reference_to_path()
    from lib.gs_parm_network import GSRegresser
    cfg = types.SimpleNamespace(raft=types.SimpleNamespace(encoder_dims=list(dims)),
                                gsnet=types.SimpleNamespace(encoder_dims=list(dims), decoder_dims=list(decoder_dims),
                                                            parm_head_dim=32))
    torch.manual_seed(3)
    return GSRegresser, GSRegresser(cfg, norm_fn=norm_fn).eval()


def _inputs(B=1, H=32, W=48):
    g = torch.Generator().manual_seed(7)
    img, depth = torch.rand(B, 3, H, W, generator=g) * 2 - 1, torch.rand(B, 1, H, W, generator=g)
    feats = [torch.randn(B, c, H // s, W // s, generator=g) for c, s in ((32, 2), (48, 4), (96, 8))]
    return img, depth, feats


@needs_ref
@pytest.mark.parametrize("tail", [False, True])
@pytest.mark.parametrize("dec", [False, True])
@pytest.mark.parametrize("deep", [False, True])
def test_restated_forward_is_the_original_on_cpu(tail, dec, deep, monkeypatch):
    """Every stage left to the module: the support checks pass on the module and its features (so the restatement runs)
    and fail on the tensors (so no kernel does); the result must be the original's bit for bit."""
    cls, m = _regresser()
    for name in ("run", "run3", "run2"):
        monkeypatch.setattr(decoder, name, lambda *a: pytest.fail("the kernels ran"))
    monkeypatch.setattr(gs_head, "run", lambda *a: pytest.fail("the kernels ran"))
    monkeypatch.setattr(gs_head, "_Tail", None)
    monkeypatch.setattr(decoder, "supported", lambda r, s, f_i, f_d: s is None)
    monkeypatch.setattr(gs_head, "supported", lambda r, img, depth, up_src: up_src is None)
    monkeypatch.setattr(decoder, "deep_supported", lambda r, f3_i, f3_d, f2_i, f2_d: False)
    img, depth, feats = _inputs()
    # the deep route's device check on img_feat3 passes (so with `deep` the restatement runs), deep_supported fails
    monkeypatch.setattr(type(feats[2]), "is_cuda", property(lambda t: True))
    fwd = gs_head.make_regresser_forward(cls.forward, tail=tail, decoder=dec, deep=deep)
    calls = {"n": 0}
    orig_call = m.decoder3.forward
    monkeypatch.setattr(m.decoder3, "forward", lambda x: (calls.__setitem__("n", calls["n"] + 1), orig_call(x))[1])
    with torch.no_grad():
        got = fwd(m, img, depth, feats)
        n_restated = calls["n"]
        want = cls.forward(m, img, depth, feats)
    assert n_restated == (2 if tail else 1)
    for g, w in zip(got, want):
        assert torch.equal(g, w)


@needs_ref
def test_deep_supported_rejects_foreign_configurations(monkeypatch):
    _, m = _regresser()
    assert decoder._deep_module_supported(m)
    assert not decoder._deep_module_supported(types.SimpleNamespace())
    for kw in (dict(decoder_dims=(48, 64, 128)), dict(decoder_dims=(48, 96, 96)), dict(norm_fn="batch"),
               dict(norm_fn="instance"), dict(dims=(32, 64, 96))):
        assert not decoder._deep_module_supported(_regresser(**kw)[1]), kw
    _, m = _regresser()
    m.up = torch.nn.Upsample(scale_factor=2, mode="bilinear", align_corners=True)
    assert not decoder._deep_module_supported(m)
    _, m = _regresser()
    m.decoder3[0].norm3.eps = 1e-6
    assert not decoder._deep_module_supported(m)
    _, m = _regresser()
    m.decoder2[1].norm1.affine = False
    assert not decoder._deep_module_supported(m)
    _, m = _regresser()
    m.decoder2[1].conv2.padding = (0, 0)
    assert not decoder._deep_module_supported(m)
    _, m = _regresser()
    f3, f2 = torch.zeros(1, 96, 4, 4), torch.zeros(1, 48, 8, 8)
    assert not decoder.deep_supported(m, f3, f3, f2, f2)                               # CPU tensors
    # shapes alone, with the device check bypassed: feat2 must be exactly twice decoder3's size
    monkeypatch.setattr(decoder, "_tensors_supported", lambda dev, *ts: True)
    fake = lambda *shape: types.SimpleNamespace(shape=shape, is_cuda=True, device="cuda", dim=lambda: len(shape))
    monkeypatch.setattr(decoder.torch, "is_tensor", lambda t: True)
    f3 = fake(2, 96, 8, 12)
    assert decoder.deep_supported(m, f3, fake(2, 96, 8, 12), fake(2, 48, 16, 24), fake(2, 48, 16, 24))
    assert not decoder.deep_supported(m, f3, fake(2, 96, 8, 12), fake(2, 48, 17, 24), fake(2, 48, 17, 24))
    assert not decoder.deep_supported(m, f3, fake(2, 96, 8, 12), fake(2, 48, 16, 24), fake(2, 48, 16, 22))
    assert not decoder.deep_supported(m, f3, fake(2, 96, 8, 11), fake(2, 48, 16, 24), fake(2, 48, 16, 24))
    assert not decoder.deep_supported(m, fake(2, 64, 8, 12), fake(2, 96, 8, 12), fake(2, 48, 16, 24),
                                      fake(2, 48, 16, 24))


def test_run_refuses_cpu_tensors():
    with pytest.raises(RuntimeError, match="decoder3"):
        decoder.run3(torch.zeros(1, 96, 4, 4), torch.zeros(1, 96, 4, 4), [torch.zeros(s) for s in decoder.D3_PARAM_SHAPES])
    with pytest.raises(RuntimeError, match="decoder2"):
        decoder.run2(torch.zeros(1, 96, 4, 4), torch.zeros(1, 48, 8, 8), torch.zeros(1, 48, 8, 8),
                     [torch.zeros(s) for s in decoder.D2_PARAM_SHAPES])
