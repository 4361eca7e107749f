"""CPU: the decoder1 entry points are exported and declared with the struct in the header's field order, bad arguments
are refused, the GPSG_DECODER switch hooks lib.gs_parm_network only when set to 1 and uninstall() restores
GSRegresser.forward, `supported` rejects foreign configurations, and the one restatement of the regressor's forward
equals the original bit for bit on the CPU in every combination of the decoder and tail switches."""
import os
import re
import sys
import types

import pytest
import torch

from gps_gaussian_b200 import _lib, decoder, gs_head, harness, patch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SYMBOLS = ("gpsg_decoder1_workspace_bytes", "gpsg_decoder1_forward")


def test_symbols_exported_and_declared():
    header = open(os.path.join(ROOT, "include", "gpsg.h")).read()
    for name in SYMBOLS:
        assert name in _lib.EXPORTED and hasattr(_lib.lib, name)
        assert re.search(r"GPSG_API\s+\w+\s+" + name + r"\(", header), name
    fields = re.search(r"typedef struct GpsgDecoder1Weights \{(.*?)\}", header, re.S).group(1)
    assert re.findall(r"const float\* (\w+);", fields) == list(_lib.DECODER1_PARAMS)
    assert [n for n, _ in _lib.Decoder1Weights._fields_] == list(_lib.DECODER1_PARAMS)
    assert len(_lib.DECODER1_PARAMS) == 20 == len(decoder.PARAM_SHAPES)


def test_workspace_bytes_and_refusals():
    f = _lib.lib.gpsg_decoder1_workspace_bytes
    assert f(2, 256, 256) >= 5 * 2 * 512 * 512 * 48 * 4
    assert f(4, 256, 256) > f(2, 256, 256) > 0 and f(1, 1, 1) > 0
    assert f(0, 8, 8) == 0 and f(2, 0, 8) == 0 and f(2, 8, 0) == 0 and f(-1, 8, 8) == 0
    w = _lib.Decoder1Weights()
    fwd = _lib.lib.gpsg_decoder1_forward
    assert fwd(0, None, 1, 0, 8, None, None, None, w, None, None) != 0                    # Hs < 1
    assert fwd(0, None, 1, 8, 0, None, None, None, w, None, None) != 0                    # Ws < 1
    assert fwd(0, None, -1, 8, 8, None, None, None, w, None, None) != 0                   # negative B
    assert fwd(0, None, 1, 8, 8, None, None, None, w, None, None) != 0                    # null pointers
    p = 256
    assert fwd(0, None, 1, 8, 8, p, p, p, w, p, p) != 0                                  # null weight pointers
    assert fwd(0, None, 0, 8, 8, None, None, None, w, None, None) == 0                    # B = 0: nothing


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
    for k in ("GPSG_GS_HEAD", "GPSG_GS_HEAD_TRAIN"):
        monkeypatch.delenv(k, raising=False)
    if value is None:
        monkeypatch.delenv("GPSG_DECODER", raising=False)
    else:
        monkeypatch.setenv("GPSG_DECODER", value)
    patch.install()
    bound = value == "1"
    assert patch.decoder() is bound
    assert ("lib.gs_parm_network" in patch._targets()) is bound
    assert (mod.GSRegresser.__dict__["forward"] is not orig) is bound
    if bound:
        assert mod.GSRegresser.forward.__module__ == gs_head.__name__
        with torch.no_grad():                       # a module without the regressor's layers: the reference answers
            assert mod.GSRegresser().forward(torch.zeros(1, 3, 4, 4), torch.zeros(1, 1, 4, 4),
                                             [torch.zeros(1, 32, 2, 2)] * 3) == "reference"
    patch.uninstall()
    assert mod.GSRegresser.__dict__["forward"] is orig


@pytest.mark.parametrize("env,want", [({"GPSG_DECODER": "1"}, (False, False, True)),
                                      ({"GPSG_DECODER": "1", "GPSG_GS_HEAD": "1"}, (True, False, True)),
                                      ({"GPSG_DECODER": "1", "GPSG_GS_HEAD_TRAIN": "1"}, (True, True, True)),
                                      ({"GPSG_GS_HEAD": "1"}, (True, False, False))])
def test_switches_compose(monkeypatch, clean_patch, env, want):
    mod = _fake_module(monkeypatch)
    for k in ("GPSG_DECODER", "GPSG_GS_HEAD", "GPSG_GS_HEAD_TRAIN"):
        monkeypatch.delenv(k, raising=False)
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    seen = {}
    real = gs_head.make_regresser_forward
    monkeypatch.setattr(gs_head, "make_regresser_forward",
                        lambda orig, train=False, tail=True, decoder=False: seen.setdefault(
                            "parts", (tail, train, decoder)) and real(orig, train, tail, decoder))
    patch.install()
    assert seen["parts"] == want
    assert mod.GSRegresser.forward.__module__ == gs_head.__name__


needs_ref = pytest.mark.skipif(harness.staged_reference() is None, reason="oracle/_ref not staged")


def _regresser(decoder_dims=(48, 64, 96), norm_fn="group"):
    harness.add_reference_to_path()
    from lib.gs_parm_network import GSRegresser
    cfg = types.SimpleNamespace(raft=types.SimpleNamespace(encoder_dims=[32, 48, 96]),
                                gsnet=types.SimpleNamespace(encoder_dims=[32, 48, 96], decoder_dims=list(decoder_dims),
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
def test_restated_forward_is_the_original_on_cpu(tail, dec, monkeypatch):
    """decoder1 and the tail left to the module: the support checks pass on the module and its features (so the
    restatement runs) and fail on the decoder2 output (so no kernel does); the result must be the original's bit for
    bit."""
    cls, m = _regresser()
    monkeypatch.setattr(decoder, "run", lambda *a: pytest.fail("the kernels ran"))
    monkeypatch.setattr(gs_head, "run", lambda *a: pytest.fail("the kernels ran"))
    monkeypatch.setattr(gs_head, "_Tail", None)
    monkeypatch.setattr(decoder, "supported", lambda r, s, f_i, f_d: s is None)
    monkeypatch.setattr(gs_head, "supported", lambda r, img, depth, up_src: up_src is None)
    fwd = gs_head.make_regresser_forward(cls.forward, tail=tail, decoder=dec)
    img, depth, feats = _inputs()
    calls = {"n": 0}
    orig_call = m.decoder1.forward
    monkeypatch.setattr(m.decoder1, "forward", lambda x: (calls.__setitem__("n", calls["n"] + 1), orig_call(x))[1])
    with torch.no_grad():
        got = fwd(m, img, depth, feats)
        n_restated = calls["n"]
        want = cls.forward(m, img, depth, feats)
    # once by the original or the restatement; twice when the tail was asked for and fell back to the original
    assert n_restated == (2 if tail else 1)
    for g, w in zip(got, want):
        assert torch.equal(g, w)


@needs_ref
@pytest.mark.parametrize("what", ["grad", "allow_tf32_off"])
def test_fallbacks_without_a_device(what, monkeypatch):
    cls, m = _regresser()
    fwd = gs_head.make_regresser_forward(cls.forward, tail=False, decoder=True)
    monkeypatch.setattr(decoder, "run", lambda *a: pytest.fail("the kernels ran"))
    if what == "allow_tf32_off":
        monkeypatch.setattr(torch.backends.cudnn, "allow_tf32", False)
    img, depth, feats = _inputs()
    ctx = torch.enable_grad() if what == "grad" else torch.no_grad()
    with ctx:
        got, want = fwd(m, img, depth, feats), cls.forward(m, img, depth, feats)
    for g, w in zip(got, want):
        assert torch.equal(g, w)


@needs_ref
def test_supported_rejects_foreign_configurations(monkeypatch):
    _, m = _regresser()
    assert decoder._module_supported(m)
    assert not decoder.supported(m, None, torch.zeros(1, 32, 8, 8), None)            # CPU tensors
    assert not decoder._module_supported(types.SimpleNamespace())
    for kw in (dict(decoder_dims=(64, 64, 96)), dict(decoder_dims=(48, 96, 128)), dict(norm_fn="batch"),
               dict(norm_fn="instance")):
        assert not decoder._module_supported(_regresser(**kw)[1]), kw
    _, m = _regresser()
    m.up = torch.nn.Upsample(scale_factor=2, mode="bilinear", align_corners=True)
    assert not decoder._module_supported(m)
    _, m = _regresser()
    m.decoder1[0].norm3.eps = 1e-6
    assert not decoder._module_supported(m)
    _, m = _regresser()
    m.decoder1[1].conv2.padding = (0, 0)
    assert not decoder._module_supported(m)
    # a feature map that is not twice the size of s (checked on the shapes alone, with the device check bypassed)
    _, m = _regresser()
    monkeypatch.setattr(decoder, "_tensors_supported", lambda dev, *ts: True)
    fake = lambda *shape: types.SimpleNamespace(shape=shape, is_cuda=True, device="cuda", dim=lambda: len(shape))
    monkeypatch.setattr(decoder.torch, "is_tensor", lambda t: True)
    fi = fake(2, 32, 16, 24)
    assert decoder.supported(m, fake(2, 64, 8, 12), fi, fake(2, 32, 16, 24))
    assert not decoder.supported(m, fake(2, 64, 8, 11), fi, fake(2, 32, 16, 24))
    assert not decoder.supported(m, fake(2, 64, 8, 12), fi, fake(2, 32, 16, 22))
    assert not decoder.supported(m, fake(2, 48, 8, 12), fi, fake(2, 32, 16, 24))


def test_run_refuses_cpu_tensors():
    with pytest.raises(RuntimeError, match="decoder1"):
        decoder.run(torch.zeros(1, 64, 4, 4), torch.zeros(1, 32, 8, 8), torch.zeros(1, 32, 8, 8),
                    [torch.zeros(s) for s in decoder.PARAM_SHAPES])
