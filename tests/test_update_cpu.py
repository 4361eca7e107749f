"""CPU: the update-block entry points are exported and declared, the workspace and packed sizes, refusals, the parameter
order against the reference's own BasicMultiUpdateBlock, the `supported` truth table for every fallback condition, the
GPSG_UPDATE switch (alone without GPSG_PATCH it does nothing; it composes with the other switches), and every mutant of
the fp16-route emulation caught by a stage check: the rounding mutants at 2 x 9 x 7, the index mutants (tile halos, the
convf1 window, the context stride, stale carried state, the mask's N-block offset) on a second iteration at B = 2,
H = 5, W = 130, whose two full 64-column tiles, partial third and three 2-row tiles put a seam in every direction."""
import os
import re
import subprocess
import sys
import types

import pytest
import torch

import update_cases as uc
from gps_gaussian_b200 import _lib, harness, patch, update
from oracle import update_torch64 as ut

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SYMBOLS = ("gpsg_update_workspace_bytes", "gpsg_update_packed_bytes", "gpsg_update_pack", "gpsg_update_step")
needs_ref = pytest.mark.skipif(harness.staged_reference() is None, reason="oracle/_ref not staged")


def test_symbols_exported_and_declared():
    header = open(os.path.join(ROOT, "include", "gpsg.h")).read()
    for name in SYMBOLS:
        assert name in _lib.EXPORTED and hasattr(_lib.lib, name)
        assert re.search(r"GPSG_API\s+\w+\s+" + name + r"\(", header), name
    fields = re.search(r"typedef struct GpsgUpdateWeights \{(.*?)\}", header, re.S).group(1)
    assert re.findall(r"const float\* (\w+);", fields) == list(_lib.UPDATE_PARAMS)
    assert [n for n, _ in _lib.UpdateWeights._fields_] == list(_lib.UPDATE_PARAMS)
    assert len(_lib.UPDATE_PARAMS) == 24 == len(update.PARAM_SHAPES)
    assert update.PARAM_SHAPES == uc.PARAM_SHAPES


def _align(n):
    return (n + 255) // 256 * 256


@pytest.mark.parametrize("B,H,W", [(2, 128, 128), (4, 128, 128), (1, 1, 1), (3, 9, 70)])
def test_workspace_bytes(B, H, W):
    want = sum(_align(B * H * W * c * 2) for _, c in update.REGIONS)
    assert _lib.lib.gpsg_update_workspace_bytes(B, H, W) == want


def test_packed_bytes():
    gemm = (2 * 9 * 64 * 64 + 9 * 128 * 128 + 9 * 224 * 192 + 9 * 224 * 96 + 2 * 9 * 96 * 256 + 256 * 576
            + 9 * 256 * 8)
    floats = 64 * 36 + 64 * 98 + 64 + 64 + 128 + 128 + 192 + 96 + 512 + 576 + 8
    assert _lib.lib.gpsg_update_packed_bytes() == _align(2 * gemm) + _align(4 * floats)


def test_refusals():
    f = _lib.lib.gpsg_update_workspace_bytes
    for args in ((0, 8, 8), (1, 0, 8), (1, 8, 0), (-1, 8, 8)):
        assert f(*args) == 0, args
    step = _lib.lib.gpsg_update_step
    assert step(0, None, 0, 8, 8, 1, None, None, None, None, 0, None, None, None) != 0
    assert b"update" in _lib.lib.gpsg_last_error()
    assert step(0, None, 1, 8, 8, 2, 1, 1, None, 1, 0, None, 256, 256) != 0          # corr dtype
    assert b"corr_dtype" in _lib.lib.gpsg_last_error()
    assert step(0, None, 2, 8, 8, 1, 256, 256, None, 256, 100, None, 256, 256) != 0  # czrq batch stride
    assert b"czrq_batch_stride" in _lib.lib.gpsg_last_error()
    assert _lib.lib.gpsg_update_pack(0, None, _lib.UpdateWeights(), 256) != 0
    assert b"NULL weight" in _lib.lib.gpsg_last_error()


def test_pack_refuses_cpu_tensors():
    with pytest.raises(RuntimeError, match="update"):
        update.pack([torch.zeros(s) for s in update.PARAM_SHAPES])


# ---- the reference's modules -------------------------------------------------------------------------------------------

def _args(**kw):
    a = types.SimpleNamespace(mixed_precision=True, n_gru_layers=1, slow_fast_gru=None, hidden_dims=[96, 96, 96],
                              corr_levels=4, corr_radius=4, n_downsample=3, corr_implementation="reg_cuda")
    for k, v in kw.items():
        setattr(a, k, v)
    return a


def _block(**kw):
    harness.add_reference_to_path()
    from core.update import BasicMultiUpdateBlock
    torch.manual_seed(0)
    a = _args(**kw)
    return BasicMultiUpdateBlock(a, hidden_dims=a.hidden_dims)


@needs_ref
def test_param_order_matches_state_dict():
    blk = _block()
    names = [k for k in blk.state_dict() if not k.startswith(("gru16.", "gru32."))]
    ps = update.params_of(blk)
    assert len(names) == len(ps) == 24
    sd = blk.state_dict()
    for n, p, s in zip(names, ps, update.PARAM_SHAPES):
        assert sd[n].data_ptr() == p.data_ptr() and tuple(p.shape) == s, n


ARG_FALLBACKS = [dict(mixed_precision=False), dict(n_gru_layers=2), dict(n_gru_layers=3), dict(slow_fast_gru=True),
                 dict(hidden_dims=[128, 128, 128]), dict(corr_levels=3), dict(corr_radius=3), dict(n_downsample=2),
                 dict(corr_implementation="alt")]


@pytest.mark.parametrize("kw", ARG_FALLBACKS, ids=lambda kw: "-".join(f"{k}={v}" for k, v in kw.items()))
def test_args_truth_table(kw):
    assert update._args_supported(_args())
    assert update._args_supported(_args(corr_implementation="reg"))
    assert not update._args_supported(_args(**kw))


def _swap(blk, path, new):
    *head, last = path.split(".")
    obj = blk
    for h in head:
        obj = obj[int(h)] if h.isdigit() else getattr(obj, h)
    if last.isdigit():
        obj[int(last)] = new
    else:
        setattr(obj, last, new)


FOREIGN = {
    "convc1_kernel": ("encoder.convc1", lambda: torch.nn.Conv2d(36, 64, 3, padding=1)),
    "convf1_padding": ("encoder.convf1", lambda: torch.nn.Conv2d(2, 64, 7, padding=2)),
    "convz_no_bias": ("gru08.convz", lambda: torch.nn.Conv2d(224, 96, 3, padding=1, bias=False)),
    "convq_dilated": ("gru08.convq", lambda: torch.nn.Conv2d(224, 96, 3, padding=2, dilation=2)),
    "flow_head_relu": ("flow_head.relu", lambda: torch.nn.GELU()),
    "mask_act": ("mask.1", lambda: torch.nn.GELU()),
    "mask2_subclass": ("mask.2", lambda: type("MyConv", (torch.nn.Conv2d,), {})(256, 576, 1)),
    "conv_reflect": ("encoder.conv", lambda: torch.nn.Conv2d(128, 126, 3, padding=1, padding_mode="reflect")),
}


@needs_ref
@pytest.mark.parametrize("what", sorted(FOREIGN))
def test_block_truth_table(what):
    blk = _block()
    mod = sys.modules["core.update"]
    assert update._block_supported(blk, mod)
    path, make = FOREIGN[what]
    _swap(blk, path, make())
    assert not update._block_supported(blk, mod)


@needs_ref
def test_supported_refuses_cpu_tensors():
    harness.add_reference_to_path()
    from core.raft_stereo_human import FlowUpdateModule
    m = FlowUpdateModule(_args())
    B, H, W = 1, 4, 4
    czrq = torch.zeros(B, 288, H, W, dtype=torch.float16)
    assert not update.supported(m, torch.zeros(B, 32, H, W, dtype=torch.float16),
                                [torch.zeros(B, 96, H, W, dtype=torch.float16)], [list(czrq.split(96, 1))])


# ---- the switch --------------------------------------------------------------------------------------------------------

@pytest.fixture
def clean_patch():
    patch.uninstall()
    yield
    patch.uninstall()


def _fake_raft(monkeypatch):
    mod = types.ModuleType("core.raft_stereo_human")

    class FlowUpdateModule:
        def forward(self, *a, **k):
            return "reference"

        def upsample_flow(self, flow, mask):
            return "reference upsample"
    mod.FlowUpdateModule = FlowUpdateModule
    monkeypatch.setitem(sys.modules, "core.raft_stereo_human", mod)
    return mod


SWITCHES = ("GPSG_UPDATE", "GPSG_FLOW_HEAD", "GPSG_ENCODER", "GPSG_ENCODER_DEEP", "GPSG_DECODER", "GPSG_GS_HEAD")


@pytest.mark.parametrize("value", [None, "0", "true", "1"])
@pytest.mark.parametrize("flow_head", [False, True])
def test_switch_binds_only_when_set(monkeypatch, clean_patch, value, flow_head):
    mod = _fake_raft(monkeypatch)
    cls = mod.FlowUpdateModule
    fwd, up = cls.__dict__["forward"], cls.__dict__["upsample_flow"]
    for k in SWITCHES:
        monkeypatch.delenv(k, raising=False)
    if value is not None:
        monkeypatch.setenv("GPSG_UPDATE", value)
    if flow_head:
        monkeypatch.setenv("GPSG_FLOW_HEAD", "1")
    patch.install()
    bound = value == "1"
    assert patch.update() is bound and patch.flow_head() is flow_head
    assert ("core.raft_stereo_human" in patch._targets()) is (bound or flow_head)
    assert (cls.__dict__["forward"] is not fwd) is bound
    assert (cls.__dict__["upsample_flow"] is not up) is flow_head
    if bound:
        assert cls.forward.__module__ == update.__name__
        with torch.no_grad():                       # a module without the reference's update block: the reference answers
            assert cls().forward(None, None, [None], [None]) == "reference"
    patch.uninstall()
    assert cls.__dict__["forward"] is fwd and cls.__dict__["upsample_flow"] is up


def test_switch_composes_with_every_other(monkeypatch, clean_patch):
    mod = _fake_raft(monkeypatch)
    for k in SWITCHES:
        monkeypatch.setenv(k, "1")
    patch.install()
    assert patch.update() and patch.flow_head() and patch.encoder() and patch.encoder_deep() and patch.decoder()
    assert patch.gs_head()
    t = patch._targets()
    for name in ("core.raft_stereo_human", "core.extractor", "lib.gs_parm_network", "lib.loss"):
        assert name in t, name
    assert mod.FlowUpdateModule.forward.__module__ == update.__name__
    assert "flow_head" in mod.FlowUpdateModule.upsample_flow.__module__


def test_update_alone_without_patch_does_nothing():
    env = harness.script_env(patch=False, extra={"GPSG_UPDATE": "1"})
    code = "import sys; print('gps_gaussian_b200.patch' in sys.modules)"
    r = subprocess.run([sys.executable, "-c", code], env=env, text=True, capture_output=True, timeout=120)
    assert r.returncode == 0 and r.stdout.strip() == "False", r.stdout + r.stderr


# ---- the emulation's mutants ------------------------------------------------------------------------------------------

def _gru_exact(ps):
    """params whose GRU convolutions are zero: their sums are exact, so the GRU's elementwise rounding is fixed"""
    ps = list(ps)
    for i in (10, 12, 14):
        ps[i] = torch.zeros_like(ps[i])
    return ps


def _off_fp16(ps):
    """biases moved off the fp16 grid (fp32-exact): their fp16 rounding shows"""
    return [p + 3 * 2.0 ** -16 if p.dim() == 1 else p for p in ps]


@pytest.fixture(scope="module")
def mutant_case():
    B, H, W = 2, 9, 7
    inp = uc.inputs(B, H, W)
    sets = [_off_fp16(uc.params(0)), _gru_exact(_off_fp16(uc.params(0)))]
    return inp, sets


def _worst(ps, g):
    chk = ut.stage_checks(ps, g)
    return {k: ut.ratio(g[k], *chk[k]) for k in ut.KEYS}


def test_emulation_passes_its_checks(mutant_case):
    inp, sets = mutant_case
    for ps in sets:
        g = ut.emulate(ps, inp["corr"], inp["coords1"], inp["net"], inp["czrq"])
        assert max(_worst(ps, g).values()) == 0.0


@pytest.mark.parametrize("mutant", ut.MUTANTS)
def test_every_mutant_caught(mutant_case, mutant):
    inp, sets = mutant_case
    worst = 0.0
    for ps in sets:
        g = ut.emulate(ps, inp["corr"], inp["coords1"], inp["net"], inp["czrq"], mutant=mutant)
        worst = max(worst, max(_worst(ps, g).values()))
    assert worst > 1.0, mutant


# ---- the emulation's index mutants: two column tiles and a partial third, three row tiles ------------------------------

@pytest.fixture(scope="module")
def index_case():
    """The second iteration at B = 2, H = 5, W = 130, from the emulated first, with cz / cr / cq split from channels
    32 .. 319 of a [B,384,H,W] context."""
    B, H, W = 2, 5, 130
    inp = uc.inputs(B, H, W)
    outer = uc.inputs(B, H, W, seed=7)["czrq"]
    wide = torch.cat([outer[:, :32], inp["czrq"], outer[:, 32:96]], 1)
    czrq = wide[:, 32:320]
    ps = _off_fp16(uc.params(0))
    first = ut.emulate(ps, inp["corr"], inp["coords1"], inp["net"], czrq)
    return ps, inp["corr"], first, czrq


def _second(case, mutant=None):
    ps, corr, first, czrq = case
    return ut.emulate(ps, corr, first["coords1"], first["h"], czrq, mutant=mutant, prev=first)


def test_emulation_passes_its_checks_on_tiles(index_case):
    ps, _, first, _ = index_case
    assert max(_worst(ps, first).values()) == 0.0
    assert max(_worst(ps, _second(index_case)).values()) == 0.0


@pytest.mark.parametrize("mutant", ut.INDEX_MUTANTS)
def test_every_index_mutant_caught(index_case, mutant):
    ps = index_case[0]
    worst = _worst(ps, _second(index_case, mutant))
    print(f"{mutant}: {worst}")
    assert max(worst.values()) > 1.0, (mutant, worst)
