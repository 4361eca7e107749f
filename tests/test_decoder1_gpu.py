"""GPU: the regressor's decoder1 (csrc/decoder1.cu through gps_gaussian_b200.decoder) against the fp64 restatement
(oracle/decoder1_torch64.py), per element and with NaN exactly where fp64 has it.  Two checks per case: `out` within the
end-to-end bounds of fp64 from the inputs, and every stage (the five stored convolution outputs and out) within its own
derived bound of fp64 from the kernels' stored input to that stage.  Sizes: B in {1, 2, 4} at 1024^2 input (s 256^2,
features 512^2), the golden cases of the reference's modules, and small odd shapes whose tiles do not divide them.
Every output and workspace buffer is poisoned with NaN before each launch.  The worst utilisation per case goes to
$GPSG_PARITY_LOG.

Through `gs_head.make_regresser_forward(..., decoder=True)` on the reference's own GSRegresser: no-grad TF32 calls take
the kernels (with the tail on the module's layers or on its own kernels), everything else is bit for bit the original
forward.  With the staged reference: the RtStereoHumanModel eval forward at 1024^2 with GPSG_DECODER on and off, and
test_view_interp.py run unmodified with GPSG_PATCH=1 GPSG_ENCODER=1 GPSG_GS_HEAD=1 GPSG_DECODER=1."""
import os
import subprocess
import sys
import types

import pytest
import torch

import decoder1_cases as dc
from helpers import record
from gps_gaussian_b200 import decoder, gs_head, harness, patch
from oracle import decoder1_torch64 as dt

pytestmark = pytest.mark.gpu
needs_ref = pytest.mark.skipif(harness.staged_reference() is None, reason="oracle/_ref not staged")
RAWS = ("y1", "yd", "y2", "y3", "y4")


@pytest.fixture(autouse=True)
def poisoned_outputs(monkeypatch):
    """torch.empty inside decoder returns NaN-filled buffers (the uint8 workspace as 0xFF bytes, a NaN pattern for
    fp32), so an output element the kernels skip shows."""
    def nan(fn):
        def make(*a, **k):
            t = fn(*a, **k)
            if t.is_floating_point():
                t.fill_(float("nan"))
            elif t.dtype == torch.uint8:
                t.fill_(0xFF)
            return t
        return make
    fake = types.SimpleNamespace(**{n: getattr(torch, n) for n in dir(torch) if not n.startswith("__")})
    fake.empty, fake.empty_like = nan(torch.empty), nan(torch.empty_like)
    monkeypatch.setattr(decoder, "torch", fake)


def _check(tag, s, fi, fd, ps, want=None, end_to_end=True):
    """Kernels on the device; per sample: out against fp64 within the chained bounds (end_to_end) and each stage within
    its own bound.  want: golden out (fp64) in place of forward64's."""
    dev = [p.cuda() for p in ps]
    out, raws = decoder.forward_with_workspace(s.cuda(), fi.cuda(), fd.cuda(), dev)
    worst = {}
    for n in range(s.shape[0]):
        args = [t[n:n + 1].cuda() for t in (s, fi, fd)]
        if end_to_end:
            ref = dt.forward64(*args, dev)["out"] if want is None else want[n:n + 1].cuda()
            worst["out"] = max(worst.get("out", 0.0), dt.ratio(out[n:n + 1], ref, dt.bounds(*args, dev)["out"]))
        stages = dt.stage_checks(*args, dev, [r[n:n + 1] for r in raws])
        got = dict(zip(RAWS, (r[n:n + 1] for r in raws)), out=out[n:n + 1])
        for k, (w, b) in stages.items():
            worst["stage_" + k] = max(worst.get("stage_" + k, 0.0), dt.ratio(got[k], w, b))
        del stages
        torch.cuda.empty_cache()
    record(f"decoder1:{tag}", **worst)
    print(f"{tag}: utilisation {worst}")
    assert max(worst.values()) <= 1.0, worst
    return out, raws


@pytest.mark.parametrize("B", [1, 2, 4])
def test_script_size(B):
    case = dc.Case(f"b{B}_1024", B, 256, 256, 10 + B)
    # the end-to-end bound chains worst cases through five GroupNorms; at this size the stage checks carry it
    _check(case.id, *dc.inputs(case), end_to_end=False)


SMALL = dc.SWEEP + [dc.Case("odd_37x65", 2, 37, 65, 20), dc.Case("column_35x1", 1, 35, 1, 22),
                    dc.Case("row_1x150", 2, 1, 150, 23), dc.Case("b3_9x33", 3, 9, 33, 24)]


@pytest.mark.parametrize("case", SMALL, ids=lambda c: c.id)
def test_small_shapes(case):
    out, _ = _check(case.id, *dc.inputs(case))
    if case.special in ("nan", "inf"):
        assert torch.isnan(out[0]).all() and not torch.isnan(out[1:]).any()


@pytest.mark.parametrize("name", dc.GOLDEN_CASES)
def test_golden(name):
    s, fi, fd, ps, want = dc.golden(name)
    _check("golden_" + name, s, fi, fd, ps, want)


def test_non_finite_pixel_poisons_only_its_sample():
    s, fi, fd, ps = dc.inputs(dc.Case("b3", 3, 32, 48, 30))
    dev = [p.cuda() for p in ps]
    clean = decoder.run(s.cuda(), fi.cuda(), fd.cuda(), dev)
    for bad in (float("nan"), float("inf")):
        for which in ("s", "fi", "fd"):
            t = {"s": s.clone(), "fi": fi.clone(), "fd": fd.clone()}
            t[which][1, 2, 20, 7] = bad
            got = decoder.run(t["s"].cuda(), t["fi"].cuda(), t["fd"].cuda(), dev)
            assert torch.isnan(got[1]).all(), which
            assert torch.equal(got[0], clean[0]) and torch.equal(got[2], clean[2]), which


def test_bit_reproducible():
    s, fi, fd, ps = dc.inputs(dc.Case("b2", 2, 128, 128, 31))
    dev = [p.cuda() for p in ps]
    a, b = (decoder.run(s.cuda(), fi.cuda(), fd.cuda(), dev) for _ in range(2))
    assert torch.equal(a.view(torch.int32), b.view(torch.int32))


# ---- the rebound GSRegresser.forward ------------------------------------------------------------------------------

def _regresser(decoder_dims=(48, 64, 96), norm_fn="group"):
    harness.add_reference_to_path()
    from lib.gs_parm_network import GSRegresser
    cfg = types.SimpleNamespace(raft=types.SimpleNamespace(encoder_dims=[32, 48, 96]),
                                gsnet=types.SimpleNamespace(encoder_dims=[32, 48, 96], decoder_dims=list(decoder_dims),
                                                            parm_head_dim=32))
    torch.manual_seed(3)
    m = GSRegresser(cfg, norm_fn=norm_fn).eval()
    g = torch.Generator().manual_seed(4)
    with torch.no_grad():
        for mod in m.modules():
            if isinstance(mod, torch.nn.GroupNorm) and mod.affine:
                mod.weight.copy_(0.5 + torch.rand(mod.weight.shape, generator=g))
                mod.bias.copy_(torch.rand(mod.bias.shape, generator=g) - 0.5)
    return GSRegresser, m


def _reg_inputs(B, H, W, device="cuda", dtype=torch.float32):
    g = torch.Generator().manual_seed(B * H + W)
    img = torch.rand(B, 3, H, W, generator=g) * 2 - 1
    depth = torch.rand(B, 1, H, W, generator=g)
    feats = [torch.randn(B, c, H // s, W // s, generator=g) for c, s in ((32, 2), (48, 4), (96, 8))]
    return [t.to(device, dtype) for t in (img, depth)] + [[f.to(device, dtype) for f in feats]]


def _captured(m, cls, img, depth, feats):
    """The module's own decoder2 output and depth_feat1 in the original forward."""
    seen = {}
    hooks = [m.decoder2.register_forward_hook(lambda mod, i, o: seen.__setitem__("s", o.clone())),
             m.depth_encoder.register_forward_hook(lambda mod, i, o: seen.__setitem__("fd", o[0].clone()))]
    try:
        cls.forward(m, img, depth, feats)
    finally:
        for h in hooks:
            h.remove()
    return seen["s"], seen["fd"]


@needs_ref
@pytest.mark.parametrize("tail", [False, True])
def test_rebound_forward_runs_the_kernels(tail, monkeypatch):
    cls, m = _regresser()
    m.cuda()
    fwd = gs_head.make_regresser_forward(cls.forward, tail=tail, decoder=True)
    seen = {}
    run_dec, run_tail = decoder.run, gs_head.run
    monkeypatch.setattr(decoder, "run", lambda *a: seen.setdefault("dec", run_dec(*a)))
    monkeypatch.setattr(gs_head, "run", lambda x, *a: (seen.setdefault("tail_in", x), run_tail(x, *a))[1])
    img, depth, feats = _reg_inputs(2, 64, 96)
    decoder.reset_counts()
    with torch.no_grad():
        got = fwd(m, img, depth, feats)
        s, fd = _captured(m, cls, img, depth, feats)
        if not tail:                           # the reference's tail on the module's layers, from the kernels' output
            out = m.out_relu(m.out_conv(torch.cat([m.up(seen["dec"]), img, depth], 1)))
            want = (torch.nn.functional.normalize(m.rot_head(out), dim=1),
                    torch.clamp_max(m.scale_head(out), 0.01), m.opacity_head(out))
            for g, w in zip(got, want):
                assert torch.equal(g, w)
    assert decoder.counts()["forward"] == 1
    assert ("tail_in" in seen) is tail and (not tail or seen["tail_in"] is seen["dec"])
    ps = [p.detach() for p in decoder.params_of(m)]
    args = (s, feats[0], fd)
    ratio = dt.ratio(seen["dec"], dt.forward64(*args, ps)["out"], dt.bounds(*args, ps)["out"])
    record(f"decoder1:rebound:tail={tail}", out=ratio)
    assert ratio <= 1.0


@needs_ref
@pytest.mark.parametrize("what", ["grad", "autocast", "allow_tf32_off", "cpu", "fp16_input", "dims", "batch",
                                  "align_corners"])
def test_rebound_forward_falls_back_bit_for_bit(what, monkeypatch):
    kw = dict(decoder_dims=(64, 64, 96)) if what == "dims" else (dict(norm_fn="batch") if what == "batch" else {})
    cls, m = _regresser(**kw)
    if what == "align_corners":
        m.up = torch.nn.Upsample(scale_factor=2, mode="bilinear", align_corners=True)
    device = "cpu" if what == "cpu" else "cuda"
    dtype = torch.float16 if what == "fp16_input" else torch.float32
    m.to(device, dtype)
    fwd = gs_head.make_regresser_forward(cls.forward, tail=False, decoder=True)
    monkeypatch.setattr(decoder, "run", lambda *a: pytest.fail("the kernels ran"))
    monkeypatch.setattr(decoder, "forward_with_workspace", lambda *a, **k: pytest.fail("the kernels ran"))
    if what == "allow_tf32_off":
        monkeypatch.setattr(torch.backends.cudnn, "allow_tf32", False)
    img, depth, feats = _reg_inputs(1, 32, 48, device, dtype)
    grad = torch.enable_grad() if what == "grad" else torch.no_grad()
    with grad, torch.autocast("cuda", dtype=torch.float16, enabled=what == "autocast"):
        got = fwd(m, img, depth, feats)
        want = cls.forward(m, img, depth, feats)
    for g, w in zip(got, want):
        assert torch.equal(g, w)


# ---- the reference's model and scripts with the switch --------------------------------------------------------------

@pytest.fixture(scope="module")
def dataset_1024(tmp_path_factory):
    from gps_gaussian_b200 import synth_dataset
    root = str(tmp_path_factory.mktemp("decoderdata"))
    synth_dataset.write_dataset(root, n_train=1, n_val=1, res=1024, hr=True)
    return root


def _install(on, monkeypatch):
    patch.uninstall()
    if on:
        monkeypatch.setenv("GPSG_DECODER", "1")
    else:
        monkeypatch.delenv("GPSG_DECODER", raising=False)
    for k in ("GPSG_GS_HEAD", "GPSG_GS_HEAD_TRAIN", "GPSG_ENCODER"):
        monkeypatch.delenv(k, raising=False)
    harness.add_reference_to_path()
    patch.install()
    import lib.gs_parm_network
    assert (lib.gs_parm_network.GSRegresser.forward.__module__ == gs_head.__name__) is on


@needs_ref
def test_eval_forward_switch_on_off(dataset_1024, monkeypatch):
    """The eval forward at 1024^2, switch on against off.  Tolerance: the kernels may move the regressor's maps by at most
    twice what the reference's own TF32 decoder1 moves them, measured as the switched-off forward against one whose
    decoder1 runs with cuDNN's TF32 off (full fp32).  The kernels differ from cuDNN only by where TF32 rounding and fp32
    re-association fall, so they must stay within that scale."""
    outs = {}
    decoder.reset_counts()
    try:
        for run in ("off", "fp32", "on"):
            _install(run == "on", monkeypatch)
            monkeypatch.setattr(torch.backends.cudnn, "allow_tf32", True)
            cfg = harness.load_cfg(dataset_1024, src_res=1024, batch_size=1)
            st = harness.C3State(cfg)
            st.model.eval()
            hooks = []
            if run == "fp32":
                dec1 = st.model.gs_parm_regresser.decoder1
                hooks = [dec1.register_forward_pre_hook(lambda *a: setattr(torch.backends.cudnn, "allow_tf32", False)),
                         dec1.register_forward_hook(lambda *a: setattr(torch.backends.cudnn, "allow_tf32", True))]
            data = st.batch(0)
            with torch.no_grad():
                out, _, _ = st.model({k: dict(v) if isinstance(v, dict) else v for k, v in data.items()}, is_train=False)
            for h in hooks:
                h.remove()
            outs[run] = {f"{v}_{k}": out[v][k].float().clone() for v in ("lmain", "rmain")
                         for k in ("rot_maps", "scale_maps", "opacity_maps")}
            del st, out, data
            torch.cuda.empty_cache()
    finally:
        patch.uninstall()
    assert decoder.counts()["forward"] >= 1
    ref, yard, on = outs["off"], outs["fp32"], outs["on"]
    assert ref.keys() == on.keys() and ref
    stats = {}
    for k in ref:
        fin = torch.isfinite(ref[k])
        assert torch.equal(torch.isfinite(on[k]), fin), k
        stats[k] = (float((on[k] - ref[k])[fin].abs().mean()), float((yard[k] - ref[k])[fin].abs().mean()))
    record("decoder1:eval_switch", **{k: v[0] for k, v in stats.items()})
    print({k: f"switch {a:.3e} / reference fp32 decoder1 {b:.3e}" for k, (a, b) in stats.items()})
    for k, (a, b) in stats.items():
        assert a <= 2 * b, (k, a, b)


@needs_ref
def test_view_interp_runs_unmodified_with_every_regressor_switch(tmp_path):
    from gps_gaussian_b200 import synth_dataset
    dataset = str(tmp_path / "data")
    synth_dataset.write_dataset(dataset, n_train=1, n_val=2, res=256, hr=True)
    work = harness.make_workdir(str(tmp_path / "work"), dataset, src_res=256, num_steps=3, batch_size=1)
    harness.add_reference_to_path()
    cfg = harness.load_cfg(dataset, src_res=256, batch_size=1)
    from lib.network import RtStereoHumanModel
    torch.manual_seed(5)
    ckpt = str(tmp_path / "init.pth")
    torch.save({"network": RtStereoHumanModel(cfg, with_gs_render=True).state_dict()}, ckpt)
    extra = {"GPSG_ENCODER": "1", "GPSG_GS_HEAD": "1", "GPSG_DECODER": "1"}
    r = subprocess.run([sys.executable, "-c", _COUNTING_RUNNER + harness.SCRIPT_RUNNER, "test_view_interp.py",
                        "--test_data_root", os.path.join(dataset, "val"), "--ckpt_path", ckpt, "--novel_view_nums", "2"],
                       cwd=work, env=harness.script_env(patch=True, extra=extra), text=True, capture_output=True,
                       timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-6000:]
    line = [ln for ln in r.stdout.splitlines() if ln.startswith("decoder1 runs:")][-1]
    assert int(line.split(":")[1]) > 0, line


_COUNTING_RUNNER = ("import atexit\n"
                    "from gps_gaussian_b200 import decoder\n"
                    "atexit.register(lambda: print('decoder1 runs:', decoder.counts()['forward'], flush=True))\n")
