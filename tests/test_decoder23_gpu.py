"""GPU: the regressor's decoder3 and decoder2 (csrc/decoder23.cu through gps_gaussian_b200.decoder) against the fp64
restatement (oracle/decoder23_torch64.py), per element and with NaN exactly where fp64 has it.  Two checks per stage and
case: `out` within the end-to-end bounds of fp64 from the inputs, and every step (the five stored convolution outputs
and out) within its own derived bound of fp64 from the kernels' stored input to that step.  Sizes: B in {1, 2, 4} at the
stage sizes of a 1024^2 input (decoder3 at 128^2, decoder2 at 256^2), the golden cases of the reference's modules, and
small odd shapes whose tiles do not divide them.  Every output and workspace buffer is poisoned with NaN before each
launch.  The worst utilisation per case goes to $GPSG_PARITY_LOG.

Through `gs_head.make_regresser_forward(..., decoder=True, deep=True)` on the reference's own GSRegresser: no-grad TF32
calls run decoder3 -> decoder2 -> decoder1 -> tail on the kernels, each output handed to the next stage as it is, and
everything else is bit for bit the original forward.  With the staged reference: the RtStereoHumanModel eval forward at
1024^2 with GPSG_DECODER_DEEP on and off, and test_view_interp.py run unmodified with every encoder and regressor switch
on."""
import os
import subprocess
import sys
import types

import pytest
import torch

import decoder23_cases as dc
from helpers import record
from gps_gaussian_b200 import decoder, gs_head, harness, patch
from oracle import decoder23_torch64 as dt

pytestmark = pytest.mark.gpu
needs_ref = pytest.mark.skipif(harness.staged_reference() is None, reason="oracle/_ref not staged")


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


def _launch(stage, srcs, ps):
    if stage == "d3":
        return decoder.forward3_with_workspace(*srcs, ps)
    return decoder.forward2_with_workspace(*srcs, ps)


def _check(tag, stage, srcs, ps, want=None, end_to_end=True):
    """One stage on the device; per sample: out against fp64 within the chained bounds (end_to_end) and each step
    within its own bound.  want: golden out (fp64) in place of forward64's."""
    dev = [p.cuda() for p in ps]
    srcs = [t.cuda() for t in srcs]
    out, raws = _launch(stage, srcs, dev)
    worst = {}
    for n in range(srcs[0].shape[0]):
        args = [t[n:n + 1] for t in srcs]
        if end_to_end:
            ref = dt.forward64(stage, args, dev)["out"] if want is None else want[n:n + 1].cuda()
            worst["out"] = max(worst.get("out", 0.0), dt.ratio(out[n:n + 1], ref, dt.bounds(stage, args, dev)["out"]))
        stages = dt.stage_checks(stage, args, dev, [r[n:n + 1] for r in raws])
        got = dict(zip(dt.RAW_KEYS, (r[n:n + 1] for r in raws)), out=out[n:n + 1])
        for k, (w, b) in stages.items():
            worst["stage_" + k] = max(worst.get("stage_" + k, 0.0), dt.ratio(got[k], w, b))
        del stages
        torch.cuda.empty_cache()
    record(f"decoder23:{stage}:{tag}", **worst)
    print(f"{stage} {tag}: utilisation {worst}")
    assert max(worst.values()) <= 1.0, worst
    return out, raws


def _both(tag, d, want3=None, want2=None, end_to_end=True):
    """decoder3 on (f3i, f3d), then decoder2 on the kernels' decoder3 output and (f2i, f2d)."""
    out3, _ = _check(tag, "d3", *dc.stage_args(d, "d3"), want=want3, end_to_end=end_to_end)
    out2, _ = _check(tag, "d2", *dc.stage_args(d, "d2", s=out3.cpu()), want=want2, end_to_end=end_to_end)
    return out3, out2


@pytest.mark.parametrize("B", [1, 2, 4])
def test_script_size(B):
    # the end-to-end bound chains worst cases through five GroupNorms; at this size the stage checks carry it
    _both(f"b{B}_1024", dc.inputs(dc.Case(f"b{B}_1024", B, 128, 128, 10 + B)), end_to_end=False)


SMALL = dc.SWEEP + [dc.Case("one_1x1", 1, 1, 1, 19), dc.Case("odd_37x65", 2, 37, 65, 20),
                    dc.Case("column_35x1", 1, 35, 1, 22), dc.Case("row_1x150", 2, 1, 150, 23),
                    dc.Case("b3_9x33", 3, 9, 33, 24)]


@pytest.mark.parametrize("case", SMALL, ids=lambda c: c.id)
def test_small_shapes(case):
    out3, out2 = _both(case.id, dc.inputs(case))
    if case.special in ("nan", "inf"):
        for out in (out3, out2):
            assert torch.isnan(out[0]).all() and not torch.isnan(out[1:]).any()


@pytest.mark.parametrize("name", dc.GOLDEN_CASES)
def test_golden(name):
    d = dc.golden(name)
    _check("golden_" + name, "d3", *dc.stage_args(d, "d3"), want=d["out3"])
    # decoder2 from the golden fp64 decoder3 output rounded to fp32, against the golden decoder2 of that fp64 input:
    # only the end-to-end bound would see the rounding, so it is checked stage by stage
    _check("golden_" + name, "d2", *dc.stage_args(d, "d2", s=d["out3"].float()), end_to_end=False)


def test_non_finite_pixel_poisons_only_its_sample():
    d = dc.inputs(dc.Case("b3", 3, 16, 24, 30))
    p3, p2 = ([p.cuda() for p in d[k]] for k in ("p3", "p2"))
    t = {k: d[k].cuda() for k in ("f3i", "f3d", "f2i", "f2d", "s")}
    clean3, clean2 = decoder.run3(t["f3i"], t["f3d"], p3), decoder.run2(t["s"], t["f2i"], t["f2d"], p2)
    for bad in (float("nan"), float("inf")):
        for which in ("f3i", "f3d", "s", "f2i", "f2d"):
            u = {k: v.clone() for k, v in t.items()}
            u[which][1, 2, 5, 7] = bad
            got = decoder.run3(u["f3i"], u["f3d"], p3) if which.startswith("f3") else \
                decoder.run2(u["s"], u["f2i"], u["f2d"], p2)
            clean = clean3 if which.startswith("f3") else clean2
            assert torch.isnan(got[1]).all(), which
            assert torch.equal(got[0], clean[0]) and torch.equal(got[2], clean[2]), which


def test_bit_reproducible():
    d = dc.inputs(dc.Case("b2", 2, 64, 64, 31))
    p3, p2 = ([p.cuda() for p in d[k]] for k in ("p3", "p2"))
    a3, b3 = (decoder.run3(d["f3i"].cuda(), d["f3d"].cuda(), p3) for _ in range(2))
    assert torch.equal(a3.view(torch.int32), b3.view(torch.int32))
    a2, b2 = (decoder.run2(a3, d["f2i"].cuda(), d["f2d"].cuda(), p2) for _ in range(2))
    assert torch.equal(a2.view(torch.int32), b2.view(torch.int32))


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


@needs_ref
def test_rebound_forward_runs_every_stage_on_the_kernels(monkeypatch):
    cls, m = _regresser()
    m.cuda()
    fwd = gs_head.make_regresser_forward(cls.forward, tail=True, decoder=True, deep=True)
    seen = {}
    run3, run2, run1, run_tail = decoder.run3, decoder.run2, decoder.run, gs_head.run
    monkeypatch.setattr(decoder, "run3", lambda *a: seen.setdefault("d3", run3(*a)))
    monkeypatch.setattr(decoder, "run2", lambda s, *a: (seen.setdefault("d2_in", s), seen.setdefault("d2", run2(s, *a)))[1])
    monkeypatch.setattr(decoder, "run", lambda s, *a: (seen.setdefault("d1_in", s), seen.setdefault("d1", run1(s, *a)))[1])
    monkeypatch.setattr(gs_head, "run", lambda x, *a: (seen.setdefault("tail_in", x), run_tail(x, *a))[1])
    img, depth, feats = _reg_inputs(2, 64, 96)
    decoder.reset_counts()
    decoder.reset_deep_counts()
    with torch.no_grad():
        fwd(m, img, depth, feats)
        fd = m.depth_encoder(depth)
    assert decoder.deep_counts() == {"decoder3": 1, "decoder2": 1} and decoder.counts()["forward"] == 1
    assert seen["d2_in"] is seen["d3"] and seen["d1_in"] is seen["d2"] and seen["tail_in"] is seen["d1"]
    p3, p2 = ([p.detach() for p in ps] for ps in decoder.deep_params_of(m))
    for stage, srcs, ps, got in (("d3", (feats[2], fd[2]), p3, seen["d3"]),
                                 ("d2", (seen["d3"], feats[1], fd[1]), p2, seen["d2"])):
        ratio = dt.ratio(got, dt.forward64(stage, srcs, ps)["out"], dt.bounds(stage, srcs, ps)["out"])
        record(f"decoder23:rebound:{stage}", out=ratio)
        assert ratio <= 1.0


@needs_ref
@pytest.mark.parametrize("what", ["grad", "autocast", "allow_tf32_off", "cpu", "fp16_input", "dims", "batch",
                                  "align_corners", "deep_off"])
def test_rebound_forward_falls_back_bit_for_bit(what, monkeypatch):
    kw = dict(decoder_dims=(48, 64, 128)) if what == "dims" else (dict(norm_fn="batch") if what == "batch" else {})
    cls, m = _regresser(**kw)
    if what == "align_corners":
        m.up = torch.nn.Upsample(scale_factor=2, mode="bilinear", align_corners=True)
    device = "cpu" if what == "cpu" else "cuda"
    dtype = torch.float16 if what == "fp16_input" else torch.float32
    m.to(device, dtype)
    fwd = gs_head.make_regresser_forward(cls.forward, tail=False, decoder=False, deep=what != "deep_off")
    for name in ("run3", "run2", "forward3_with_workspace", "forward2_with_workspace"):
        monkeypatch.setattr(decoder, name, lambda *a, **k: pytest.fail("the kernels ran"))
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
    root = str(tmp_path_factory.mktemp("decoder23data"))
    synth_dataset.write_dataset(root, n_train=1, n_val=1, res=1024, hr=True)
    return root


def _install(deep, monkeypatch):
    patch.uninstall()
    monkeypatch.setenv("GPSG_DECODER", "1")
    if deep:
        monkeypatch.setenv("GPSG_DECODER_DEEP", "1")
    else:
        monkeypatch.delenv("GPSG_DECODER_DEEP", raising=False)
    for k in ("GPSG_GS_HEAD", "GPSG_GS_HEAD_TRAIN", "GPSG_ENCODER", "GPSG_ENCODER_DEEP"):
        monkeypatch.delenv(k, raising=False)
    harness.add_reference_to_path()
    patch.install()
    assert patch.decoder_deep() is deep


@needs_ref
def test_eval_forward_deep_on_off(dataset_1024, monkeypatch):
    """The eval forward at 1024^2 with GPSG_DECODER=1, GPSG_DECODER_DEEP on against off.  Tolerance: the kernels may move
    the regressor's maps by at most twice what the reference's own TF32 decoder3 / decoder2 move them, measured as the
    deep-off forward against one whose decoder3 and decoder2 run with cuDNN's TF32 off (full fp32)."""
    outs = {}
    decoder.reset_deep_counts()
    try:
        for run in ("off", "fp32", "on"):
            _install(run == "on", monkeypatch)
            monkeypatch.setattr(torch.backends.cudnn, "allow_tf32", True)
            cfg = harness.load_cfg(dataset_1024, src_res=1024, batch_size=1)
            st = harness.C3State(cfg)
            st.model.eval()
            hooks = []
            if run == "fp32":
                for mod in (st.model.gs_parm_regresser.decoder3, st.model.gs_parm_regresser.decoder2):
                    hooks += [mod.register_forward_pre_hook(lambda *a: setattr(torch.backends.cudnn, "allow_tf32", False)),
                              mod.register_forward_hook(lambda *a: setattr(torch.backends.cudnn, "allow_tf32", True))]
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
    assert decoder.deep_counts()["decoder2"] >= 1
    ref, yard, on = outs["off"], outs["fp32"], outs["on"]
    assert ref.keys() == on.keys() and ref
    stats = {}
    for k in ref:
        fin = torch.isfinite(ref[k])
        assert torch.equal(torch.isfinite(on[k]), fin), k
        stats[k] = (float((on[k] - ref[k])[fin].abs().mean()), float((yard[k] - ref[k])[fin].abs().mean()))
    record("decoder23:eval_switch", **{k: v[0] for k, v in stats.items()})
    print({k: f"deep {a:.3e} / reference fp32 decoder3+2 {b:.3e}" for k, (a, b) in stats.items()})
    for k, (a, b) in stats.items():
        assert a <= 2 * b, (k, a, b)


@needs_ref
def test_view_interp_runs_unmodified_with_every_encoder_and_regressor_switch(tmp_path):
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
    extra = {"GPSG_ENCODER": "1", "GPSG_ENCODER_DEEP": "1", "GPSG_GS_HEAD": "1", "GPSG_DECODER": "1",
             "GPSG_DECODER_DEEP": "1"}
    r = subprocess.run([sys.executable, "-c", _COUNTING_RUNNER + harness.SCRIPT_RUNNER, "test_view_interp.py",
                        "--test_data_root", os.path.join(dataset, "val"), "--ckpt_path", ckpt, "--novel_view_nums", "2"],
                       cwd=work, env=harness.script_env(patch=True, extra=extra), text=True, capture_output=True,
                       timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-6000:]
    line = [ln for ln in r.stdout.splitlines() if ln.startswith("decoder23 runs:")][-1]
    assert int(line.split(":")[1]) > 0, line


_COUNTING_RUNNER = ("import atexit\n"
                    "from gps_gaussian_b200 import decoder\n"
                    "atexit.register(lambda: print('decoder23 runs:', decoder.deep_counts()['decoder2'], flush=True))\n")
