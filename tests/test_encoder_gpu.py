"""GPU: the UnetExtractor's half-resolution stem (csrc/encoder_stem.cu through gps_gaussian_b200.encoder) against the
fp64 restatement (oracle/encoder_torch64.py) in both precisions, Cin 1 and 3, per element and with NaN exactly where
fp64 has it.  Two checks per case: x1 within the end-to-end bounds of fp64 from the input, and every stage (the five
stored convolution outputs and x1) within its own derived bound of fp64 from the kernels' stored input to that stage.
Sizes: B in {1, 2, 4} at 1024^2, the golden cases of the reference's module, and small odd shapes whose tiles do not
divide them.  Every output buffer is poisoned with NaN before each launch.  The worst utilisation per case goes to
$GPSG_PARITY_LOG.

Through `make_extractor_forward` on the reference's own UnetExtractor: no-grad fp32 and fp16-autocast calls take the
kernels, everything else is bit for bit the original forward.  With the staged reference: the RtStereoHumanModel eval
forward at 1024^2 with GPSG_ENCODER on and off, and test_view_interp.py run unmodified with GPSG_PATCH=1
GPSG_ENCODER=1 GPSG_GS_HEAD=1."""
import os
import subprocess
import sys
import types

import pytest
import torch

import encoder_cases as ec
from helpers import record
from gps_gaussian_b200 import encoder, harness, patch
from oracle import encoder_torch64 as et

pytestmark = pytest.mark.gpu
needs_ref = pytest.mark.skipif(harness.staged_reference() is None, reason="oracle/_ref not staged")
MODES = ("tf32", "fp16")


@pytest.fixture(autouse=True)
def poisoned_outputs(monkeypatch):
    """torch.empty inside encoder returns NaN-filled floating buffers, so an output element the kernels skip shows."""
    def nan(fn):
        def make(*a, **k):
            t = fn(*a, **k)
            if t.is_floating_point():
                t.fill_(float("nan"))
            return t
        return make
    fake = types.SimpleNamespace(**{n: getattr(torch, n) for n in dir(torch) if not n.startswith("__")})
    fake.empty, fake.empty_like = nan(torch.empty), nan(torch.empty_like)
    monkeypatch.setattr(encoder, "torch", fake)


def _check(tag, x, ps, mode, want=None, end_to_end=True):
    """Kernels on the device; per sample: x1 against fp64 within the chained bounds (end_to_end) and each stage within
    its own bound.  want: golden x1 (fp64) in place of forward64's."""
    dev = [p.cuda() for p in ps]
    x1, raws = encoder.forward_with_workspace(x.cuda(), dev, mode)
    worst = {}
    for n in range(x.shape[0]):
        xs = x[n:n + 1].cuda()
        if end_to_end:
            ref = et.forward64(xs, dev)["x1"] if want is None else want[n:n + 1].cuda()
            worst["x1"] = max(worst.get("x1", 0.0), et.ratio(x1[n:n + 1], ref, et.bounds(xs, dev, mode)["x1"]))
        stages = et.stage_checks(xs, dev, [r[n:n + 1] for r in raws], mode)
        got = dict(zip(("y0", "y1", "y2", "y3", "y4"), (r[n:n + 1] for r in raws)), x1=x1[n:n + 1])
        for k, (w, b) in stages.items():
            worst["stage_" + k] = max(worst.get("stage_" + k, 0.0), et.ratio(got[k], w, b))
    record(f"encoder:{tag}:{mode}", **worst)
    print(f"{tag} {mode}: utilisation {worst}")
    assert max(worst.values()) <= 1.0, worst
    return x1, raws


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("cin", [3, 1])
@pytest.mark.parametrize("B", [1, 2, 4])
def test_script_size(B, cin, mode):
    case = ec.Case(f"b{B}_c{cin}_1024", cin, B, 1024, 1024, 10 + B + cin)
    x, ps = ec.inputs(case)
    # the end-to-end bound chains worst cases (see oracle/encoder_torch64.py); at this size the stage checks carry it
    _check(case.id, x, ps, mode, end_to_end=False)


SMALL = ec.SWEEP + [ec.Case("rgb_odd_37x131", 3, 2, 37, 131, 20), ec.Case("depth_odd_9x257", 1, 3, 9, 257, 21),
                    ec.Case("rgb_column_70x1", 3, 1, 70, 1, 22), ec.Case("depth_row_1x300", 1, 2, 1, 300, 23)]


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("case", SMALL, ids=lambda c: c.id)
def test_small_shapes(case, mode):
    x, ps = ec.inputs(case)
    x1, _ = _check(case.id, x, ps, mode)
    if case.special in ("nan", "inf"):
        assert torch.isnan(x1[0]).all() and not torch.isnan(x1[1:]).any()


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("name", ec.GOLDEN_CASES)
def test_golden(name, mode):
    x, ps, want = ec.golden(name)
    _check("golden_" + name, x, ps, mode, want)


@pytest.mark.parametrize("mode", MODES)
def test_non_finite_pixel_poisons_only_its_sample(mode):
    x, ps = ec.inputs(ec.Case("b3", 3, 3, 64, 96, 30))
    dev = [p.cuda() for p in ps]
    clean = encoder.run(x.cuda(), dev, mode)
    for bad in (float("nan"), float("inf")):
        xb = x.clone()
        xb[1, 2, 40, 7] = bad
        got = encoder.run(xb.cuda(), dev, mode)
        assert torch.isnan(got[1]).all()
        assert torch.equal(got[0], clean[0]) and torch.equal(got[2], clean[2])


@pytest.mark.parametrize("mode", MODES)
def test_bit_reproducible(mode):
    x, ps = ec.inputs(ec.Case("b2", 3, 2, 512, 512, 31))
    dev = [p.cuda() for p in ps]
    a, b = encoder.run(x.cuda(), dev, mode), encoder.run(x.cuda(), dev, mode)
    assert torch.equal(a.view(torch.int32), b.view(torch.int32))


# ---- the rebound UnetExtractor.forward --------------------------------------------------------------------------------

def _extractor(cin=3, **kw):
    harness.add_reference_to_path()
    from core.extractor import UnetExtractor
    torch.manual_seed(4)
    m = UnetExtractor(in_channel=cin, **{"encoder_dim": [32, 48, 96], **kw}).eval()
    g = torch.Generator().manual_seed(5)
    with torch.no_grad():
        for mod in m.modules():
            if isinstance(mod, torch.nn.GroupNorm) and mod.affine:
                mod.weight.copy_(0.5 + torch.rand(mod.weight.shape, generator=g))
                mod.bias.copy_(torch.rand(mod.bias.shape, generator=g) - 0.5)
    return UnetExtractor, m


@needs_ref
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("cin", [3, 1])
def test_rebound_forward_runs_the_kernels(cin, mode):
    cls, m = _extractor(cin)
    m.cuda()
    fwd = encoder.make_extractor_forward(cls.forward)
    x = torch.rand(2, cin, 96, 160, device="cuda")
    encoder.reset_counts()
    with torch.no_grad(), torch.autocast("cuda", dtype=torch.float16, enabled=mode == "fp16"):
        x1, x2, x3 = fwd(m, x)
        want2 = m.res2(x1)
        want3 = m.res3(want2)
    assert encoder.counts()[mode] == 1
    assert x1.dtype == torch.float32 and torch.equal(x2, want2) and torch.equal(x3, want3)
    ps = [p.detach() for p in encoder.params_of(m)]
    ratio = et.ratio(x1, et.forward64(x, ps)["x1"], et.bounds(x, ps, mode)["x1"])
    record(f"encoder:rebound:{cin}:{mode}", x1=ratio)
    assert ratio <= 1.0


@needs_ref
@pytest.mark.parametrize("what", ["grad", "bf16_autocast", "allow_tf32_off", "cpu", "fp16_input", "dim64", "batch"])
def test_rebound_forward_falls_back_bit_for_bit(what, monkeypatch):
    kw = dict(encoder_dim=[64, 96, 128]) if what == "dim64" else (dict(norm_fn="batch") if what == "batch" else {})
    cls, m = _extractor(3, **kw)
    device = "cpu" if what == "cpu" else "cuda"
    m.to(device, torch.float16 if what == "fp16_input" else torch.float32)
    fwd = encoder.make_extractor_forward(cls.forward)
    monkeypatch.setattr(encoder, "run", lambda *a: pytest.fail("the kernels ran"))
    monkeypatch.setattr(encoder, "forward_with_workspace", lambda *a, **k: pytest.fail("the kernels ran"))
    if what == "allow_tf32_off":
        monkeypatch.setattr(torch.backends.cudnn, "allow_tf32", False)
    x = torch.rand(2, 3, 64, 96, device=device, dtype=torch.float16 if what == "fp16_input" else torch.float32)
    grad = torch.enable_grad() if what == "grad" else torch.no_grad()
    with grad, torch.autocast("cuda", dtype=torch.bfloat16, enabled=what == "bf16_autocast"):
        torch.manual_seed(0)
        got = fwd(m, x)
        torch.manual_seed(0)
        want = cls.forward(m, x)
    for g, w in zip(got, want):
        assert torch.equal(g, w)


# ---- the reference's model and scripts with the switch --------------------------------------------------------------

@pytest.fixture(scope="module")
def dataset_1024(tmp_path_factory):
    from gps_gaussian_b200 import synth_dataset
    root = str(tmp_path_factory.mktemp("encoderdata"))
    synth_dataset.write_dataset(root, n_train=1, n_val=1, res=1024, hr=True)
    return root


def _install(on, monkeypatch):
    patch.uninstall()
    if on:
        monkeypatch.setenv("GPSG_ENCODER", "1")
    else:
        monkeypatch.delenv("GPSG_ENCODER", raising=False)
    harness.add_reference_to_path()
    patch.install()
    import core.extractor
    assert (core.extractor.UnetExtractor.forward.__module__ == encoder.__name__) is on


def _fp32_stem_forward(orig):
    """UnetExtractor.forward with in_ds + res1 in full fp32 (autocast and TF32 off): the yardstick run."""
    def forward(self, x):
        with torch.autocast("cuda", enabled=False):
            x1 = self.res1(self.in_ds(x.float()))
        x2 = self.res2(x1)
        return x1, x2, self.res3(x2)
    return forward


@needs_ref
def test_eval_forward_switch_on_off(dataset_1024, monkeypatch):
    """The eval forward at 1024^2 (the stage-2 config: the image encoder under fp16 autocast, the depth encoder in fp32),
    switch on against off.  Tolerance: the kernels may move the flow, depth and Gaussian maps by at most twice what the
    reduced precision of the reference's own stems moves them, measured as the switched-off forward against one whose
    stems run in full fp32 (autocast and TF32 off for in_ds + res1 and cuDNN TF32 off elsewhere).  The kernels differ
    from cuDNN only by where fp16 / TF32 rounding and fp32 re-association fall, so they must stay within that scale."""
    outs = {}
    encoder.reset_counts()
    try:
        for run in ("off", "fp32", "on"):
            _install(run == "on", monkeypatch)
            monkeypatch.setattr(torch.backends.cudnn, "allow_tf32", run != "fp32")
            import core.extractor
            cls = core.extractor.UnetExtractor
            saved = cls.__dict__["forward"]
            if run == "fp32":
                cls.forward = _fp32_stem_forward(saved)
            cfg = harness.load_cfg(dataset_1024, src_res=1024, batch_size=1)
            st = harness.C3State(cfg)
            st.model.eval()
            data = st.batch(0)
            with torch.no_grad():
                out, _, _ = st.model({k: dict(v) if isinstance(v, dict) else v for k, v in data.items()}, is_train=False)
            outs[run] = {f"{v}_{k}": out[v][k].float().clone() for v in ("lmain", "rmain")
                         for k in ("flow_pred", "depth", "rot_maps", "scale_maps", "opacity_maps") if k in out[v]}
            cls.forward = saved
            del st, out, data
            torch.cuda.empty_cache()
    finally:
        patch.uninstall()
    c = encoder.counts()
    assert c["tf32"] >= 1 and c["fp16"] >= 1                     # the depth encoder in fp32, the image encoder in fp16
    ref, yard, on = outs["off"], outs["fp32"], outs["on"]
    assert ref.keys() == on.keys() and ref
    stats = {}
    for k in ref:
        fin = torch.isfinite(ref[k])
        assert torch.equal(torch.isfinite(on[k]), fin), k
        stats[k] = (float((on[k] - ref[k])[fin].abs().mean()), float((yard[k] - ref[k])[fin].abs().mean()))
    record("encoder:eval_switch", **{k: v[0] for k, v in stats.items()})
    print({k: f"switch {a:.3e} / reference fp32 stems {b:.3e}" for k, (a, b) in stats.items()})
    for k, (a, b) in stats.items():
        assert a <= 2 * b, (k, a, b)


@needs_ref
def test_view_interp_runs_unmodified_with_encoder_and_gs_head(tmp_path):
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
    r = subprocess.run([sys.executable, "-c", _COUNTING_RUNNER + harness.SCRIPT_RUNNER, "test_view_interp.py",
                        "--test_data_root", os.path.join(dataset, "val"), "--ckpt_path", ckpt, "--novel_view_nums", "2"],
                       cwd=work, env=harness.script_env(patch=True, extra={"GPSG_ENCODER": "1", "GPSG_GS_HEAD": "1"}),
                       text=True, capture_output=True, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-6000:]
    line = [ln for ln in r.stdout.splitlines() if ln.startswith("encoder runs:")][-1]
    fp16, tf32 = (int(v) for v in line.split(":")[1].split())
    assert fp16 >= 1 and tf32 >= 1, line                    # the image encoder under autocast, the depth encoder in fp32


_COUNTING_RUNNER = ("import atexit\n"
                    "from gps_gaussian_b200 import encoder\n"
                    "atexit.register(lambda: print('encoder runs:', encoder.counts()['fp16'], encoder.counts()['tf32'],"
                    " flush=True))\n")
