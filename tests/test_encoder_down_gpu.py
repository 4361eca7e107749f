"""GPU: the UnetExtractor's stride-2 residual stages res2 / res3 (csrc/encoder_down.cu through
gps_gaussian_b200.encoder.run_down) against the fp64 restatement (oracle/encoder_down_torch64.py) in both precisions.
Every stage (the five stored convolution outputs and the stage output) is checked within its own derived bound of fp64
from the kernels' stored input to that stage (the chained end-to-end bounds are too loose past two GroupNorms to say
anything; the golden cases pin fp64 to the reference's own modules on the CPU).  Sizes: the stages of a 1024^2 input at
B = 1, 2, 4, odd shapes whose tiles do not divide them, down to 1 x 1, and the golden inputs.  Every output buffer is poisoned with NaN before each launch.

Through `make_extractor_forward(orig, deep=True)` on the reference's own UnetExtractor: no-grad fp32 and fp16-autocast
calls run x1, x2 and x3 on the kernels, everything else is bit for bit the original forward.  With the staged
reference: the RtStereoHumanModel eval forward at 1024^2 with GPSG_ENCODER_DEEP on and off, and test_view_interp.py run
unmodified with every regressor and encoder switch on."""
import os
import subprocess
import sys
import types

import numpy as np
import pytest
import torch

from helpers import record
from gps_gaussian_b200 import encoder, harness, patch
from oracle import encoder_down_torch64 as ed

pytestmark = pytest.mark.gpu
needs_ref = pytest.mark.skipif(harness.staged_reference() is None, reason="oracle/_ref not staged")
MODES = ("tf32", "fp16")
STAGES = {"res2": (32, 48), "res3": (48, 96)}
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "encoder_down_golden.npz")


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


def params(cin, c, seed):
    """Conv2d's default init (uniform in +-1/sqrt(fan_in)), GroupNorm weights in [0.5, 1.5], biases in [-0.5, 0.5]."""
    g = torch.Generator().manual_seed(seed)
    out = []
    for i, s in enumerate(encoder.down_param_shapes(cin, c)):
        if len(s) == 4:
            k = 1.0 / (s[1] * s[2] * s[3]) ** 0.5
            out.append((torch.rand(s, generator=g) * 2 - 1) * k)
        elif i % 4 == 1:                                   # conv bias
            k = 1.0 / (cin * 9 if i == 1 else (cin if i == 9 else c * 9)) ** 0.5
            out.append((torch.rand(s, generator=g) * 2 - 1) * k)
        elif i % 4 == 2:
            out.append(0.5 + torch.rand(s, generator=g))
        else:
            out.append(torch.rand(s, generator=g) - 0.5)
    return out


def stage_input(cin, B, H, W, seed):
    """A post-ReLU feature map like the previous stage's output: non-negative, with exact zeros."""
    g = torch.Generator().manual_seed(seed)
    return torch.relu(torch.randn(B, cin, H, W, generator=g))


def _check(tag, x, ps, mode):
    dev = [p.cuda() for p in ps]
    out, raws = encoder.down_forward_with_workspace(x.cuda(), dev, mode)
    worst = {}
    for n in range(x.shape[0]):
        xs = x[n:n + 1].cuda()
        stages = ed.stage_checks(xs, dev, [r[n:n + 1] for r in raws], mode)
        got = dict(zip(ed.KEYS, [r[n:n + 1] for r in raws] + [out[n:n + 1]]))
        for k, (w, b) in stages.items():
            worst["stage_" + k] = max(worst.get("stage_" + k, 0.0), ed.ratio(got[k], w, b))
    record(f"encoder_down:{tag}:{mode}", **worst)
    print(f"{tag} {mode}: utilisation {worst}")
    assert max(worst.values()) <= 1.0, worst
    return out, raws


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("stage", ["res2", "res3"])
@pytest.mark.parametrize("B", [1, 2, 4])
def test_script_size(B, stage, mode):
    cin, c = STAGES[stage]
    H = 512 if stage == "res2" else 256                    # the stage inputs of a 1024^2 image
    _check(f"{stage}_b{B}", stage_input(cin, B, H, H, B + cin), params(cin, c, 40 + B), mode)


SMALL = [(1, 9, 5), (2, 17, 130), (1, 1, 1), (3, 2, 1), (1, 1, 300), (2, 70, 3), (1, 5, 129), (2, 33, 257)]


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("stage", ["res2", "res3"])
@pytest.mark.parametrize("shape", SMALL, ids=lambda s: "x".join(map(str, s)))
def test_small_shapes(shape, stage, mode):
    cin, c = STAGES[stage]
    B, H, W = shape
    _check(f"{stage}_{B}x{H}x{W}", stage_input(cin, B, H, W, H * W), params(cin, c, H + W), mode)


@pytest.mark.parametrize("mode", MODES)
def test_golden(mode):
    z = np.load(GOLDEN)
    names = sorted(k[:-2] for k in z.files if k.endswith("_x"))
    assert names
    for name in names:
        x = torch.from_numpy(z[name + "_x"])
        stage = name.split("_")[0]
        ps = [torch.from_numpy(z[f"{name}_p{i}"] if f"{name}_p{i}" in z.files else z[f"{stage}_p{i}"])
              for i in range(20)]
        _check("golden_" + name, x, ps, mode)


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("stage", ["res2", "res3"])
def test_non_finite_pixel_poisons_only_its_sample(stage, mode):
    cin, c = STAGES[stage]
    x, ps = stage_input(cin, 3, 40, 72, 7), params(cin, c, 8)
    dev = [p.cuda() for p in ps]
    clean = encoder.run_down(x.cuda(), dev, mode)
    assert torch.isfinite(clean).all()
    for bad in (float("nan"), float("inf")):
        xb = x.clone()
        xb[1, 5, 21, 9] = bad
        got = encoder.run_down(xb.cuda(), dev, mode)
        # every group of sample 1 reads the bad pixel through conv1 / the downsample, whose outputs mix all channels
        assert torch.isnan(got[1]).all()
        assert torch.equal(got[0], clean[0]) and torch.equal(got[2], clean[2])


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("stage", ["res2", "res3"])
@pytest.mark.parametrize("bad", [float("nan"), float("inf")])
def test_non_finite_channel_stays_in_its_group(bad, stage, mode):
    """A non-finite bias makes one channel of a raw output non-finite; its GroupNorm group turns NaN and the other groups
    keep their statistics: conv1's bad channel leaves ya's other channels and yd as they were, and block 1's conv2's
    reaches the output only in its own group, every other channel bit-identical to the clean run."""
    cin, c = STAGES[stage]
    x, ps = stage_input(cin, 2, 21, 34, 11), params(cin, c, 12)
    dev = [p.cuda() for p in ps]
    clean, craws = encoder.down_forward_with_workspace(x.cuda(), dev, mode)
    g = 1
    for idx, raw in ((1, 0), (17, 4)):                     # b0_conv1 bias -> ya; b1_conv2 bias -> ye
        bad_ps = [p.clone() for p in dev]
        bad_ps[idx][8 * g + 3] = bad
        out, raws = encoder.down_forward_with_workspace(x.cuda(), bad_ps, mode)
        other = torch.ones(c, dtype=torch.bool, device="cuda")
        other[8 * g + 3] = False
        assert not torch.isfinite(raws[raw][:, 8 * g + 3]).any()
        assert torch.equal(raws[raw][:, other], craws[raw][:, other])
        if raw == 0:
            assert torch.equal(raws[1], craws[1])          # the downsample branch never reads ya
        else:
            grp = torch.zeros(c, dtype=torch.bool, device="cuda")
            grp[8 * g:8 * g + 8] = True
            assert torch.isnan(out[:, grp]).all()
            assert torch.equal(out[:, ~grp], clean[:, ~grp])


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("stage", ["res2", "res3"])
def test_bit_reproducible(stage, mode):
    cin, c = STAGES[stage]
    x, ps = stage_input(cin, 2, 256, 256, 9), params(cin, c, 10)
    dev = [p.cuda() for p in ps]
    a, b = encoder.run_down(x.cuda(), dev, mode), encoder.run_down(x.cuda(), dev, mode)
    assert torch.equal(a.view(torch.int32), b.view(torch.int32))


def test_foreign_dims_refused():
    x = torch.rand(1, 64, 8, 8, device="cuda")
    with pytest.raises(RuntimeError):
        encoder.run_down(x, [p.cuda() for p in params(64, 96, 0)], "tf32")


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
@pytest.mark.parametrize("B", [1, 2, 4])
def test_deep_forward_runs_the_kernels(B, cin, mode):
    cls, m = _extractor(cin)
    m.cuda()
    fwd = encoder.make_extractor_forward(cls.forward, deep=True)
    x = torch.rand(B, cin, 1024, 1024, device="cuda")
    encoder.reset_counts()
    encoder.reset_down_counts()
    with torch.no_grad(), torch.autocast("cuda", dtype=torch.float16, enabled=mode == "fp16"):
        x1, x2, x3 = fwd(m, x)
    assert encoder.counts()[mode] == 1 and encoder.down_counts()[mode] == 2
    assert torch.equal(x1, encoder.run(x, encoder.params_of(m), mode))
    assert x2.shape == (B, 48, 256, 256) and x3.shape == (B, 96, 128, 128)
    assert x2.dtype == torch.float32 and x3.dtype == torch.float32
    for name, v, want in (("res2", x1, x2), ("res3", x2, x3)):
        ps = [p.detach() for p in encoder.down_params_of(getattr(m, name))]
        out, _ = _check(f"deep_{name}_b{B}_c{cin}", v, ps, mode)
        assert torch.equal(out, want)


@needs_ref
@pytest.mark.parametrize("what", ["grad", "bf16_autocast", "allow_tf32_off", "dim64", "batch", "shallow"])
def test_deep_forward_falls_back_bit_for_bit(what, monkeypatch):
    kw = dict(encoder_dim=[64, 96, 128]) if what == "dim64" else (dict(norm_fn="batch") if what == "batch" else {})
    cls, m = _extractor(3, **kw)
    m.cuda()
    fwd = encoder.make_extractor_forward(cls.forward, deep=what != "shallow")
    monkeypatch.setattr(encoder, "run_down", lambda *a: pytest.fail("the down kernels ran"))
    monkeypatch.setattr(encoder, "down_forward_with_workspace", lambda *a, **k: pytest.fail("the down kernels ran"))
    if what == "allow_tf32_off":
        monkeypatch.setattr(torch.backends.cudnn, "allow_tf32", False)
    x = torch.rand(2, 3, 64, 96, device="cuda")
    grad = torch.enable_grad() if what == "grad" else torch.no_grad()
    with grad, torch.autocast("cuda", dtype=torch.bfloat16, enabled=what == "bf16_autocast"):
        got = fwd(m, x)
        if what == "shallow":                              # deep=False: the stem kernels, then the module's res2, res3
            x1 = encoder.run(x, encoder.params_of(m), "tf32")
            want = (x1, m.res2(x1), m.res3(m.res2(x1)))
        else:
            want = cls.forward(m, x)
    for g, w in zip(got, want):
        assert torch.equal(g, w)


@needs_ref
def test_deep_forward_falls_back_on_a_foreign_norm(monkeypatch):
    cls, m = _extractor(3)
    m.res3[1].norm2 = torch.nn.GroupNorm(6, 96).eval()     # another group count: the stem alone takes the kernels
    m.cuda()
    fwd = encoder.make_extractor_forward(cls.forward, deep=True)
    monkeypatch.setattr(encoder, "run_down", lambda *a: pytest.fail("the down kernels ran"))
    x = torch.rand(1, 3, 64, 96, device="cuda")
    with torch.no_grad():
        got = fwd(m, x)
        x1 = encoder.run(x, encoder.params_of(m), "tf32")
        want = (x1, m.res2(x1), m.res3(m.res2(x1)))
    for g, w in zip(got, want):
        assert torch.equal(g, w)


# ---- the reference's model and scripts with the switch --------------------------------------------------------------

@pytest.fixture(scope="module")
def dataset_1024(tmp_path_factory):
    from gps_gaussian_b200 import synth_dataset
    root = str(tmp_path_factory.mktemp("encoderdowndata"))
    synth_dataset.write_dataset(root, n_train=1, n_val=1, res=1024, hr=True)
    return root


ALL_ON = {"GPSG_ENCODER": "1", "GPSG_GS_HEAD": "1", "GPSG_DECODER": "1"}


def _install(env, monkeypatch):
    patch.uninstall()
    for k in ("GPSG_ENCODER", "GPSG_ENCODER_DEEP", "GPSG_GS_HEAD", "GPSG_DECODER"):
        monkeypatch.delenv(k, raising=False)
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    harness.add_reference_to_path()
    patch.install()


def _fp32_encoder_forward(orig):
    """UnetExtractor.forward entirely in fp32 (autocast and TF32 off): the yardstick run."""
    def forward(self, x):
        with torch.autocast("cuda", enabled=False):
            x1 = self.res1(self.in_ds(x.float()))
            x2 = self.res2(x1)
            return x1, x2, self.res3(x2)
    return forward


@needs_ref
def test_eval_forward_switch_on_off(dataset_1024, monkeypatch):
    """The eval forward at 1024^2 with every other switch on, GPSG_ENCODER_DEEP on against off.  Tolerance: the kernels
    may move the flow, depth and Gaussian maps by at most twice what the reduced precision of the reference's own encoders
    moves them, measured as the switched-off forward against one whose encoders run in full fp32 (autocast and TF32 off)
    with cuDNN TF32 off elsewhere."""
    outs = {}
    encoder.reset_down_counts()
    try:
        for run in ("off", "fp32", "on"):
            _install({**ALL_ON, "GPSG_ENCODER_DEEP": "1"} if run == "on" else {} if run == "fp32" else ALL_ON,
                     monkeypatch)
            assert patch.encoder_deep() is (run == "on")
            monkeypatch.setattr(torch.backends.cudnn, "allow_tf32", run != "fp32")
            import core.extractor
            cls = core.extractor.UnetExtractor
            saved = cls.__dict__["forward"]
            if run == "fp32":
                cls.forward = _fp32_encoder_forward(saved)
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
    c = encoder.down_counts()
    assert c["tf32"] >= 2 and c["fp16"] >= 2                 # the depth encoder in fp32, the image encoder in fp16
    ref, yard, on = outs["off"], outs["fp32"], outs["on"]
    assert ref.keys() == on.keys() and ref
    stats = {}
    for k in ref:
        fin = torch.isfinite(ref[k])
        assert torch.equal(torch.isfinite(on[k]), fin), k
        stats[k] = (float((on[k] - ref[k])[fin].abs().mean()), float((yard[k] - ref[k])[fin].abs().mean()))
    record("encoder_down:eval_switch", **{k: v[0] for k, v in stats.items()})
    print({k: f"switch {a:.3e} / reference fp32 encoders {b:.3e}" for k, (a, b) in stats.items()})
    for k, (a, b) in stats.items():
        assert a <= 2 * b, (k, a, b)


@needs_ref
def test_view_interp_runs_unmodified_with_every_switch(tmp_path):
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
    env = harness.script_env(patch=True, extra={**ALL_ON, "GPSG_ENCODER_DEEP": "1"})
    r = subprocess.run([sys.executable, "-c", _COUNTING_RUNNER + harness.SCRIPT_RUNNER, "test_view_interp.py",
                        "--test_data_root", os.path.join(dataset, "val"), "--ckpt_path", ckpt, "--novel_view_nums", "2"],
                       cwd=work, env=env, text=True, capture_output=True, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-6000:]
    line = [ln for ln in r.stdout.splitlines() if ln.startswith("encoder_down runs:")][-1]
    fp16, tf32 = (int(v) for v in line.split(":")[1].split())
    assert fp16 >= 2 and tf32 >= 2, line


_COUNTING_RUNNER = ("import atexit\n"
                    "from gps_gaussian_b200 import encoder\n"
                    "atexit.register(lambda: print('encoder_down runs:', encoder.down_counts()['fp16'],"
                    " encoder.down_counts()['tf32'], flush=True))\n")
