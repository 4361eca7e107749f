"""GPU: the disparity update block (csrc/update_block.cu through gps_gaussian_b200.update) against the fp64 restatement
and the fp16-route stage bounds (oracle/update_torch64.py).

Every stage of one iteration is checked per element from the kernels' own stored inputs to it: the fp16 route is a
monotone function of the exact convolution sums, so the bound is zero wherever the fp32 accumulation error cannot move
a rounding.  Sizes: the 1/8-resolution maps of a 1024^2 pair at B = 2 and 4, odd shapes down to 1 x 1 and widths that
are not a multiple of the 64-column tile, corr in fp16 and fp32, and the golden inputs; the outputs and the workspace
are NaN before each launch.  Three test-mode and three
training-mode iterations through `make_update_forward` on the reference's own FlowUpdateModule: the kernel route's error
against the fp64 loop is at most twice that of the module's own autocast route.  flow_init, non-finite inputs, repeats,
every fallback bit for bit, and with the staged reference the RtStereoHumanModel eval forward with GPSG_UPDATE on and
off and test_view_interp.py run unmodified with every switch on."""
import os
import subprocess
import sys
import types

import numpy as np
import pytest
import torch

import update_cases as uc
from helpers import record
from gps_gaussian_b200 import harness, patch, update
from oracle import update_torch64 as ut

pytestmark = pytest.mark.gpu
needs_ref = pytest.mark.skipif(harness.staged_reference() is None, reason="oracle/_ref not staged")
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "update_golden.npz")


@pytest.fixture(autouse=True)
def poisoned_outputs(monkeypatch):
    """torch.empty inside update returns NaN-filled floating buffers and 0xFF-filled bytes (NaN in every fp16 view of
    the workspace), so an element the kernels skip shows."""
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
    monkeypatch.setattr(update, "torch", fake)


def params(seed):
    """Conv2d's default init: weights and biases uniform in +-1/sqrt(fan_in), fp32."""
    g = torch.Generator().manual_seed(seed)
    out = []
    for i, s in enumerate(update.PARAM_SHAPES):
        fan = update.PARAM_SHAPES[i - (i % 2)]
        k = 1.0 / (fan[1] * fan[2] * fan[3]) ** 0.5
        out.append(((torch.rand(s, generator=g) * 2 - 1) * k).float())
    return out


def inputs(B, H, W, seed, corr_dtype=torch.float16):
    g = torch.Generator().manual_seed(seed)
    corr = (torch.randn(B, 36, H, W, generator=g) * 2).to(corr_dtype)
    ys, xs = torch.meshgrid(torch.arange(H, dtype=torch.float32), torch.arange(W, dtype=torch.float32), indexing="ij")
    coords1 = torch.stack([xs, ys])[None] + torch.randn(B, 2, H, W, generator=g) * 3
    net = torch.tanh(torch.randn(B, 96, H, W, generator=g)).half()
    czrq = (torch.randn(B, 288, H, W, generator=g) * 0.7).half()
    return dict(corr=corr, coords1=coords1.float(), net=net, czrq=czrq)


def _check(tag, ps, inp, mask=True):
    dev = {k: v.cuda() for k, v in inp.items()}
    got = update.step_with_workspace(dev["corr"], dev["coords1"], dev["net"], dev["czrq"], [p.cuda() for p in ps],
                                     mask=mask)
    got["czrq"] = dev["czrq"]
    worst = {}
    chk = ut.stage_checks(ps, got)
    for k in ut.KEYS:
        if k in ("m1", "mask") and not mask:
            continue
        worst[k] = ut.ratio(got[k], *chk[k])
    record(f"update:{tag}", **worst)
    print(f"{tag}: utilisation {worst}")
    assert max(worst.values()) <= 1.0, worst
    return got


@pytest.mark.parametrize("B", [2, 4])
def test_script_size(B):
    _check(f"b{B}_128", params(B), inputs(B, 128, 128, 10 + B))


SMALL = [(1, 1, 1), (2, 3, 5), (1, 9, 7), (2, 5, 70), (1, 17, 130), (3, 2, 65), (1, 1, 300), (2, 64, 64)]


@pytest.mark.parametrize("corr_dtype", [torch.float16, torch.float32], ids=["fp16", "fp32"])
@pytest.mark.parametrize("shape", SMALL, ids=lambda s: "x".join(map(str, s)))
def test_small_shapes(shape, corr_dtype):
    B, H, W = shape
    _check(f"{B}x{H}x{W}", params(H + W), inputs(B, H, W, H * W, corr_dtype))


def test_without_mask():
    got = _check("nomask_2x9x70", params(3), inputs(2, 9, 70, 4), mask=False)
    assert "mask" not in got


# ---- the reference's modules --------------------------------------------------------------------------------------------

def _args(**kw):
    a = types.SimpleNamespace(mixed_precision=True, n_gru_layers=1, slow_fast_gru=None, hidden_dims=[96, 96, 96],
                              corr_levels=4, corr_radius=4, n_downsample=3, corr_implementation="reg")
    for k, v in kw.items():
        setattr(a, k, v)
    return a


def _module(seed=0, **kw):
    harness.add_reference_to_path()
    import core.raft_stereo_human as rsh
    torch.manual_seed(seed)
    return rsh, rsh.FlowUpdateModule(_args(**kw)).cuda().eval()


@needs_ref
def test_golden():
    """The golden single-iteration cases (the reference's own BasicMultiUpdateBlock in fp64): every stage within its
    bound, and the kernels' h, delta and mask no further from the golden than twice the module's autocast route."""
    z = np.load(GOLDEN)
    ps = uc.params(0)
    _, m = _module()
    blk = m.update_block
    with torch.no_grad():
        for p, v in zip(update.params_of(blk), ps):
            p.copy_(v)
    for B, H, W in uc.STEP_CASES:
        inp = uc.inputs(B, H, W)
        got = _check(f"golden_{B}x{H}x{W}", [p.float() for p in ps],
                     dict(corr=inp["corr"].half(), coords1=inp["coords1"].float(), net=inp["net"].half(),
                          czrq=inp["czrq"].half()))
        tag = f"step_{B}x{H}x{W}_"
        flow = (inp["coords1"].float() - ut.grid(B, H, W).float()).cuda()
        cz, cr, cq = inp["czrq"].half().cuda().split(96, 1)
        with torch.no_grad(), torch.autocast("cuda", dtype=torch.float16):
            net, mask, delta = blk([inp["net"].half().cuda()], [[cz, cr, cq]], inp["corr"].half().cuda(), flow,
                                   iter32=False, iter16=False)
        for k, ref in (("h", net[0]), ("delta", delta), ("mask", mask)):
            want = torch.from_numpy(z[tag + k])
            e_k = float((got[k].double().cpu() - want).abs().mean())
            e_r = float((ref.double().cpu() - want).abs().mean())
            assert e_k <= 2 * e_r + 1e-7, (tag, k, e_k, e_r)


def _forward_inputs(B, H, W, seed, D=64):
    g = torch.Generator().manual_seed(seed)
    f1 = (torch.randn(B, D, H, W, generator=g)).half().cuda()
    f2 = (torch.randn(B, D, H, W, generator=g)).half().cuda()
    net = torch.tanh(torch.randn(B, 96, H, W, generator=g)).half().cuda()
    ctx = (torch.randn(B, 288, H, W, generator=g) * 0.7).half().cuda()
    return f1, f2, net, ctx


def _run(fwd, m, f1, f2, net, ctx, iters, flow_init=None, test_mode=True):
    with torch.no_grad():
        return fwd(m, f1, f2, [net.clone()], [list(ctx.split(96, 1))], iters, flow_init, test_mode)


def _err(a, b):
    return float((a.double() - b.double()).abs().mean())


@needs_ref
@pytest.mark.parametrize("test_mode", [True, False], ids=["test", "train"])
@pytest.mark.parametrize("shape", [(2, 128, 128), (1, 20, 37)], ids=lambda s: "x".join(map(str, s)))
@pytest.mark.parametrize("flow_init", [False, True], ids=["zero", "flow_init"])
def test_loop_against_fp64(shape, test_mode, flow_init):
    B, H, W = shape
    rsh, m = _module(seed=B + H)
    orig = rsh.FlowUpdateModule.__dict__["forward"]
    ours = update.make_update_forward(orig)
    f1, f2, net, ctx = _forward_inputs(B, H, W, H * W)
    fi = (torch.randn(B, 2, H, W, generator=torch.Generator().manual_seed(9)) * 2).cuda() if flow_init else None
    if fi is not None:
        fi[:, 1] = 0
    update.reset_update_counts()
    got = _run(ours, m, f1, f2, net, ctx, 3, fi, test_mode)
    assert update.update_counts() == {"steps": 3, "forwards": 1}
    ref = _run(orig, m, f1, f2, net, ctx, 3, fi, test_mode)
    want = ut.loop64(update.params_of(m.update_block), f1, f2, net, ctx, 3, fi, test_mode)
    got, ref, want = ([got], [ref], [want]) if test_mode else (got, ref, want)
    assert len(got) == len(ref) == len(want) == (1 if test_mode else 3)
    for i, (g, r, w) in enumerate(zip(got, ref, want)):
        assert g.shape == r.shape == w.shape and g.dtype == r.dtype
        e_k, e_r = _err(g, w), _err(r, w)
        record(f"update:loop_{B}x{H}x{W}_{test_mode}_{flow_init}_{i}", kernels=e_k, reference=e_r)
        print(f"prediction {i}: kernels {e_k:.3e} / reference autocast {e_r:.3e}")
        assert e_k <= 2 * e_r, (i, e_k, e_r)


@needs_ref
def test_repeats_bit_identical_and_hidden_state_returned():
    rsh, m = _module()
    ours = update.make_update_forward(rsh.FlowUpdateModule.__dict__["forward"])
    f1, f2, net, ctx = _forward_inputs(2, 128, 128, 3)
    outs = []
    for _ in range(2):
        nl = [net.clone()]
        with torch.no_grad():
            outs.append((ours(m, f1, f2, nl, [list(ctx.split(96, 1))], 3, None, True), nl[0].clone()))
    assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])
    assert outs[0][1].shape == net.shape and outs[0][1].dtype == torch.float16
    assert not torch.equal(outs[0][1], net)


@needs_ref
@pytest.mark.parametrize("where", ["corr", "net"])
def test_non_finite_stays_in_its_sample(where, monkeypatch):
    rsh, m = _module()
    ours = update.make_update_forward(rsh.FlowUpdateModule.__dict__["forward"])
    f1, f2, net, ctx = _forward_inputs(2, 32, 40, 5)
    clean = _run(ours, m, f1, f2, net, ctx, 3)
    if where == "net":
        net = net.clone()
        net[1, 7, 10, 11] = float("nan")
    else:
        real = update.step

        def poisoned(corr, *a, **k):
            corr = corr.clone()
            corr[1, 3, 4, 5] = float("inf")
            return real(corr, *a, **k)
        monkeypatch.setattr(update, "step", poisoned)
    bad = _run(ours, m, f1, f2, net, ctx, 3)
    assert torch.equal(bad[0], clean[0])
    assert not torch.isfinite(bad[1]).all()


@needs_ref
@pytest.mark.parametrize("what", ["grad", "fp32_eval", "corr_radius", "n_downsample", "foreign_layer", "cpu",
                                  "net_fp32", "iters0"])
def test_fallbacks_bit_for_bit(what):
    kw = dict(mixed_precision=False) if what == "fp32_eval" else dict(corr_radius=3) if what == "corr_radius" \
        else dict(n_downsample=2) if what == "n_downsample" else {}
    rsh, m = _module(**kw)
    if what == "foreign_layer":
        m.update_block.mask[1] = torch.nn.LeakyReLU(0.0)
    orig = rsh.FlowUpdateModule.__dict__["forward"]
    ours = update.make_update_forward(orig)
    f1, f2, net, ctx = _forward_inputs(1, 16, 24, 6)
    iters = 0 if what == "iters0" else 2
    if what == "cpu":
        m = m.cpu()
        f1, f2, net, ctx = f1.cpu(), f2.cpu(), net.float().cpu(), ctx.float().cpu()
    if what == "net_fp32":
        net = net.float()
    if what == "fp32_eval":
        f1, f2, net, ctx = f1.float(), f2.float(), net.float(), ctx.float()
    update.reset_update_counts()
    results = []
    for fwd in (ours, orig):
        torch.manual_seed(0)
        try:
            with torch.set_grad_enabled(what == "grad"):
                out = fwd(m, f1, f2, [net.clone()], [list(ctx.split(96, 1))], iters, None, True)
            results.append(out.detach() if torch.is_tensor(out) else out)
        except Exception as exc:                # iters = 0: the reference's own error, both times
            results.append(type(exc))
    assert update.update_counts()["steps"] == 0
    a, b = results
    assert (torch.equal(a, b) if torch.is_tensor(a) else a == b), what


# ---- the reference's model and scripts with the switch --------------------------------------------------------------

@pytest.fixture(scope="module")
def dataset_1024(tmp_path_factory):
    from gps_gaussian_b200 import synth_dataset
    root = str(tmp_path_factory.mktemp("updatedata"))
    synth_dataset.write_dataset(root, n_train=1, n_val=1, res=1024, hr=True)
    return root


ALL_ON = {"GPSG_FLOW_HEAD": "1", "GPSG_ENCODER": "1", "GPSG_ENCODER_DEEP": "1", "GPSG_GS_HEAD": "1",
          "GPSG_DECODER": "1"}


def _install(env, monkeypatch):
    patch.uninstall()
    for k in (*ALL_ON, "GPSG_UPDATE"):
        monkeypatch.delenv(k, raising=False)
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    harness.add_reference_to_path()
    patch.install()


@needs_ref
def test_eval_forward_switch_on_off(dataset_1024, monkeypatch):
    """The eval forward at 1024^2 with every other switch on, GPSG_UPDATE on against off.  Tolerance: the kernels may
    move the flow by at most twice what the reference's fp16 update block moves it, measured as the switched-off forward
    against one whose update block runs in fp32 (mixed_precision off inside FlowUpdateModule only)."""
    outs = {}
    update.reset_update_counts()
    try:
        for run in ("off", "fp32", "on"):
            _install({**ALL_ON, "GPSG_UPDATE": "1"} if run == "on" else ALL_ON, monkeypatch)
            assert patch.update() is (run == "on")
            cfg = harness.load_cfg(dataset_1024, src_res=1024, batch_size=1)
            st = harness.C3State(cfg)
            st.model.eval()
            if run == "fp32":
                _fp32_update_module(st.model.raft_stereo.update_module)
            data = st.batch(0)
            with torch.no_grad():
                out, _, _ = st.model({k: dict(v) if isinstance(v, dict) else v for k, v in data.items()}, is_train=False)
            outs[run] = {f"{v}_flow_pred": out[v]["flow_pred"].float().clone() for v in ("lmain", "rmain")}
            del st, out, data
            torch.cuda.empty_cache()
    finally:
        patch.uninstall()
    assert update.update_counts()["forwards"] >= 1
    ref, yard, on = outs["off"], outs["fp32"], outs["on"]
    for k in ref:
        fin = torch.isfinite(ref[k])
        assert torch.equal(torch.isfinite(on[k]), fin), k
        a, b = float((on[k] - yard[k])[fin].abs().mean()), float((ref[k] - yard[k])[fin].abs().mean())
        record("update:eval_switch", **{k: a, k + "_reference": b})
        print(f"{k}: switch {a:.3e} / reference fp16 {b:.3e}")
        assert a <= 2 * b, (k, a, b)


def _fp32_update_module(um):
    """The yardstick run: this FlowUpdateModule with mixed_precision off and its fp16 inputs from cnet cast to fp32, so
    that the update block runs in fp32 while the rest of the model keeps its precision."""
    import copy
    a = copy.deepcopy(um.args)
    if hasattr(a, "defrost"):
        a.defrost()
    a.mixed_precision = False
    um.args = a
    orig = um.forward

    def forward(fmap1, fmap2, net_list, inp_list, iters=12, flow_init=None, test_mode=False):
        return orig(fmap1.float(), fmap2.float(), [n.float() for n in net_list],
                    [[t.float() for t in level] for level in inp_list], iters, flow_init, test_mode)
    um.forward = forward


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
    env = harness.script_env(patch=True, extra={**ALL_ON, "GPSG_UPDATE": "1"})
    r = subprocess.run([sys.executable, "-c", _COUNTING_RUNNER + harness.SCRIPT_RUNNER, "test_view_interp.py",
                        "--test_data_root", os.path.join(dataset, "val"), "--ckpt_path", ckpt, "--novel_view_nums", "2"],
                       cwd=work, env=env, text=True, capture_output=True, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-6000:]
    line = [ln for ln in r.stdout.splitlines() if ln.startswith("update runs:")][-1]
    forwards, steps = (int(v) for v in line.split(":")[1].split())
    assert forwards >= 2 and steps >= 3 * forwards, line


_COUNTING_RUNNER = ("import atexit\n"
                    "from gps_gaussian_b200 import update\n"
                    "atexit.register(lambda: print('update runs:', update.update_counts()['forwards'],"
                    " update.update_counts()['steps'], flush=True))\n")
