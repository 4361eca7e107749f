"""GPU: the regressor's full-resolution tail (csrc/gs_head.cu through gps_gaussian_b200.gs_head) against the fp64
restatement (oracle/gs_head_torch64.py), per element, within `gs_head_torch64.bounds`, and NaN exactly where fp64 is:
B in {1, 2, 4} at 1024^2, small non-square shapes whose tiles do not divide them (every border row and column is an
element of the check), NaN and inf depth pixels, and the golden cases of the reference's own module.  Every output
buffer is poisoned with NaN before each launch.  The worst error-to-bound ratio per case goes to $GPSG_PARITY_LOG.

Through `make_regresser_forward` on the reference's own GSRegresser: grad disabled -> the kernels; grad enabled -> bit
for bit the original forward; unsupported inputs or modules (CPU, fp16, another head_dim) -> the original.  With the
staged reference: the eval forward of RtStereoHumanModel + pts2render at 1024^2 with GPSG_GS_HEAD on and off, and
test_view_interp.py run unmodified with the switch on."""
import glob
import os
import subprocess
import sys
import types

import pytest
import torch

import gs_head_cases as gc
from helpers import record
from gps_gaussian_b200 import gs_head, harness, patch
from oracle import gs_head_torch64 as gt

pytestmark = pytest.mark.gpu
needs_ref = pytest.mark.skipif(harness.staged_reference() is None, reason="oracle/_ref not staged")
OUTS = ("rot", "scale", "opacity")


@pytest.fixture(autouse=True)
def poisoned_outputs(monkeypatch):
    """torch.empty inside gs_head returns NaN-filled buffers, so an output element the kernels skip shows."""
    def nan(fn):
        def make(*a, **k):
            t = fn(*a, **k)
            if t.is_floating_point():
                t.fill_(float("nan"))
            return t
        return make
    fake = types.SimpleNamespace(**{n: getattr(torch, n) for n in dir(torch) if not n.startswith("__")})
    fake.empty, fake.empty_like = nan(torch.empty), nan(torch.empty_like)
    monkeypatch.setattr(gs_head, "torch", fake)


def _check(tag, src, img, depth, ps, want=None):
    """Kernels on the device; each batch element against its own fp64 truth (the golden outputs when given)."""
    dev = lambda t: t.cuda()
    got = dict(zip(OUTS, gs_head.run(dev(src), dev(img), dev(depth), [dev(p) for p in ps])))
    worst = {k: 0.0 for k in OUTS}
    for n in range(src.shape[0]):
        sl = lambda t: t[n:n + 1].cuda()
        args = (sl(src), sl(img), sl(depth), [dev(p) for p in ps])
        ref = gt.forward64(*args) if want is None else {k: sl(v) for k, v in want.items()}
        b = gt.bounds(*args)
        for k in OUTS:
            worst[k] = max(worst[k], gt.ratio(got[k][n:n + 1], ref[k], b[k]))
    record("gs_head:" + tag, **worst)
    print(f"{tag}: utilisation {worst}")
    assert max(worst.values()) <= 1.0, worst
    return got


@pytest.mark.parametrize("B", [1, 2, 4])
def test_training_size(B):
    case = gc.Case(f"b{B}_1024", B, 1024, 1024, 10 + B)
    _check(case.id, *gc.inputs(case))


SMALL = gc.SWEEP + [gc.Case("one_pixel_pair_2x2", 1, 2, 2, 20), gc.Case("b3_6x130", 3, 6, 130, 21),
                    gc.Case("column_34x2", 1, 34, 2, 22), gc.Case("odd_tiles_50x98", 2, 50, 98, 23),
                    gc.Case("nan_depth_1024x64", 1, 1024, 64, 24, "nan_depth")]


@pytest.mark.parametrize("case", SMALL, ids=lambda c: c.id)
def test_small_shapes(case):
    got = _check(case.id, *gc.inputs(case))
    if case.special in ("nan_depth", "inf_depth"):
        assert all(bool(torch.isnan(got[k]).any()) for k in OUTS)


@pytest.mark.parametrize("name", gc.GOLDEN_CASES)
def test_golden(name):
    src, img, depth, ps, want = gc.golden(name)
    _check("golden_" + name, src, img, depth, ps, want)


# ---- the rebound GSRegresser.forward ------------------------------------------------------------------------------

def _regresser(head_dim=32):
    harness.add_reference_to_path()
    from lib.gs_parm_network import GSRegresser
    cfg = types.SimpleNamespace(raft=types.SimpleNamespace(encoder_dims=[32, 48, 96]),
                                gsnet=types.SimpleNamespace(encoder_dims=[32, 48, 96], decoder_dims=[48, 64, 96],
                                                            parm_head_dim=head_dim))
    torch.manual_seed(3)
    return GSRegresser, GSRegresser(cfg).eval()


def _reg_inputs(B, H, W, device="cuda", dtype=torch.float32):
    g = torch.Generator().manual_seed(B * H + W)
    img = torch.rand(B, 3, H, W, generator=g) * 2 - 1
    depth = torch.rand(B, 1, H, W, generator=g)
    feats = [torch.randn(B, c, H // s, W // s, generator=g) for c, s in ((32, 2), (48, 4), (96, 8))]
    return [t.to(device, dtype) for t in (img, depth)] + [[f.to(device, dtype) for f in feats]]


def test_rebound_forward_grad_disabled_runs_the_kernels(monkeypatch):
    cls, m = _regresser()
    m.cuda()
    fwd = gs_head.make_regresser_forward(cls.forward)
    seen = {}
    run = gs_head.run

    def counted(up_src, *a):
        seen["src"] = up_src.clone()
        return run(up_src, *a)
    monkeypatch.setattr(gs_head, "run", counted)
    img, depth, feats = _reg_inputs(2, 64, 96)
    with torch.no_grad():
        got = fwd(m, img, depth, feats)
        captured = {}
        hook = m.decoder1.register_forward_hook(lambda mod, i, o: captured.setdefault("x", o.clone()))
        try:
            cls.forward(m, img, depth, feats)
        finally:
            hook.remove()
    assert torch.equal(seen["src"], captured["x"])               # the module's own decoders, bit for bit
    args = (captured["x"], img, depth, [p.detach() for p in gs_head.params_of(m)])
    ref, b = gt.forward64(*args), gt.bounds(*args)
    worst = {k: gt.ratio(g, ref[k], b[k]) for k, g in zip(OUTS, got)}
    record("gs_head:rebound_no_grad", **worst)
    assert max(worst.values()) <= 1.0, worst


def test_rebound_forward_grad_enabled_is_the_original(monkeypatch):
    cls, m = _regresser()
    m.cuda()
    fwd = gs_head.make_regresser_forward(cls.forward)
    monkeypatch.setattr(gs_head, "run", lambda *a: pytest.fail("the kernels ran with grad enabled"))
    img, depth, feats = _reg_inputs(1, 32, 48)
    torch.manual_seed(0)
    got = fwd(m, img, depth, feats)
    want = cls.forward(m, img, depth, feats)
    for g, w in zip(got, want):
        assert g.requires_grad and torch.equal(g, w)


@pytest.mark.parametrize("what", ["cpu", "fp16", "head_dim_16"])
def test_rebound_forward_unsupported_is_the_original(what, monkeypatch):
    cls, m = _regresser(16 if what == "head_dim_16" else 32)
    device, dtype = ("cpu", torch.float32) if what == "cpu" else ("cuda", torch.float16 if what == "fp16" else torch.float32)
    m.to(device, dtype)
    fwd = gs_head.make_regresser_forward(cls.forward)
    monkeypatch.setattr(gs_head, "run", lambda *a: pytest.fail("the kernels ran on unsupported inputs"))
    img, depth, feats = _reg_inputs(1, 32, 48, device, dtype)
    with torch.no_grad():
        got = fwd(m, img, depth, feats)
        want = cls.forward(m, img, depth, feats)
    for g, w in zip(got, want):
        assert torch.equal(g, w)


# ---- the reference's model and scripts with the switch --------------------------------------------------------------

@pytest.fixture(scope="module")
def dataset_1024(tmp_path_factory):
    from gps_gaussian_b200 import synth_dataset
    root = str(tmp_path_factory.mktemp("gsheaddata"))
    synth_dataset.write_dataset(root, n_train=1, n_val=1, res=1024, hr=True)
    return root


def _install(on, monkeypatch):
    patch.uninstall()
    if on:
        monkeypatch.setenv("GPSG_GS_HEAD", "1")
    else:
        monkeypatch.delenv("GPSG_GS_HEAD", raising=False)
    harness.add_reference_to_path()
    patch.install()
    import lib.gs_parm_network
    assert (lib.gs_parm_network.GSRegresser.forward.__module__ == gs_head.__name__) is on


@needs_ref
def test_eval_forward_and_render_switch_on_off(dataset_1024, monkeypatch):
    ran = {"n": 0}
    run = gs_head.run

    def counted(*a):
        ran["n"] += 1
        return run(*a)
    monkeypatch.setattr(gs_head, "run", counted)
    imgs = {}
    try:
        for on, tf32 in ((False, True), (False, False), (True, True)):
            _install(on, monkeypatch)
            monkeypatch.setattr(torch.backends.cudnn, "allow_tf32", tf32)
            from lib.GaussianRender import pts2render
            cfg = harness.load_cfg(dataset_1024, src_res=1024, batch_size=1)
            st = harness.C3State(cfg)
            st.model.eval()
            data = st.batch(0)
            with torch.no_grad():
                out, _, _ = st.model({k: dict(v) if isinstance(v, dict) else v for k, v in data.items()}, is_train=False)
                out = pts2render(out, bg_color=cfg.dataset.bg_color)
            imgs[(on, tf32)] = out["novel_view"]["img_pred"].float()
            del st, out, data
            torch.cuda.empty_cache()
    finally:
        patch.uninstall()
    assert ran["n"] == 1                                             # the switched-on forward ran the kernels once
    d_switch = float((imgs[(True, True)] - imgs[(False, True)]).abs().mean())
    d_tf32 = float((imgs[(False, False)] - imgs[(False, True)]).abs().mean())
    m_switch = float((imgs[(True, True)] - imgs[(False, True)]).abs().max())
    m_tf32 = float((imgs[(False, False)] - imgs[(False, True)]).abs().max())
    record("gs_head:render_switch", mean_switch=d_switch, mean_tf32=d_tf32, max_switch=m_switch, max_tf32=m_tf32)
    print(f"render: switch on vs off mean |d| {d_switch:.3e} (max {m_switch:.3e}); cuDNN TF32 on vs off mean |d| "
          f"{d_tf32:.3e} (max {m_tf32:.3e})")
    assert d_switch <= 2 * d_tf32


@needs_ref
def test_view_interp_runs_unmodified_with_gs_head(tmp_path, monkeypatch):
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
    # the script runs unmodified; the runner only counts the kernel launches of the rebound forward and prints the count
    r = subprocess.run([sys.executable, "-c", _COUNTING_RUNNER + harness.SCRIPT_RUNNER, "test_view_interp.py",
                        "--test_data_root", os.path.join(dataset, "val"), "--ckpt_path", ckpt, "--novel_view_nums", "2"],
                       cwd=work, env=harness.script_env(patch=True, extra={"GPSG_GS_HEAD": "1"}), text=True,
                       capture_output=True, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-6000:]
    assert len(glob.glob(os.path.join(work, "interp_out", "*.jpg"))) == 2 * 2          # 2 val samples x 2 novel views
    assert "gs_head runs: 4" in r.stdout, r.stdout[-3000:]                            # one regressor call per view


_COUNTING_RUNNER = ("import atexit\n"
                    "from gps_gaussian_b200 import gs_head\n"
                    "_runs, _run = [0], gs_head.run\n"
                    "def _counted(*a):\n"
                    "    _runs[0] += 1\n"
                    "    return _run(*a)\n"
                    "gs_head.run = _counted\n"
                    "atexit.register(lambda: print('gs_head runs:', _runs[0], flush=True))\n")
