"""GPU: the backward of the regressor's full-resolution tail (csrc/gs_head.cu through gps_gaussian_b200.gs_head).

- Per element against fp64 autograd on the kernels' own intermediate (oracle/gs_head_grad_torch64.backward64 with `mid`),
  within `grad_bounds`, NaN and inf exactly where fp64 has them, and d_src against the fp64 upsample adjoint of the
  kernels' own dcat (`src_stage`), every output and workspace buffer poisoned with NaN:
  B in {1, 2, 4} at 1024^2, the forward tests' small shapes, and the golden cases of the reference's own autograd.
- Per tensor against cuDNN: each gradient's relative L2 error against fp64 is at most twice that of the same chain in
  torch ops with cuDNN's TF32 convolutions.
- Bit-reproducible: two backward calls agree bit for bit.
- Non-finite upstream gradients: non-finite exactly where the golden is; a GradScaler step on them is skipped.
- The reference's stage-2 step (harness.c3_step) with GPSG_GS_HEAD_TRAIN on and off, and train_stage2.py run unmodified
  with the switch, counting the backward calls."""
import glob
import os
import subprocess
import sys
import types

import pytest
import torch
from torch import nn

import gs_head_cases as gc
import gs_head_grad_cases as gg
from helpers import record
from gps_gaussian_b200 import gs_head, harness, patch
from oracle import gs_head_grad_torch64 as gt

pytestmark = pytest.mark.gpu
needs_ref = pytest.mark.skipif(harness.staged_reference() is None, reason="oracle/_ref not staged")
KEYS = gg.GRAD_KEYS
FP32_FLOOR = 8 * 2.0 ** -24


@pytest.fixture
def poisoned(monkeypatch):
    """torch.empty inside gs_head returns NaN-filled buffers (outputs, the forward's and the backward's workspaces)."""
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


def _kernels(src, img, depth, ps, grads, dcat=False):
    """(dict of the 16 gradients, mid NCHW) from the kernels, all on the device; with `dcat`, also dcat[:, :48] NCHW,
    which the backward leaves in its (NaN-poisoned) workspace."""
    B, _, H, W = img.shape
    rot, scale, opacity, ws = gs_head.forward_with_mid(src, img, depth, ps)
    bws = gs_head.torch.empty(int(gs_head._lib.lib.gpsg_gs_head_backward_workspace_bytes(B, H, W)) // 4,
                              dtype=torch.float32, device=src.device)
    d_src, d_depth, pg = gs_head.backward(src, img, depth, ps, ws, *grads, workspace=bws)
    mid = ws[:B * H * W * 32].view(B, H, W, 32).permute(0, 3, 1, 2)
    got = dict(zip(KEYS, [d_src, d_depth] + pg))
    if dcat:
        return got, mid, bws[:B * H * W * 48].view(B, H, W, 48).permute(0, 3, 1, 2)
    return got, mid


def _check(tag, src, img, depth, ps, grads):
    dev = lambda t: t.cuda()
    args = (dev(src), dev(img), dev(depth), [dev(p) for p in ps], [dev(g) for g in grads])
    got, mid, dcat = _kernels(*args, dcat=True)
    want = gt.backward64(*args, mid=mid)
    bnd = gt.grad_bounds(*args, mid, ctas=torch.cuda.get_device_properties(0).multi_processor_count)
    worst = {k: gt.ratio(got[k], want[k], bnd[k]) for k in KEYS}
    worst["d_src_stage"] = gt.ratio(got["d_src"], *gt.src_stage(dcat))       # the upsample adjoint on its own input
    record("gs_head_grad:" + tag, **worst)
    print(f"{tag}: utilisation {worst}")
    assert max(worst.values()) <= 1.0, worst
    return got


@pytest.mark.parametrize("B", [1, 2, 4])
def test_training_size(B, poisoned):
    case = gc.Case(f"train_b{B}", B, 1024, 1024, 40 + B)
    src, img, depth, ps = gc.inputs(case)
    _check(case.id, src, img, depth, ps, gg.upstream(B, 1024, 1024, case.seed))


@pytest.mark.parametrize("case", gc.SWEEP, ids=lambda c: c.id)
def test_small_shapes(case, poisoned):
    src, img, depth, ps = gc.inputs(case)
    _check(case.id, src, img, depth, ps, gg.upstream(case.B, case.H, case.W, case.seed))


@pytest.mark.parametrize("name", gg.GOLDEN_CASES)
def test_golden(name, poisoned):
    src, img, depth, ps, grads = gg.golden(name)[:5]
    _check("golden_" + name, src, img, depth, ps, grads)


def _rel(got, want):
    return float((got.double() - want).norm() / want.norm())


def test_relative_error_against_cudnn_tf32():
    """Each gradient's relative L2 error against fp64 <= 2x that of cuDNN's TF32 backward of the same chain.  A bias
    gradient with no TF32 operand in its chain can be accurate to a few fp32 ulps in both, where the comparison is a coin
    toss: errors are measured against at least 8 u (u = 2^-24) relative."""
    assert torch.backends.cudnn.allow_tf32
    case = gc.Case("cudnn", 2, 512, 512, 77)
    src, img, depth, ps = gc.inputs(case)
    src, img, depth, ps = src.cuda(), img.cuda(), depth.cuda(), [p.cuda() for p in ps]
    grads = [g.cuda() for g in gg.upstream(2, 512, 512, 77)]
    want = gt.backward64(src, img, depth, ps, grads)
    got, _ = _kernels(src, img, depth, ps, grads)
    # the same chain in torch ops: cuDNN convolutions in TF32, fp32 elsewhere
    s = src.clone().requires_grad_()
    d = depth.clone().requires_grad_()
    q = [p.clone().requires_grad_() for p in ps]
    x = torch.cat([nn.functional.interpolate(s, scale_factor=2, mode="bilinear"), img, d], 1)
    m = torch.relu(nn.functional.conv2d(x, q[0], q[1], padding=1))
    pre = [nn.functional.conv2d(torch.relu(nn.functional.conv2d(m, q[2 + 4 * k], q[3 + 4 * k], padding=1)),
                                q[4 + 4 * k], q[5 + 4 * k]) for k in range(3)]
    outs = (nn.functional.normalize(pre[0], dim=1),
            torch.clamp_max(nn.functional.softplus(pre[1], beta=100, threshold=20), 0.01), torch.sigmoid(pre[2]))
    torch.autograd.backward(outs, grads)
    ref = dict(zip(KEYS, [s.grad, d.grad] + [p.grad for p in q]))
    ratios = {}
    for k in KEYS:
        ek, ec = _rel(got[k], want[k]), _rel(ref[k], want[k])
        ratios[k] = max(ek, FP32_FLOOR) / max(ec, FP32_FLOOR)
        print(f"{k}: kernels {ek:.3e}, cuDNN TF32 {ec:.3e}")
    record("gs_head_grad:vs_cudnn", **ratios)
    assert max(ratios.values()) <= 2.0, ratios


def test_bit_reproducible():
    case = gc.Case("repro", 2, 256, 320, 9)
    src, img, depth, ps = gc.inputs(case)
    src, img, depth, ps = src.cuda(), img.cuda(), depth.cuda(), [p.cuda() for p in ps]
    grads = [g.cuda() for g in gg.upstream(2, 256, 320, 9)]
    a, _ = _kernels(src, img, depth, ps, grads)
    b, _ = _kernels(src, img, depth, ps, grads)
    for k in KEYS:
        assert torch.equal(a[k], b[k]), k


class _TailModule(nn.Module):
    """The regressor's tail layers with the reference's names and types, for gs_head_train."""
    def __init__(self):
        super().__init__()
        self.decoder_dims, self.head_dim = [48, 64, 96], 32
        self.up = nn.Upsample(scale_factor=2, mode="bilinear")
        self.out_conv = nn.Conv2d(52, 32, 3, padding=1)
        self.out_relu = nn.ReLU(inplace=True)
        self.rot_head = nn.Sequential(nn.Conv2d(32, 32, 3, padding=1), nn.ReLU(inplace=True), nn.Conv2d(32, 4, 1))
        self.scale_head = nn.Sequential(nn.Conv2d(32, 32, 3, padding=1), nn.ReLU(inplace=True), nn.Conv2d(32, 3, 1),
                                        nn.Softplus(beta=100))
        self.opacity_head = nn.Sequential(nn.Conv2d(32, 32, 3, padding=1), nn.ReLU(inplace=True), nn.Conv2d(32, 1, 1),
                                          nn.Sigmoid())

    def forward(self, src, img, depth):
        out = self.out_relu(self.out_conv(torch.cat([self.up(src), img, depth], 1)))
        return (nn.functional.normalize(self.rot_head(out), dim=1), torch.clamp_max(self.scale_head(out), 0.01),
                self.opacity_head(out))


def test_nonfinite_upstream_gradient():
    src, img, depth, ps, grads, _, finite, _ = gg.golden("inf_g_scale")
    got, _ = _kernels(src.cuda(), img.cuda(), depth.cuda(), [p.cuda() for p in ps], [g.cuda() for g in grads])
    for k in KEYS:
        assert torch.equal(torch.isfinite(got[k]).cpu(), finite[k]), k
    assert not all(bool(torch.isfinite(got[k]).all()) for k in KEYS[2:])
    # a GradScaler step on these gradients is skipped, with the kernels as with the torch chain
    for on in (False, True):
        torch.manual_seed(3)
        mod = _TailModule().cuda()
        before = [p.detach().clone() for p in mod.parameters()]
        opt = torch.optim.SGD(mod.parameters(), lr=0.1)
        scaler = torch.amp.GradScaler("cuda", init_scale=1024.0)
        s = src.cuda().requires_grad_()
        outs = gs_head.gs_head_train(s, img.cuda(), depth.cuda(), mod) if on else mod(s, img.cuda(), depth.cuda())
        loss = sum((o * g.cuda()).sum() for o, g in zip(outs, grads))
        scaler.scale(loss).backward()
        scaler.step(opt)
        scaler.update()
        assert scaler.get_scale() < 1024.0, on
        assert all(torch.equal(a, b) for a, b in zip(before, mod.parameters())), on


# ---- the reference's training step and script with the switch -------------------------------------------------------

@pytest.fixture(scope="module")
def dataset_512(tmp_path_factory):
    from gps_gaussian_b200 import synth_dataset
    root = str(tmp_path_factory.mktemp("gsheadtrain"))
    synth_dataset.write_dataset(root, n_train=2, n_val=1, res=512, hr=True)
    return root


def _install(on, monkeypatch):
    patch.uninstall()
    monkeypatch.delenv("GPSG_GS_HEAD", raising=False)
    if on:
        monkeypatch.setenv("GPSG_GS_HEAD_TRAIN", "1")
    else:
        monkeypatch.delenv("GPSG_GS_HEAD_TRAIN", raising=False)
    harness.add_reference_to_path()
    patch.install()
    import lib.gs_parm_network
    assert (lib.gs_parm_network.GSRegresser.forward.__module__ == gs_head.__name__) is on
    assert patch.gs_head_train() is on


@needs_ref
def test_stage2_step_switch_on_off(dataset_512, monkeypatch):
    res = {}
    try:
        for on in (False, True):
            _install(on, monkeypatch)
            gs_head.reset_counts()
            cfg = harness.load_cfg(dataset_512, src_res=512, num_steps=3, batch_size=2)
            st = harness.C3State(cfg)
            out = harness.c3_step(st, st.batch(0))
            reg = st.model.gs_parm_regresser
            tail = [p for n, p in reg.named_parameters() if n.split(".")[0] in
                    ("out_conv", "rot_head", "scale_head", "opacity_head")]
            cat = lambda ps: torch.cat([p.grad.reshape(-1) for p in ps if p.grad is not None]).double()
            res[on] = (float(out["loss"]), cat(st.model.parameters()), cat(tail),
                       out["scale_after"] >= out["scale_before"])
            assert gs_head.counts()["backward"] == (1 if on else 0)
            del st, out
            torch.cuda.empty_cache()
    finally:
        patch.uninstall()
    (la, ga, ta, oka), (lb, gb, tb, okb) = res[False], res[True]
    cos = lambda a, b: float((a * b).sum() / (a.norm() * b.norm()))
    print(f"stage 2 step: loss {la:.6f} vs {lb:.6f}; model grad cosine {cos(ga, gb):.6f}, tail {cos(ta, tb):.6f}")
    record("gs_head_grad:stage2_step", loss_off=la, loss_on=lb, cos_model=cos(ga, gb), cos_tail=cos(ta, tb))
    assert oka and okb
    assert abs(la - lb) < 2e-3 * max(1.0, abs(la))
    assert cos(ta, tb) > 0.999
    assert cos(ga, gb) > 0.99


_COUNTING_RUNNER = ("import atexit\n"
                    "from gps_gaussian_b200 import gs_head\n"
                    "atexit.register(lambda: print('gs_head backward calls:', gs_head.counts()['backward'], flush=True))\n")


@needs_ref
def test_train_stage2_runs_unmodified_with_gs_head_train(dataset_512, tmp_path):
    work = harness.make_workdir(str(tmp_path / "work"), dataset_512, src_res=512, num_steps=3, batch_size=2)
    r = subprocess.run([sys.executable, "-c", _COUNTING_RUNNER + harness.SCRIPT_RUNNER, "train_stage2.py"],
                       cwd=work, env=harness.script_env(patch=True, extra={"GPSG_GS_HEAD_TRAIN": "1"}), text=True,
                       capture_output=True, timeout=1500)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-6000:]
    assert "FINISHED TRAINING" in r.stdout
    assert "gs_head backward calls: 3" in r.stdout, r.stdout[-3000:]
    ckpts = glob.glob(os.path.join(work, "experiments", "*", "ckpt", "*_final.pth"))
    assert len(ckpts) == 1
    sd = torch.load(ckpts[0], map_location="cpu")
    assert all(bool(torch.isfinite(v).all()) for v in sd["network"].values() if v.is_floating_point())
