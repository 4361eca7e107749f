"""The disparity head on hardware (csrc/flow_head.cu through gps_gaussian_b200.flow_head): the golden cases, the oracle at
the stage-1 and stage-2 shapes, determinism, no host synchronisation, CUDA-graph replay, the sequence loss against the
reference's own function on the same device tensors, and both training stages with GPSG_FLOW_HEAD on and off.  Every
output buffer is poisoned with NaN before each launch."""
import contextlib
import glob
import math
import os
import types
import warnings

import numpy as np
import pytest
import torch

from gps_gaussian_b200 import flow_head, harness, patch
from oracle import flow_head_oracle as fo

pytestmark = pytest.mark.gpu
needs_ref = pytest.mark.skipif(harness.staged_reference() is None, reason="oracle/_ref not staged")
GOLDEN = np.load(os.path.join(os.path.dirname(__file__), "golden", "flow_head_golden.npz"))
UP = sorted({k[3:-len("_factor")] for k in GOLDEN.files if k.startswith("up_") and k.endswith("_factor")})
SL = sorted({k[3:-len("_raises")] for k in GOLDEN.files if k.startswith("sl_") and k.endswith("_raises")})


@pytest.fixture(autouse=True)
def poisoned_outputs(monkeypatch):
    """torch.empty / empty_like inside flow_head return NaN-filled buffers, so an output element the kernels skip shows."""
    def nan(fn):
        def make(*a, **k):
            t = fn(*a, **k)
            if t.is_floating_point():
                t.fill_(float("nan"))
            return t
        return make
    fake = types.SimpleNamespace(**{n: getattr(torch, n) for n in dir(torch) if not n.startswith("__")})
    fake.empty, fake.empty_like = nan(torch.empty), nan(torch.empty_like)
    monkeypatch.setattr(flow_head, "torch", fake)


def _up_inputs(name, dev="cuda"):
    g = lambda k: GOLDEN[f"up_{name}_{k}"]
    mdt = torch.float16 if g("mask").dtype == np.float16 else torch.float32
    flow = torch.tensor(g("flow"), dtype=torch.float32, device=dev, requires_grad=True)
    mask = torch.tensor(g("mask"), dtype=mdt, device=dev, requires_grad=True)
    return int(g("factor")), flow, mask, torch.tensor(g("g"), dtype=torch.float32, device=dev)


def _close(got, want, rel, what):
    got, want = got.astype(np.float64), want.astype(np.float64)
    nan = np.isnan(want)
    assert np.array_equal(np.isnan(got), nan), (what, "NaN positions differ")
    if (~nan).any():
        scale = max(1.0, float(np.abs(want[~nan]).max()))
        err = float(np.abs(got[~nan] - want[~nan]).max())
        assert err <= rel * scale, (what, err, rel * scale)


# fp64 goldens run with fp32 inputs: rounding the logits to fp32 moves each weight by |m| * 2^-24 relative, |m| < 16 here,
# so 2^-17 (as for the fp32 goldens, see test_flow_head_cpu.py) still holds with margin.  fp16 masks: 9 fp16 ulps.
BOUND = {"f64": 2.0 ** -16, "f32": 2.0 ** -17, "f16": 9 * 2.0 ** -11}


@pytest.mark.parametrize("name", UP)
def test_golden_upsample(name):
    f, flow, mask, g = _up_inputs(name)
    kind = name.rsplit("_", 1)[1]
    out = flow_head.convex_upsample(flow, mask, f)
    assert out.dtype == torch.float32
    _close(out.detach().cpu().numpy(), GOLDEN[f"up_{name}_out"], BOUND[kind], "out")
    (out * g).sum().backward()
    assert mask.grad.dtype == mask.dtype and flow.grad.dtype == torch.float32
    _close(flow.grad.cpu().numpy(), GOLDEN[f"up_{name}_d_flow"], BOUND[kind], "d_flow")
    _close(mask.grad.float().cpu().numpy(), GOLDEN[f"up_{name}_d_mask"], BOUND[kind], "d_mask")


def _stage_inputs(stage, seed=0):
    gen = torch.Generator(device="cuda").manual_seed(seed)
    N, mdt = (12, torch.float32) if stage == 1 else (4, torch.float16)
    H = W = 128
    flow = torch.randn(N, 2, H, W, device="cuda", generator=gen) * 8.0
    flow[:, 1] = 0.0                                        # the stereo head's y flow (delta_flow[:, 1] = 0)
    mask = (torch.randn(N, 9 * 64, H, W, device="cuda", generator=gen) * 4.0).to(mdt)
    g = torch.zeros(N, 2, 8 * H, 8 * W, device="cuda")
    g[:, 0] = torch.randn(N, 8 * H, 8 * W, device="cuda", generator=gen)      # the caller keeps channel 0
    return flow, mask, g


def _run(flow, mask, g, fn=None):
    fl, m = flow.detach().clone().requires_grad_(), mask.detach().clone().requires_grad_()
    out = (fn or (lambda a, b: flow_head.convex_upsample(a, b, 8)))(fl, m)
    out.backward(g)
    return out.detach(), fl.grad, m.grad


@pytest.mark.parametrize("stage", [1, 2])
def test_stage_shapes_against_oracle_and_op_chain(stage):
    flow, mask, g = _stage_inputs(stage)
    out, dflow, dmask = _run(flow, mask, g)
    dt = np.float16 if stage == 2 else np.float32
    for n in (0, flow.shape[0] - 1):                        # pixels are independent across the batch
        fl, m, gg = flow[n:n + 1].cpu().numpy(), mask[n:n + 1].cpu().numpy(), g[n:n + 1].cpu().numpy()
        bound = BOUND["f16" if stage == 2 else "f32"]
        _close(out[n:n + 1].cpu().numpy(), fo.convex_upsample(fl, m, 8, dt), bound, "out")
        want_dflow, want_dmask = fo.convex_upsample_backward(fl, m, 8, gg, dt)
        _close(dflow[n:n + 1].cpu().numpy(), want_dflow, bound, "d_flow")
        _close(dmask[n:n + 1].float().cpu().numpy(), want_dmask.astype(np.float32), bound, "d_mask")
        if stage == 2:
            # The oracle rounds at the same points (weights and dL/dweight to fp16) and adds in the same order, so the
            # output and dL/dmask agree bit for bit except where CUDA's expf and numpy's exp differ by an fp32 ulp
            # next to an fp16 rounding boundary.  Leaving out either rounding would change most elements.
            for got, want, what in ((out[n:n + 1].cpu().numpy(), fo.convex_upsample(fl, m, 8, dt), "out"),
                                    (dmask[n:n + 1].cpu().numpy(), want_dmask, "d_mask")):
                same = float(np.mean((got == want) | (np.isnan(got) & np.isnan(want))))
                print(f"stage 2, n={n}: {what} bit-identical to the fp16-boundary oracle: {same:.5f}")
                assert same >= 0.98, (what, same)
    if harness.staged_reference() is None:
        print(f"stage {stage}: oracle bounds hold; oracle/_ref not staged, no op-chain comparison")
        return
    harness.add_reference_to_path()
    from core.raft_stereo_human import FlowUpdateModule
    me = types.SimpleNamespace(args=types.SimpleNamespace(n_downsample=3))
    ref = _run(flow, mask, g, lambda a, b: FlowUpdateModule.upsample_flow(me, a, b))
    same = [float((_bits(a) == _bits(b)).float().mean()) for a, b in zip((out, dflow, dmask), ref)]
    print(f"stage {stage}: bit-identical to the op chain: out {same[0]:.4f}, d_flow {same[1]:.4f}, d_mask {same[2]:.4f}")


def _bits(t):
    return t.view(torch.int16 if t.dtype == torch.float16 else torch.int32)


def test_reruns_bit_identical_and_deterministic_mode():
    flow, mask, g = _stage_inputs(2, seed=1)
    a = _run(flow, mask, g)
    b = _run(flow, mask, g)
    torch.use_deterministic_algorithms(True)
    try:
        c = _run(flow, mask, g)
    finally:
        torch.use_deterministic_algorithms(False)
    for x, y, z in zip(a, b, c):
        assert torch.equal(_bits(x), _bits(y)) and torch.equal(_bits(x), _bits(z))


def test_upsample_no_sync_and_cuda_graph():
    flow, mask, g = _stage_inputs(1, seed=2)
    flow, mask, g = flow[:2].contiguous(), mask[:2].contiguous(), g[:2].contiguous()
    want = _run(flow, mask, g)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        _run(flow, mask, g)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    fl, m = flow.detach().clone().requires_grad_(), mask.detach().clone().requires_grad_()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):                               # warm-up on the capture stream
        flow_head.convex_upsample(fl, m, 8).backward(g)
    torch.cuda.current_stream().wait_stream(s)
    fl.grad, m.grad = None, None
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = flow_head.convex_upsample(fl, m, 8)
        out.backward(g)
    graph.replay()
    torch.cuda.synchronize()
    for x, y in zip((out, fl.grad, m.grad), want):
        assert torch.equal(x, y)


# ---- sequence loss ----------------------------------------------------------------------------------------------------

def _reference_loss():
    harness.add_reference_to_path()
    import lib.loss
    return patch.original(lib.loss, "sequence_loss")


@contextlib.contextmanager
def _count_syncs():
    rec = []
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("warn")
    try:
        with warnings.catch_warnings(record=True) as w:
            warnings.simplefilter("always")
            yield rec
    finally:
        torch.cuda.set_sync_debug_mode("default")
    rec.extend(x for x in w if "synchroniz" in str(x.message))


def _sl_inputs(P=3, N=4, H=256, W=256, seed=3, empty=False, gt_dtype=torch.float32):
    """gt_dtype fp16 is what training passes: the loader's cache stores the flow in fp16 (lib/human_loader.py:157-159)."""
    gen = torch.Generator(device="cuda").manual_seed(seed)
    gt = (torch.rand(N, 1, H, W, device="cuda", generator=gen) * -40).to(gt_dtype)
    valid = torch.rand(N, 1, H, W, device="cuda", generator=gen)
    if empty:
        valid.fill_(0.25)
    gt[valid < 0.5] = float("inf")                                            # inf outside the valid set is allowed
    finite = gt.float().nan_to_num(posinf=0.0)
    preds = [(finite + torch.randn(N, 1, H, W, device="cuda", generator=gen) * 3 / (i + 1)) for i in range(P)]
    preds[-1].view(-1)[::7] = finite.view(-1)[::7]                             # ties: sign(0) = 0
    return [p.requires_grad_() for p in preds], gt, valid


@needs_ref
@pytest.mark.parametrize("gt_dtype", [torch.float32, torch.float16])
@pytest.mark.parametrize("P", [2, 3])
def test_sequence_loss_against_reference(P, gt_dtype):
    ref_fn = _reference_loss()
    preds, gt, valid = _sl_inputs(P, gt_dtype=gt_dtype)
    with _count_syncs() as syncs:
        loss, metrics = flow_head.sequence_loss(preds, gt, valid)
    assert len(syncs) == 1, [str(s.message) for s in syncs]
    g = torch.tensor(1.7, device="cuda")
    torch.autograd.backward(loss, g)
    ours = [p.grad.clone() for p in preds]
    for p in preds:
        p.grad = None
    ref_loss, ref_metrics = ref_fn(preds, gt, valid)
    torch.autograd.backward(ref_loss, g)
    assert loss.dtype == torch.float32 and loss.dim() == 0
    # the loss and the EPE mean re-associate an fp32 sum of up to 2.6e5 terms (torch's tree vs our fixed-order fp64
    # partials): within 1e-5 relative; the threshold fractions are exact counts times the same fp32 reciprocal
    print(f"P={P} gt {gt_dtype}: loss {float(loss):.8f} vs {float(ref_loss):.8f}; metrics {metrics} vs {ref_metrics}")
    assert abs(float(loss) - float(ref_loss)) <= 1e-5 * abs(float(ref_loss))
    assert abs(metrics["train_epe"] - ref_metrics["train_epe"]) <= 1e-5 * abs(ref_metrics["train_epe"])
    assert metrics["train_1px"] == ref_metrics["train_1px"] and metrics["train_3px"] == ref_metrics["train_3px"]
    assert all(type(v) is float for v in metrics.values())
    for a, p in zip(ours, preds):
        assert torch.equal(a.view(torch.int32), p.grad.view(torch.int32))              # bit-identical, signed zeros too


@needs_ref
def test_sequence_loss_nan_and_assertion_cases():
    ref_fn = _reference_loss()
    preds, gt, valid = _sl_inputs(3, N=1, H=32, W=32, empty=True)
    loss, metrics = flow_head.sequence_loss(preds, gt, valid)
    ref_loss, ref_metrics = ref_fn(preds, gt, valid)
    assert math.isnan(float(loss)) and math.isnan(float(ref_loss))
    assert all(math.isnan(metrics[k]) and math.isnan(ref_metrics[k]) for k in metrics)
    loss.backward()
    assert all(not p.grad.any() for p in preds)
    preds, gt, valid = _sl_inputs(2, N=1, H=32, W=32, gt_dtype=torch.float16)
    for fn in (flow_head.sequence_loss, ref_fn):
        with pytest.raises(ZeroDivisionError):
            fn(preds[:1], gt, valid)
    gt.view(-1)[int(torch.nonzero(valid.view(-1) >= 0.5)[0])] = -float("inf")
    for fn in (flow_head.sequence_loss, ref_fn):
        with pytest.raises(AssertionError):
            fn(preds, gt, valid)


@pytest.mark.parametrize("name", SL)
def test_golden_sequence_loss(name):
    sl = lambda k: GOLDEN[f"sl_{name}_{k}"]
    raises = str(sl("raises"))
    preds = [torch.tensor(p, device="cuda", requires_grad=True) for p in sl("preds")]
    gt, valid = torch.tensor(sl("gt"), device="cuda"), torch.tensor(sl("valid"), device="cuda")
    if raises:
        with pytest.raises({"AssertionError": AssertionError, "ZeroDivisionError": ZeroDivisionError}[raises]):
            flow_head.sequence_loss(preds, gt, valid)
        return
    loss, metrics = flow_head.sequence_loss(preds, gt, valid)
    (loss * float(sl("g"))).backward()
    want = float(sl("loss_f32"))
    m = np.array([metrics["train_epe"], metrics["train_1px"], metrics["train_3px"]])
    if math.isnan(want):
        assert math.isnan(float(loss)) and np.isnan(m).all()
    else:
        assert abs(float(loss) - want) <= 1e-6 * abs(want)
        assert np.allclose(m, sl("metrics_f32"), rtol=1e-6, atol=0)
    # the CPU reference divides by the count where CUDA multiplies by its reciprocal: one ulp apart at most
    got = np.stack([p.grad.cpu().numpy() for p in preds])
    assert np.allclose(got, sl("grads_f32"), rtol=2.0 ** -22, atol=0)


# ---- both training stages with the switch on and off --------------------------------------------------------------

@pytest.fixture(scope="module")
def dataset(tmp_path_factory):
    from gps_gaussian_b200 import synth_dataset
    root = str(tmp_path_factory.mktemp("flowheaddata"))
    synth_dataset.write_dataset(root, n_train=2, n_val=2, res=256, hr=True)
    return root


def _with_switch(on, monkeypatch, body):
    """body() with GPSG_FLOW_HEAD on or off, and how often the fused Functions ran inside it: the loss's flow_gt dtypes
    and the number of upsamplings.  The rebound names alone do not show it; unsupported inputs would fall back."""
    ran = {"loss_gt": [], "upsample": 0}
    sl_apply, up_apply = flow_head._SequenceLoss.apply, flow_head._ConvexUpsample.apply

    def counted_loss(gt, *a):
        ran["loss_gt"].append(gt.dtype)
        return sl_apply(gt, *a)

    def counted_upsample(*a):
        ran["upsample"] += 1
        return up_apply(*a)
    monkeypatch.setattr(flow_head._SequenceLoss, "apply", staticmethod(counted_loss))
    monkeypatch.setattr(flow_head._ConvexUpsample, "apply", staticmethod(counted_upsample))
    patch.uninstall()
    if on:
        monkeypatch.setenv("GPSG_FLOW_HEAD", "1")
    else:
        monkeypatch.delenv("GPSG_FLOW_HEAD", raising=False)
    harness.add_reference_to_path()
    patch.install()
    try:
        import core.raft_stereo_human, lib.network
        assert (lib.network.sequence_loss is flow_head.sequence_loss) is on
        assert (core.raft_stereo_human.FlowUpdateModule.upsample_flow.__module__ == flow_head.__name__) is on
        return body(), ran
    finally:
        patch.uninstall()
        monkeypatch.delenv("GPSG_FLOW_HEAD", raising=False)


def _grads(model):
    return torch.cat([p.grad.reshape(-1) for p in model.parameters() if p.grad is not None]).double()


@needs_ref
def test_stage1_step_switch_on_off(dataset, monkeypatch):
    monkeypatch.setattr(torch.backends.cudnn, "allow_tf32", False)
    monkeypatch.setattr(torch.backends.cuda.matmul, "allow_tf32", False)
    res = {}
    for on in (False, True):
        def body():
            cfg = harness.load_cfg(dataset, stage=1, src_res=256, num_steps=3, batch_size=2)
            st = harness.Stage1State(cfg)
            out = harness.stage1_step(st, st.batch(0))
            return float(out["flow_loss"]), _grads(st.model), out["metrics"]
        res[on], ran = _with_switch(on, monkeypatch, body)
        iters = harness.load_cfg(dataset, stage=1, src_res=256).raft.train_iters
        assert (len(ran["loss_gt"]), ran["upsample"]) == ((1, iters) if on else (0, 0)), ran
    (la, ga, ma), (lb, gb, mb) = res[False], res[True]
    cos = float((ga * gb).sum() / (ga.norm() * gb.norm()))
    print(f"stage 1: fused loss on flow_gt {ran['loss_gt']}, {ran['upsample']} fused upsamplings; flow_loss {la:.7f} vs "
          f"{lb:.7f}; grad cosine {cos:.7f}; metrics {ma} vs {mb}")
    assert abs(la - lb) <= 1e-5 * abs(la)
    assert cos > 0.999


@needs_ref
def test_stage2_step_switch_on_off(dataset, monkeypatch):
    res = {}
    for on in (False, True):
        def body():
            cfg = harness.load_cfg(dataset, src_res=256, num_steps=3, batch_size=2)
            st = harness.C3State(cfg)
            out = harness.c3_step(st, st.batch(0))
            return float(out["loss"]), _grads(st.model), out["scale_after"] >= out["scale_before"]
        res[on], ran = _with_switch(on, monkeypatch, body)
        iters = harness.load_cfg(dataset, src_res=256).raft.train_iters
        assert (len(ran["loss_gt"]), ran["upsample"]) == ((1, iters) if on else (0, 0)), ran
    (la, ga, oka), (lb, gb, okb) = res[False], res[True]
    cos = float((ga * gb).sum() / (ga.norm() * gb.norm()))
    print(f"stage 2: fused loss on flow_gt {ran['loss_gt']}, {ran['upsample']} fused upsamplings; loss {la:.6f} vs {lb:.6f}; grad cosine {cos:.6f}")
    assert oka and okb
    assert abs(la - lb) < 2e-3 * max(1.0, abs(la))                       # test_c3_gpu's bound for the patched step
    assert cos > 0.999


@needs_ref
def test_scripts_run_unmodified_with_flow_head(dataset, tmp_path, monkeypatch):
    monkeypatch.setenv("GPSG_FLOW_HEAD", "1")
    work = harness.make_workdir(str(tmp_path / "work"), dataset, src_res=256, num_steps=3, batch_size=2,
                                stage1=dict(src_res=256, num_steps=3, batch_size=2))
    p = harness.run_script(work, "train_stage1.py", patch=True, timeout=1500)
    assert p.returncode == 0, p.stdout[-3000:] + p.stderr[-6000:]
    ckpt1 = glob.glob(os.path.join(work, "experiments", "GPS-GS_stage1_*", "ckpt", "*_final.pth"))
    assert len(ckpt1) == 1
    with open(os.path.join(work, "config", "stage2.yaml"), "w") as f:
        f.write(harness.stage2_yaml(dataset, src_res=256, num_steps=3, batch_size=2, stage1_ckpt=ckpt1[0]))
    q = harness.run_script(work, "train_stage2.py", patch=True, timeout=1500)
    assert q.returncode == 0, q.stdout[-3000:] + q.stderr[-6000:]
    ckpt2 = glob.glob(os.path.join(work, "experiments", "GPS-GS_stage2_*", "ckpt", "*_final.pth"))
    assert len(ckpt2) == 1
    for ck in (ckpt1[0], ckpt2[0]):
        sd = torch.load(ck, map_location="cpu")
        assert all(bool(torch.isfinite(v).all()) for v in sd["network"].values() if v.is_floating_point())
    r = harness.run_script(work, "test_view_interp.py", ["--test_data_root", os.path.join(dataset, "val"), "--ckpt_path",
                                                         ckpt2[0], "--novel_view_nums", "2"], patch=True, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-6000:]
    assert len(glob.glob(os.path.join(work, "interp_out", "*.jpg"))) == 2 * 2          # 2 val samples x 2 novel views
