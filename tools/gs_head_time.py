"""Time the regressor's full-resolution tail: the reference module's torch chain (oracle/_ref, cuDNN defaults) against the
fused kernels (gps_gaussian_b200.gs_head), and a whole RtStereoHumanModel eval forward with GPSG_GS_HEAD off and on.

    python tools/gs_head_time.py [--seconds 2] [--rounds 3] [--no-model] [--trace] [--train] [--out DIR]

On cuda:0, in one process:
  * the tail alone at B = 2 (one inference frame: two source views) and B = 4 (a stage-2 eval batch), 1024^2: from the
    decoder1 output [B,48,512,512], img and depth to the three maps, under no_grad.  The two arms alternate for
    `--rounds` rounds; each round warms up and then times a window of at least `--seconds` with CUDA events.  Each kernel
    is also timed alone, and its achieved FLOP/s and HBM bytes/s are computed from the shape counts below;
  * the eval forward of the reference's RtStereoHumanModel on a synthetic 1024^2 pair (batch 1), switch off / on.
  * --trace: instead, one torch.profiler trace of the switched-on eval forward (DIR/gs_head_eval.pt.trace.json) and the
    table of CUDA kernels that ran in it.
  * --train: instead, forward + backward of the tail at B = 4, 1024^2 (a stage-2 training batch: two samples x two
    source views), the reference module's chain under autograd (cuDNN defaults) against gs_head_train, alternated rounds
    as above; each backward kernel timed by the profiler with its share of the TF32 or HBM bound; and one whole
    harness.c3_step at src_res 1024, batch 2, with GPSG_GS_HEAD_TRAIN off and on: step time and peak allocated memory.
Prints one JSON object with the GPU name and power limit (also written to DIR/gs_head_time.json with --out)."""
import argparse
import json
import os
import subprocess
import sys
import tempfile

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from gps_gaussian_b200 import gs_head, harness, patch  # noqa: E402

DATASHEET_BW = 3.35e12      # H100 SXM HBM3, NVIDIA data sheet
DATASHEET_TF32 = 495e12     # H100 SXM dense TF32, NVIDIA data sheet


def work(B, H=1024, W=1024):
    """Algorithmic FLOPs (2 per MAC, unpadded K) and HBM bytes of the two kernels from the shapes."""
    px = B * H * W
    f1 = 2 * px * 32 * 52 * 9
    f2 = 2 * px * (96 * 32 * 9 + 32 * 8)
    src, io = B * 48 * (H // 2) * (W // 2) * 4, px * 4 * 4          # decoder output; img + depth
    mid = px * 32 * 4
    return {"stage1": dict(flop=f1, bytes=src + io + mid), "stage2": dict(flop=f2, bytes=mid + px * 8 * 4)}


def train_work(B, H=1024, W=1024):
    """Algorithmic FLOPs and HBM bytes of the forward + backward kernels from the shapes (K unpadded)."""
    px = B * H * W
    w = work(B, H, W)
    src = B * 48 * (H // 2) * (W // 2) * 4
    w.update({
        "bwd_heads": dict(flop=2 * px * (96 * 32 * 9 + 2 * 32 * 8), bytes=px * (32 + 8 + 96) * 4),
        "bwd_mid": dict(flop=2 * px * 32 * 96 * 9, bytes=px * (96 + 32 + 32) * 4),
        "wgrad_heads": dict(flop=2 * px * 96 * 32 * 9, bytes=px * (96 + 32) * 4),
        "bwd_cat": dict(flop=2 * px * 52 * 32 * 9, bytes=px * (32 + 48 + 1) * 4),
        "bwd_src": dict(flop=2 * px * 48 * 4, bytes=px * 48 * 4 + src),
        "wgrad_out": dict(flop=2 * px * 32 * 52 * 9, bytes=px * (32 + 4) * 4 + src),
    })
    return w


_KERNEL_NAMES = (("gs_head_stage1", "stage1"), ("gs_head_stage2", "stage2"), ("gs_head_bwd_heads", "bwd_heads"),
                 ("gs_head_bwd_mid", "bwd_mid"), ("gs_head_wgrad<96", "wgrad_heads"), ("gs_head_bwd_cat", "bwd_cat"),
                 ("gs_head_bwd_src", "bwd_src"), ("gs_head_wgrad<32", "wgrad_out"), ("gs_head_bwd_reduce", "bwd_reduce"))


def _per_kernel(prof, w):
    per = {}
    for e in prof.key_averages():
        for pat, name in _KERNEL_NAMES:
            if pat in e.key:
                ms = e.device_time_total / max(e.count, 1) / 1e3
                row = dict(ms=round(ms, 4))
                if name in w:
                    t = ms * 1e-3
                    f, b = w[name]["flop"], w[name]["bytes"]
                    row.update(flop=f, bytes=b, TFLOPs=round(f / t / 1e12, 1), TBps=round(b / t / 1e12, 3),
                               bound="compute" if f / DATASHEET_TF32 > b / DATASHEET_BW else "memory",
                               share_of_bound=round(max(f / DATASHEET_TF32, b / DATASHEET_BW) / t, 3))
                per[name] = row
    return per


def _train_tail(seconds, rounds, B=4):
    m = _module().train()
    H = W = 1024
    x = torch.randn(B, 48, H // 2, W // 2, device="cuda", requires_grad=True)
    img = torch.rand(B, 3, H, W, device="cuda") * 2 - 1
    depth = torch.rand(B, 1, H, W, device="cuda", requires_grad=True)
    grads = [torch.randn(B, c, H, W, device="cuda") for c in (4, 3, 1)]

    def step(fwd):
        m.zero_grad(set_to_none=True)
        x.grad = depth.grad = None
        torch.autograd.backward(fwd(), grads)

    arms = {"torch": lambda: step(lambda: _torch_tail(m, x, img, depth)),
            "fused": lambda: step(lambda: gs_head.gs_head_train(x, img, depth, m))}
    row = {k: [] for k in arms}
    for _ in range(rounds):
        for name, fn in arms.items():
            row[name].append(round(_window(fn, seconds), 4))
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(10):
            arms["fused"]()
        torch.cuda.synchronize()
    for name in arms:
        r = row[name]
        row[name] = dict(ms=r, best=min(r), spread=round((max(r) - min(r)) / min(r), 4))
    row["speedup"] = round(row["torch"]["best"] / row["fused"]["best"], 2)
    row["kernels"] = _per_kernel(prof, train_work(B))
    peak = {}
    for name, fn in arms.items():
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        fn()
        torch.cuda.synchronize()
        peak[name] = round((torch.cuda.max_memory_allocated() - base) / 2 ** 30, 3)
    row["peak_extra_GiB"] = peak
    return {f"B{B}_1024": row}


def _train_step(rounds, steps=5):
    from gps_gaussian_b200 import synth_dataset
    res = {}
    with tempfile.TemporaryDirectory() as root:
        synth_dataset.write_dataset(root, n_train=2, n_val=1, res=1024, hr=True)
        for on in (False, True):
            patch.uninstall()
            os.environ["GPSG_GS_HEAD_TRAIN"] = "1" if on else "0"
            harness.add_reference_to_path()
            patch.install()
            cfg = harness.load_cfg(root, src_res=1024, num_steps=100, batch_size=2)
            st = harness.C3State(cfg)
            harness.c3_step(st, st.batch(0))                              # warm-up (allocator, cuDNN plans)
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            times = []
            for _ in range(rounds):
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                for _ in range(steps):
                    harness.c3_step(st, st.batch(0))
                b.record()
                b.synchronize()
                times.append(round(a.elapsed_time(b) / steps, 2))
            res["on" if on else "off"] = dict(step_ms=times, best=min(times),
                                              max_memory_allocated_GiB=round(torch.cuda.max_memory_allocated() / 2 ** 30, 3))
            del st
            torch.cuda.empty_cache()
        patch.uninstall()
        os.environ.pop("GPSG_GS_HEAD_TRAIN", None)
    return res


def _gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception:
        return torch.cuda.get_device_name()


def _window(fn, seconds):
    """Mean ms per call over a window of at least `seconds`, after a warm-up; CUDA events around the window."""
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    n, total = 0, 0.0
    a.record()
    while total < seconds * 1e3:
        for _ in range(10):
            fn()
        n += 10
        b.record()
        b.synchronize()
        total = a.elapsed_time(b)
    return total / n


def _module():
    harness.add_reference_to_path()
    import types
    from lib.gs_parm_network import GSRegresser
    cfg = types.SimpleNamespace(raft=types.SimpleNamespace(encoder_dims=[32, 48, 96]),
                                gsnet=types.SimpleNamespace(encoder_dims=[32, 48, 96], decoder_dims=[48, 64, 96],
                                                            parm_head_dim=32))
    torch.manual_seed(0)
    return GSRegresser(cfg).cuda().eval()


def _torch_tail(m, x, img, depth):
    """The reference's own statements after decoder1 (lib/gs_parm_network.py), on the module's layers."""
    out = m.out_relu(m.out_conv(torch.cat([m.up(x), img, depth], dim=1)))
    rot = torch.nn.functional.normalize(m.rot_head(out), dim=1)
    return rot, torch.clamp_max(m.scale_head(out), 0.01), m.opacity_head(out)


def _tail(seconds, rounds):
    m = _module()
    ps = [p.detach() for p in gs_head.params_of(m)]
    res = {}
    for B in (2, 4):
        H = W = 1024
        x = torch.randn(B, 48, H // 2, W // 2, device="cuda")
        img = torch.rand(B, 3, H, W, device="cuda") * 2 - 1
        depth = torch.rand(B, 1, H, W, device="cuda")
        arms = {"torch": lambda: _torch_tail(m, x, img, depth), "fused": lambda: gs_head.run(x, img, depth, ps)}
        row = {k: [] for k in arms}
        with torch.no_grad():
            for _ in range(rounds):
                for name, fn in arms.items():
                    row[name].append(round(_window(fn, seconds), 4))
            # per-kernel device times from the profiler, over a short window of its own
            with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                for _ in range(20):
                    gs_head.run(x, img, depth, ps)
                torch.cuda.synchronize()
        kern = {}
        for e in prof.key_averages():
            if "gs_head_stage" in e.key:
                name = "stage1" if "stage1" in e.key else "stage2"
                kern[name] = e.device_time_total / max(e.count, 1) / 1e3          # ms
        w = work(B)
        per = {}
        for k, ms in kern.items():
            t = ms * 1e-3
            per[k] = dict(ms=round(ms, 4), TFLOPs=round(w[k]["flop"] / t / 1e12, 1), TBps=round(w[k]["bytes"] / t / 1e12, 3),
                          flop=w[k]["flop"], bytes=w[k]["bytes"],
                          bound="compute" if w[k]["flop"] / DATASHEET_TF32 > w[k]["bytes"] / DATASHEET_BW else "memory",
                          share_of_bound=round(max(w[k]["flop"] / DATASHEET_TF32, w[k]["bytes"] / DATASHEET_BW) / t, 3))
        for name in arms:
            r = row[name]
            row[name] = dict(ms=r, best=min(r), spread=round((max(r) - min(r)) / min(r), 4))
        row["speedup"] = round(row["torch"]["best"] / row["fused"]["best"], 2)
        row["kernels"] = per
        res[f"B{B}_1024"] = row
        del x, img, depth
        torch.cuda.empty_cache()
    return res


def _eval_setup(root):
    cfg = harness.load_cfg(root, src_res=1024, batch_size=1)
    st = harness.C3State(cfg)
    st.model.eval()
    return st, st.batch(0)


def _eval_forward(st, data):
    with torch.no_grad():
        st.model({k: dict(v) if isinstance(v, dict) else v for k, v in data.items()}, is_train=False)


def _switch(on):
    patch.uninstall()
    os.environ["GPSG_GS_HEAD"] = "1" if on else "0"
    harness.add_reference_to_path()
    patch.install()


def _model(seconds, rounds):
    from gps_gaussian_b200 import synth_dataset
    res = {"off": [], "on": []}
    with tempfile.TemporaryDirectory() as root:
        synth_dataset.write_dataset(root, n_train=1, n_val=1, res=1024, hr=True)
        _switch(False)
        st, data = _eval_setup(root)
        for _ in range(rounds):
            for on in (False, True):
                _switch(on)         # the class method is rebound in place: the model object stays the same
                res["on" if on else "off"].append(round(_window(lambda: _eval_forward(st, data), seconds), 3))
        patch.uninstall()
    for k in ("off", "on"):
        r = res[k]
        res[k] = dict(ms=r, best=min(r), spread=round((max(r) - min(r)) / min(r), 4))
    return res


def _trace(out):
    from gps_gaussian_b200 import synth_dataset
    with tempfile.TemporaryDirectory() as root:
        synth_dataset.write_dataset(root, n_train=1, n_val=1, res=1024, hr=True)
        _switch(True)
        st, data = _eval_setup(root)
        _eval_forward(st, data)
        torch.cuda.synchronize()
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CPU,
                                                torch.profiler.ProfilerActivity.CUDA]) as prof:
            _eval_forward(st, data)
            torch.cuda.synchronize()
        patch.uninstall()
    os.makedirs(out, exist_ok=True)
    prof.export_chrome_trace(os.path.join(out, "gs_head_eval.pt.trace.json"))
    kernels = sorted(((e.key, e.count, round(e.device_time_total / 1e3, 3)) for e in prof.key_averages()
                      if e.device_time_total > 0 and e.device_type == torch.autograd.DeviceType.CUDA),
                     key=lambda k: -k[2])
    return {"kernels": kernels}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=float, default=2.0)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--no-model", action="store_true")
    ap.add_argument("--trace", action="store_true")
    ap.add_argument("--train", action="store_true")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("gs_head_time.py needs a CUDA device")
    if harness.staged_reference() is None:
        raise SystemExit("oracle/_ref is not staged: the torch chain to compare against is the reference's own module")
    torch.cuda.set_device(0)
    out = {"gpu": _gpu_info(), "cudnn_allow_tf32": torch.backends.cudnn.allow_tf32}
    if a.trace:
        if not a.out:
            raise SystemExit("--trace needs --out")
        out["trace"] = _trace(a.out)
    elif a.train:
        out["train_tail"] = _train_tail(a.seconds, a.rounds)
        out["c3_step_1024_batch2"] = _train_step(a.rounds)
    else:
        out["tail"] = _tail(a.seconds, a.rounds)
        if not a.no_model:
            out["eval_forward_1024"] = _model(a.seconds, a.rounds)
    s = json.dumps(out)
    print(s)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        name = "gs_head_trace.json" if a.trace else ("gs_head_train_time.json" if a.train else "gs_head_time.json")
        with open(os.path.join(a.out, name), "w") as f:
            f.write(s + "\n")


if __name__ == "__main__":
    main()
