"""Time the UnetExtractor's half-resolution stem (in_ds + res1): the reference module's own chain (oracle/_ref, cuDNN
defaults) against the fused kernels (gps_gaussian_b200.encoder), and a whole RtStereoHumanModel eval forward with
GPSG_ENCODER off and on.

    python tools/encoder_time.py [--seconds 2] [--rounds 3] [--no-model] [--trace] [--out DIR]

On cuda:0, in one process:
  * the stem alone, Cin = 3 and Cin = 1, TF32 (autocast off, cudnn.allow_tf32) and fp16 autocast, B = 2 and B = 4 at
    1024^2, under no_grad.  The two arms alternate for `--rounds` rounds; each round warms up, then times a window of at
    least `--seconds` with CUDA events.  Per kernel: device time from torch.profiler, bytes and FLOPs from the shapes,
    and the share of its binding roofline (data-sheet HBM bandwidth or TF32 / FP16 / FP32 rate);
  * the eval forward of the reference's RtStereoHumanModel on a synthetic 1024^2 pair, switch off / on, alternated.
  * --trace: instead, one torch.profiler trace of the eval forward plus pts2render per switch setting (DIR/encoder_eval_
    {off,on}.pt.trace.json), and the device time per reference module: CUDA events recorded by forward hooks around
    each module (img encoder stem / res2 / res3, cnet, the GRU iterations, the depth encoder, decoders 3/2/1, the tail)
    and around pts2render, summed per module over the forward.
Prints one JSON object with the GPU name, power limit and max SM clock (also written to DIR/encoder_time.json)."""
import argparse
import json
import os
import subprocess
import sys
import tempfile

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from gps_gaussian_b200 import encoder, harness, patch  # noqa: E402

DATASHEET_BW = 3.35e12      # H100 SXM HBM3, NVIDIA data sheet
PEAK = {"tf32": 495e12, "fp16": 989e12, "fp32": 67e12}   # dense, NVIDIA data sheet


def work(B, cin, prec, H=1024, W=1024):
    """Algorithmic FLOPs (2 per MAC) and HBM bytes of each kernel from the shapes; e = bytes per stored element."""
    px = B * ((H + 1) // 2) * ((W + 1) // 2)
    e = 2 if prec == "fp16" else 4
    raw = px * 32 * e
    f3 = 2 * px * 32 * 32 * 9
    return {
        "stem_in": dict(flop=2 * px * 32 * 25 * cin, bytes=B * cin * H * W * 4 + raw, peak="fp32"),
        "stem_conv_a": dict(flop=f3, bytes=2 * raw, peak=prec),          # one input tensor (3 of the 4 convolutions)
        "stem_conv_r": dict(flop=f3, bytes=3 * raw, peak=prec),          # block 2's first: y0 and y2 in
        "stem_out": dict(flop=0, bytes=3 * raw + px * 32 * 4, peak=prec),
    }


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


def _extractor(cin):
    harness.add_reference_to_path()
    from core.extractor import UnetExtractor
    torch.manual_seed(0)
    return UnetExtractor(in_channel=cin, encoder_dim=[32, 48, 96]).cuda().eval()


_KERNELS = (("stem_in", "stem_in"), ("stem_conv<", "stem_conv"), ("gn_finalize<", "stem_gn_finalize"),
            ("stem_out", "stem_out"))


def _per_kernel(prof, w, calls):
    per = {}
    for ev in prof.key_averages():
        for pat, name in _KERNELS:
            if pat in ev.key:
                key = name
                if name == "stem_conv":
                    key = "stem_conv_r" if "Li2E" in ev.key or ", 2>" in ev.key else "stem_conv_a"
                n_per_call = 3 if key == "stem_conv_a" else (5 if key == "stem_gn_finalize" else 1)
                ms = ev.device_time_total / max(calls, 1) / n_per_call / 1e3
                row = dict(ms=round(ms, 4))
                if key in w:
                    t = ms * 1e-3
                    f, b, pk = w[key]["flop"], w[key]["bytes"], PEAK[w[key]["peak"]]
                    row.update(flop=f, bytes=b, TBps=round(b / t / 1e12, 3),
                               bound="compute" if f / pk > b / DATASHEET_BW else "memory",
                               share_of_bound=round(max(f / pk, b / DATASHEET_BW) / t, 3))
                per[key] = row
    return per


def _stem(seconds, rounds):
    res = {}
    for cin in (3, 1):
        m = _extractor(cin)
        ps = [p.detach() for p in encoder.params_of(m)]
        for prec in ("tf32", "fp16"):
            for B in (2, 4):
                x = torch.rand(B, cin, 1024, 1024, device="cuda")
                amp = dict(device_type="cuda", dtype=torch.float16, enabled=prec == "fp16")

                def ref():
                    with torch.no_grad(), torch.autocast(**amp):
                        return m.res1(m.in_ds(x))

                def fused():
                    return encoder.run(x, ps, prec)
                arms = {"torch": ref, "fused": fused}
                row = {k: [] for k in arms}
                for _ in range(rounds):
                    for name, fn in arms.items():
                        row[name].append(round(_window(fn, seconds), 4))
                for name in arms:
                    r = row[name]
                    row[name] = dict(ms=r, best=min(r), spread=round((max(r) - min(r)) / min(r), 4))
                row["speedup"] = round(row["torch"]["best"] / row["fused"]["best"], 2)
                with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                    for _ in range(10):
                        fused()
                    torch.cuda.synchronize()
                row["kernels"] = _per_kernel(prof, work(B, cin, prec), 10)
                w = work(B, cin, prec)
                row["bytes_total"] = w["stem_in"]["bytes"] + 3 * w["stem_conv_a"]["bytes"] + w["stem_conv_r"]["bytes"] \
                    + w["stem_out"]["bytes"]
                row["flop_total"] = w["stem_in"]["flop"] + 4 * w["stem_conv_a"]["flop"]
                res[f"cin{cin}_{prec}_B{B}"] = row
                del x
                torch.cuda.empty_cache()
    return res


def _switch(on):
    patch.uninstall()
    os.environ["GPSG_ENCODER"] = "1" if on else "0"
    harness.add_reference_to_path()
    patch.install()


def _eval_setup(root):
    cfg = harness.load_cfg(root, src_res=1024, batch_size=1)
    st = harness.C3State(cfg)
    st.model.eval()
    return cfg, st, st.batch(0)


def _eval_forward(st, data):
    with torch.no_grad():
        return st.model({k: dict(v) if isinstance(v, dict) else v for k, v in data.items()}, is_train=False)


def _model(seconds, rounds):
    from gps_gaussian_b200 import synth_dataset
    res = {"off": [], "on": []}
    with tempfile.TemporaryDirectory() as root:
        synth_dataset.write_dataset(root, n_train=1, n_val=1, res=1024, hr=True)
        _switch(False)
        _, st, data = _eval_setup(root)
        for _ in range(rounds):
            for on in (False, True):
                _switch(on)         # the class method is rebound in place: the model object stays the same
                res["on" if on else "off"].append(round(_window(lambda: _eval_forward(st, data), seconds), 3))
        patch.uninstall()
    for k in ("off", "on"):
        r = res[k]
        res[k] = dict(ms=r, best=min(r), spread=round((max(r) - min(r)) / min(r), 4))
    return res


def _module_spans(model):
    """Forward hooks recording CUDA events around the modules of the split; returns (spans, handles)."""
    rs = model.raft_stereo
    gs = model.gs_parm_regresser
    mods = {"img_encoder": model.img_encoder, "img_encoder.in_ds": model.img_encoder.in_ds,
            "img_encoder.res1": model.img_encoder.res1, "img_encoder.res2": model.img_encoder.res2,
            "img_encoder.res3": model.img_encoder.res3, "cnet": rs.cnet, "gru_iterations": rs.update_module,
            "depth_encoder": gs.depth_encoder, "decoder3": gs.decoder3, "decoder2": gs.decoder2, "decoder1": gs.decoder1,
            "regresser": gs}
    spans = {k: [] for k in mods}
    handles = []
    for name, mod in mods.items():
        def pre(m, a, name=name):
            ev = torch.cuda.Event(enable_timing=True)
            ev.record()
            spans[name].append([ev, None])

        def post(m, a, o, name=name):
            ev = torch.cuda.Event(enable_timing=True)
            ev.record()
            spans[name][-1][1] = ev
        handles += [mod.register_forward_pre_hook(pre), mod.register_forward_hook(post)]
    return spans, handles


def _split(spans):
    torch.cuda.synchronize()
    ms = {k: round(sum(a.elapsed_time(b) for a, b in v if b is not None), 3) for k, v in spans.items()}
    n = {k: len(v) for k, v in spans.items()}
    out = dict(ms)
    # the image encoder runs once on the stacked pair; with the switch on, in_ds / res1 are not called as modules
    out["img_encoder.stem"] = round(ms["img_encoder"] - ms["img_encoder.res2"] - ms["img_encoder.res3"], 3)
    out["tail"] = round(ms["regresser"] - ms["depth_encoder"] - ms["decoder3"] - ms["decoder2"] - ms["decoder1"], 3)
    out["calls"] = n
    return out


def _trace(out):
    from gps_gaussian_b200 import synth_dataset
    res = {}
    with tempfile.TemporaryDirectory() as root:
        synth_dataset.write_dataset(root, n_train=1, n_val=1, res=1024, hr=True)
        for on in (False, True):
            _switch(on)
            cfg, st, data = _eval_setup(root)
            from lib.GaussianRender import pts2render

            def run():
                o, _, _ = _eval_forward(st, data)
                with torch.no_grad():
                    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    a.record()
                    pts2render(o, bg_color=cfg.dataset.bg_color)
                    b.record()
                return a, b
            run()
            torch.cuda.synchronize()
            spans, handles = _module_spans(st.model)
            a, b = run()
            split = _split(spans)
            split["render"] = round(a.elapsed_time(b), 3)
            for h in handles:
                h.remove()
            with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CPU,
                                                    torch.profiler.ProfilerActivity.CUDA]) as prof:
                run()
                torch.cuda.synchronize()
            os.makedirs(out, exist_ok=True)
            tag = "on" if on else "off"
            prof.export_chrome_trace(os.path.join(out, f"encoder_eval_{tag}.pt.trace.json"))
            kernels = sorted(((e.key, e.count, round(e.device_time_total / 1e3, 3)) for e in prof.key_averages()
                              if e.device_time_total > 0 and e.device_type == torch.autograd.DeviceType.CUDA),
                             key=lambda k: -k[2])
            res[tag] = {"module_ms": split, "device_ms_total": round(sum(k[2] for k in kernels), 3),
                        "top_kernels": kernels[:25]}
            del st, data
            torch.cuda.empty_cache()
        patch.uninstall()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=float, default=2.0)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--no-model", action="store_true")
    ap.add_argument("--trace", action="store_true")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("encoder_time.py needs a CUDA device")
    if harness.staged_reference() is None:
        raise SystemExit("oracle/_ref is not staged: the torch chain to compare against is the reference's own module")
    torch.cuda.set_device(0)
    out = {"gpu": _gpu_info(), "cudnn_allow_tf32": torch.backends.cudnn.allow_tf32}
    if a.trace:
        if not a.out:
            raise SystemExit("--trace needs --out")
        out["trace"] = _trace(a.out)
    else:
        out["stem"] = _stem(a.seconds, a.rounds)
        if not a.no_model:
            out["eval_forward_1024"] = _model(a.seconds, a.rounds)
    s = json.dumps(out)
    print(s)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "encoder_trace.json" if a.trace else "encoder_time.json"), "w") as f:
            f.write(s + "\n")


if __name__ == "__main__":
    main()
