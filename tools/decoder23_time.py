"""Time the regressor's decoder3 and decoder2: the reference's own chain (oracle/_ref: the decoder3 module, up, cat,
the decoder2 module; cuDNN with allow_tf32) against the fused kernels (gps_gaussian_b200.decoder.run3 + run2), and a
whole RtStereoHumanModel eval forward with every other switch on and GPSG_DECODER_DEEP off and on.

    python tools/decoder23_time.py [--seconds 2] [--rounds 3] [--no-model] [--out DIR]

On cuda:0, in one process:
  * decoder2(cat(up(decoder3(cat(f3i, f3d))), f2i, f2d)) at B = 2 and B = 4 for a 1024^2 input (f3 [B,96,128,128],
    f2 [B,48,256,256]), TF32, under no_grad.  The two arms alternate for `--rounds` rounds; each round warms up, then
    times a window of at least `--seconds` with CUDA events.  Then, in a separate run under torch.profiler, the device
    time per kernel with its bytes and FLOPs from the shapes and the share of its binding bound (data-sheet HBM
    bandwidth or dense TF32 rate);
  * the eval forward of the reference's RtStereoHumanModel on a synthetic 1024^2 pair with GPSG_ENCODER,
    GPSG_ENCODER_DEEP, GPSG_GS_HEAD, GPSG_DECODER, GPSG_UPDATE and GPSG_FLOW_HEAD on, GPSG_DECODER_DEEP off / on,
    alternated.
Prints one JSON object with the GPU name and power limit read in the same run (also written to DIR/decoder23_time.json).
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import types

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from gps_gaussian_b200 import decoder, harness, patch  # noqa: E402

DATASHEET_BW = 3.35e12      # H100 SXM HBM3, NVIDIA data sheet
PEAK_TF32 = 495e12          # dense, NVIDIA data sheet


def work(B, H=128, W=128):
    """Algorithmic FLOPs (2 per MAC) and HBM bytes of each kernel from the shapes (fp32 everywhere), per launch; the
    C -> C convolutions with S = 1 run twice per stage."""
    out = {}
    for c, h, w, ins in ((96, H, W, B * H * W * 192 * 4),
                         (64, 2 * H, 2 * W, B * H * W * 96 * 4 + B * 4 * H * W * 96 * 4)):
        px = B * h * w
        raw = px * c * 4
        f3 = 2 * px * c * c * 9
        out[f"down_conv<false, 192, {c}, 3>"] = dict(flop=2 * px * c * 192 * 10, bytes=ins + 2 * raw)
        out[f"down_conv<false, {c}, {c}, 1>"] = dict(flop=f3, bytes=2 * raw)
        out[f"down_conv<false, {c}, {c}, 2>"] = dict(flop=f3, bytes=3 * raw)
        out[f"res_out<false, {c}>"] = dict(flop=0, bytes=4 * raw)
    return out


_PER_CALL = {"down_conv<false, 96, 96, 1>": 2, "down_conv<false, 64, 64, 1>": 2, "gn_finalize<96>": 5,
             "gn_finalize<64>": 5}
_KERNELS = ("dec23_pack<192, 96>", "dec23_pack<192, 64>", "down_conv<false, 192, 96, 3>", "down_conv<false, 96, 96, 1>",
            "down_conv<false, 96, 96, 2>", "gn_finalize<96>", "res_out<false, 96>", "down_conv<false, 192, 64, 3>",
            "down_conv<false, 64, 64, 1>", "down_conv<false, 64, 64, 2>", "gn_finalize<64>", "res_out<false, 64>")


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


def _regresser():
    harness.add_reference_to_path()
    from lib.gs_parm_network import GSRegresser
    cfg = types.SimpleNamespace(raft=types.SimpleNamespace(encoder_dims=[32, 48, 96]),
                                gsnet=types.SimpleNamespace(encoder_dims=[32, 48, 96], decoder_dims=[48, 64, 96],
                                                            parm_head_dim=32))
    torch.manual_seed(0)
    return GSRegresser(cfg).cuda().eval()


def _per_kernel(prof, w, calls):
    per = {}
    for ev in prof.key_averages():
        if ev.device_time_total <= 0:
            continue
        for pat in _KERNELS:
            if pat + "(" in ev.key or ev.key.endswith(pat):
                n = _PER_CALL.get(pat, 1)
                ms = ev.device_time_total / max(calls, 1) / n / 1e3
                row = dict(ms=round(ms, 4), launches_per_call=n)
                if pat in w:
                    t = ms * 1e-3
                    f, b = w[pat]["flop"], w[pat]["bytes"]
                    row.update(flop=f, bytes=b, TBps=round(b / t / 1e12, 3), TFLOPs=round(f / t / 1e12, 1),
                               bound="tf32" if f / PEAK_TF32 > b / DATASHEET_BW else "hbm",
                               share_of_bound=round(max(f / PEAK_TF32, b / DATASHEET_BW) / t, 3))
                per[pat] = row
    return per


def _decoders(seconds, rounds):
    torch.backends.cudnn.allow_tf32 = True
    m = _regresser()
    p3, p2 = ([p.detach() for p in ps] for ps in decoder.deep_params_of(m))
    res = {}
    for B in (2, 4):
        g = torch.Generator(device="cuda").manual_seed(B)
        f3i, f3d = (torch.randn(B, 96, 128, 128, device="cuda", generator=g) for _ in range(2))
        f2i, f2d = (torch.randn(B, 48, 256, 256, device="cuda", generator=g) for _ in range(2))

        def ref():
            with torch.no_grad():
                x = m.decoder3(torch.cat([f3i, f3d], dim=1))
                return m.decoder2(torch.cat([m.up(x), f2i, f2d], dim=1))

        def fused():
            return decoder.run2(decoder.run3(f3i, f3d, p3), f2i, f2d, p2)
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
        w = work(B)
        row["kernels"] = _per_kernel(prof, w, 10)
        row["bytes_total"] = sum(v["bytes"] * _PER_CALL.get(k, 1) for k, v in w.items())
        row["flop_total"] = sum(v["flop"] * _PER_CALL.get(k, 1) for k, v in w.items())
        row["bound_ms"] = round(max(row["bytes_total"] / DATASHEET_BW, row["flop_total"] / PEAK_TF32) * 1e3, 4)
        res[f"B{B}"] = row
        del f3i, f3d, f2i, f2d
        torch.cuda.empty_cache()
    return res


_OTHERS = ("GPSG_ENCODER", "GPSG_ENCODER_DEEP", "GPSG_GS_HEAD", "GPSG_DECODER", "GPSG_UPDATE", "GPSG_FLOW_HEAD")


def _switch(on):
    patch.uninstall()
    os.environ.update({k: "1" for k in _OTHERS}, GPSG_DECODER_DEEP="1" if on else "0")
    harness.add_reference_to_path()
    patch.install()


def _model(seconds, rounds):
    from gps_gaussian_b200 import synth_dataset
    res = {"off": [], "on": []}
    decoder.reset_deep_counts()
    with tempfile.TemporaryDirectory() as root:
        synth_dataset.write_dataset(root, n_train=1, n_val=1, res=1024, hr=True)
        _switch(False)
        cfg = harness.load_cfg(root, src_res=1024, batch_size=1)
        st = harness.C3State(cfg)
        st.model.eval()
        data = st.batch(0)

        def fwd():
            with torch.no_grad():
                return st.model({k: dict(v) if isinstance(v, dict) else v for k, v in data.items()}, is_train=False)
        for _ in range(rounds):
            for on in (False, True):
                _switch(on)         # the class methods are rebound in place: the model object stays the same
                res["on" if on else "off"].append(round(_window(fwd, seconds), 3))
        patch.uninstall()
    for k in ("off", "on"):
        r = res[k]
        res[k] = dict(ms=r, best=min(r), spread=round((max(r) - min(r)) / min(r), 4))
    res["decoder2_kernel_calls"] = decoder.deep_counts()["decoder2"]
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=float, default=2.0)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--no-model", action="store_true")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("decoder23_time.py needs a CUDA device")
    if harness.staged_reference() is None:
        raise SystemExit("oracle/_ref is not staged: the torch chain to compare against is the reference's own modules")
    torch.cuda.set_device(0)
    out = {"gpu": _gpu_info(), "cudnn_allow_tf32": True, "decoder3_decoder2": _decoders(a.seconds, a.rounds)}
    if not a.no_model:
        out["eval_forward_1024"] = _model(a.seconds, a.rounds)
    s = json.dumps(out)
    print(s)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "decoder23_time.json"), "w") as f:
            f.write(s + "\n")


if __name__ == "__main__":
    main()
