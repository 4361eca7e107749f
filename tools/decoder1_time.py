"""Time the regressor's decoder1: the reference's own chain (oracle/_ref: up, cat, the decoder1 module; cuDNN with
allow_tf32) against the fused kernels (gps_gaussian_b200.decoder), and a whole RtStereoHumanModel eval forward with
GPSG_ENCODER=1 GPSG_GS_HEAD=1 and GPSG_DECODER off and on.

    python tools/decoder1_time.py [--seconds 2] [--rounds 3] [--no-model] [--out DIR]

On cuda:0, in one process:
  * decoder1 alone at B = 2 and B = 4, 1024^2 input (s [B,64,256,256], features [B,32,512,512]), TF32, under no_grad.
    The two arms alternate for `--rounds` rounds; each round warms up, then times a window of at least `--seconds` with
    CUDA events.  Then, in a separate run under torch.profiler, the device time per kernel with its bytes and FLOPs from
    the shapes and the share of its binding bound (data-sheet HBM bandwidth or dense TF32 rate);
  * the eval forward of the reference's RtStereoHumanModel on a synthetic 1024^2 pair, GPSG_DECODER off / on, alternated.
Prints one JSON object with the GPU name and power limit read in the same run (also written to DIR/decoder1_time.json).
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


def work(B, Hs=256, Ws=256):
    """Algorithmic FLOPs (2 per MAC) and HBM bytes of each kernel from the shapes (fp32 everywhere)."""
    px = B * 4 * Hs * Ws
    raw = px * 48 * 4
    f3 = 2 * px * 48 * 48 * 9
    return {
        "dec_in": dict(flop=2 * px * 48 * 128 * 10, bytes=B * 64 * Hs * Ws * 4 + px * 64 * 4 + 2 * raw),
        "res_conv<false, 48, 1>": dict(flop=f3, bytes=2 * raw),       # y2 and y4 (two launches)
        "res_conv<false, 48, 2>": dict(flop=f3, bytes=3 * raw),       # y3 from yd and y2
        "res_out<false, 48>": dict(flop=0, bytes=4 * raw),
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


def _regresser():
    harness.add_reference_to_path()
    from lib.gs_parm_network import GSRegresser
    cfg = types.SimpleNamespace(raft=types.SimpleNamespace(encoder_dims=[32, 48, 96]),
                                gsnet=types.SimpleNamespace(encoder_dims=[32, 48, 96], decoder_dims=[48, 64, 96],
                                                            parm_head_dim=32))
    torch.manual_seed(0)
    return GSRegresser(cfg).cuda().eval()


_KERNELS = ("dec_pack", "dec_in", "res_conv<false, 48, 1>", "res_conv<false, 48, 2>", "gn_finalize<", "res_out<false, 48>")
_PER_CALL = {"res_conv<false, 48, 1>": 2, "gn_finalize<": 5}


def _per_kernel(prof, w, calls):
    per = {}
    for ev in prof.key_averages():
        if ev.device_time_total <= 0:
            continue
        for pat in _KERNELS:
            if pat in ev.key:
                ms = ev.device_time_total / max(calls, 1) / _PER_CALL.get(pat, 1) / 1e3
                row = dict(ms=round(ms, 4), launches_per_call=_PER_CALL.get(pat, 1))
                if pat in w:
                    t = ms * 1e-3
                    f, b = w[pat]["flop"], w[pat]["bytes"]
                    row.update(flop=f, bytes=b, TBps=round(b / t / 1e12, 3), TFLOPs=round(f / t / 1e12, 1),
                               bound="tf32" if f / PEAK_TF32 > b / DATASHEET_BW else "hbm",
                               share_of_bound=round(max(f / PEAK_TF32, b / DATASHEET_BW) / t, 3))
                per[pat.rstrip("<")] = row
    return per


def _decoder1(seconds, rounds):
    torch.backends.cudnn.allow_tf32 = True
    m = _regresser()
    ps = [p.detach() for p in decoder.params_of(m)]
    res = {}
    for B in (2, 4):
        g = torch.Generator(device="cuda").manual_seed(B)
        s = torch.rand(B, 64, 256, 256, device="cuda", generator=g)
        fi, fd = (torch.rand(B, 32, 512, 512, device="cuda", generator=g) for _ in range(2))

        def ref():
            with torch.no_grad():
                return m.decoder1(torch.cat([m.up(s), fi, fd], dim=1))

        def fused():
            return decoder.run(s, fi, fd, ps)
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
        row["bytes_total"] = w["dec_in"]["bytes"] + 2 * w["res_conv<false, 48, 1>"]["bytes"] + w["res_conv<false, 48, 2>"]["bytes"] \
            + w["res_out<false, 48>"]["bytes"]
        row["flop_total"] = w["dec_in"]["flop"] + 3 * w["res_conv<false, 48, 1>"]["flop"]
        res[f"B{B}"] = row
        del s, fi, fd
        torch.cuda.empty_cache()
    return res


def _switch(on):
    patch.uninstall()
    os.environ.update(GPSG_ENCODER="1", GPSG_GS_HEAD="1", GPSG_DECODER="1" if on else "0")
    harness.add_reference_to_path()
    patch.install()


def _model(seconds, rounds):
    from gps_gaussian_b200 import synth_dataset
    res = {"off": [], "on": []}
    decoder.reset_counts()
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
                _switch(on)         # the class method is rebound in place: the model object stays the same
                res["on" if on else "off"].append(round(_window(fwd, seconds), 3))
        patch.uninstall()
    for k in ("off", "on"):
        r = res[k]
        res[k] = dict(ms=r, best=min(r), spread=round((max(r) - min(r)) / min(r), 4))
    res["decoder1_kernel_calls"] = decoder.counts()["forward"]
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=float, default=2.0)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--no-model", action="store_true")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("decoder1_time.py needs a CUDA device")
    if harness.staged_reference() is None:
        raise SystemExit("oracle/_ref is not staged: the torch chain to compare against is the reference's own module")
    torch.cuda.set_device(0)
    out = {"gpu": _gpu_info(), "cudnn_allow_tf32": True, "decoder1": _decoder1(a.seconds, a.rounds)}
    if not a.no_model:
        out["eval_forward_1024"] = _model(a.seconds, a.rounds)
    s = json.dumps(out)
    print(s)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "decoder1_time.json"), "w") as f:
            f.write(s + "\n")


if __name__ == "__main__":
    main()
