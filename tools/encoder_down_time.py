"""Time the UnetExtractor's stride-2 stages res2 + res3: the reference modules' own chain (oracle/_ref, cuDNN defaults)
against the fused kernels (gps_gaussian_b200.encoder.run_down), and a whole RtStereoHumanModel eval forward with every
other switch on (GPSG_ENCODER, GPSG_GS_HEAD, GPSG_DECODER) and GPSG_ENCODER_DEEP off and on.  The method is
tools/encoder_time.py's, whose window and eval helpers this tool uses.

    python tools/encoder_down_time.py [--seconds 2] [--rounds 3] [--no-model] [--out DIR]

On cuda:0, in one process:
  * res2 + res3 on the stem output of a 1024^2 input (x1 [B,32,512,512]), TF32 (autocast off, cudnn.allow_tf32) and
    fp16 autocast, B = 2 and 4, under no_grad.  The two arms alternate for `--rounds` rounds of CUDA-event windows of at
    least `--seconds`.  Then, in a separate profiled run, the device time per kernel from torch.profiler with its bytes
    and FLOPs from the shapes and the share of its binding roofline (data-sheet HBM bandwidth or TF32 / FP16 rate);
  * the eval forward of the reference's RtStereoHumanModel on a synthetic 1024^2 pair, GPSG_ENCODER_DEEP off / on,
    alternated.
Prints one JSON object with the GPU name, power limit and max SM clock (also written to DIR/encoder_down_time.json)."""
import argparse
import json
import os
import re
import sys
import tempfile

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import encoder_time as et  # noqa: E402
from gps_gaussian_b200 import encoder, harness, patch  # noqa: E402


def work(B, cin, c, prec, H, W):
    """Algorithmic FLOPs (2 per MAC) and HBM bytes of each kernel of one stage from the shapes (input [B,cin,H,W]);
    e = bytes per stored element.  The halo re-reads and the weight re-reads per tile (served by L2) are not counted."""
    px = B * ((H + 1) // 2) * ((W + 1) // 2)
    e = 2 if prec == "fp16" else 4
    raw = px * c * e
    f3 = 2 * px * c * c * 9
    return {
        "conv0": dict(flop=2 * px * c * cin * 10, bytes=B * cin * H * W * 4 + 2 * raw, peak=prec),
        "conv1": dict(flop=f3, bytes=2 * raw, peak=prec),                 # yb and ye: one raw input
        "conv2": dict(flop=f3, bytes=3 * raw, peak=prec),                 # yc: yb and yd in
        "out": dict(flop=0, bytes=3 * raw + px * c * 4, peak=prec),
    }


_KERNEL = re.compile(r"(down_conv|res_conv|res_out|down_pack|gn_finalize)<([^>]*)>")


def _per_kernel(prof, calls, B, prec):
    """Device ms per launch of each kernel of res2 (C = 48) and res3 (C = 96), keyed by stage, kernel and staging mode
    S (0 the stride-2 conv1 + downsample, 1 relu(GN(y)), 2 the residual xb): res2's C -> C convolutions are res_conv,
    res3's down_conv."""
    ws = {48: work(B, 32, 48, prec, 512, 512), 96: work(B, 48, 96, prec, 256, 256)}
    per = {}
    for ev in prof.key_averages():
        m = _KERNEL.search(ev.key)
        if m is None:
            continue
        kind, args = m.group(1), [t.strip() for t in m.group(2).split(",")]
        c = int(args[0] if kind == "gn_finalize" else args[-1] if kind in ("res_out", "down_pack") else
                args[2] if kind == "down_conv" else args[1])
        k = f"conv{args[-1]}" if kind in ("down_conv", "res_conv") else "out" if kind == "res_out" else kind
        key = f"{'res3' if c == 96 else 'res2'}:{kind}" + (f"<S={args[-1]}>" if k.startswith("conv") else "")
        ms = ev.device_time_total / max(ev.count, 1) / 1e3
        row = dict(ms=round(ms, 4), launches_per_call=round(ev.count / max(calls, 1), 2))
        if k in ws[c]:
            f, b, pk = ws[c][k]["flop"], ws[c][k]["bytes"], et.PEAK[ws[c][k]["peak"]]
            row.update(flop=f, bytes=b, bound="compute" if f / pk > b / et.DATASHEET_BW else "memory",
                       share_of_bound=round(max(f / pk, b / et.DATASHEET_BW) / (ms * 1e-3), 3))
        per[key] = row
    return per


def _stages(seconds, rounds):
    harness.add_reference_to_path()
    from core.extractor import UnetExtractor
    torch.manual_seed(0)
    m = UnetExtractor(in_channel=3, encoder_dim=[32, 48, 96]).cuda().eval()
    p2 = [p.detach() for p in encoder.down_params_of(m.res2)]
    p3 = [p.detach() for p in encoder.down_params_of(m.res3)]
    res = {}
    for prec in ("tf32", "fp16"):
        for B in (2, 4):
            x1 = torch.relu(torch.randn(B, 32, 512, 512, device="cuda"))
            amp = dict(device_type="cuda", dtype=torch.float16, enabled=prec == "fp16")

            def ref():
                with torch.no_grad(), torch.autocast(**amp):
                    return m.res3(m.res2(x1))

            def fused():
                return encoder.run_down(encoder.run_down(x1, p2, prec), p3, prec)
            arms = {"torch": ref, "fused": fused}
            row = {k: [] for k in arms}
            for _ in range(rounds):
                for name, fn in arms.items():
                    row[name].append(round(et._window(fn, seconds), 4))
            for name in arms:
                r = row[name]
                row[name] = dict(ms=r, best=min(r), spread=round((max(r) - min(r)) / min(r), 4))
            row["speedup"] = round(row["torch"]["best"] / row["fused"]["best"], 2)
            with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                for _ in range(10):
                    fused()
                torch.cuda.synchronize()
            row["kernels"] = _per_kernel(prof, 10, B, prec)
            tot = [work(B, 32, 48, prec, 512, 512), work(B, 48, 96, prec, 256, 256)]
            row["bytes_total"] = sum(w["conv0"]["bytes"] + 2 * w["conv1"]["bytes"] + w["conv2"]["bytes"]
                                     + w["out"]["bytes"] for w in tot)
            row["flop_total"] = sum(w["conv0"]["flop"] + 3 * w["conv1"]["flop"] for w in tot)
            res[f"{prec}_B{B}"] = row
            del x1
            torch.cuda.empty_cache()
    return res


def _switch(deep):
    patch.uninstall()
    os.environ.update(GPSG_ENCODER="1", GPSG_GS_HEAD="1", GPSG_DECODER="1", GPSG_ENCODER_DEEP="1" if deep else "0")
    harness.add_reference_to_path()
    patch.install()
    assert patch.encoder_deep() is deep


def _model(seconds, rounds):
    from gps_gaussian_b200 import synth_dataset
    res = {"off": [], "on": []}
    with tempfile.TemporaryDirectory() as root:
        synth_dataset.write_dataset(root, n_train=1, n_val=1, res=1024, hr=True)
        _switch(False)
        _, st, data = et._eval_setup(root)
        for _ in range(rounds):
            for deep in (False, True):
                _switch(deep)       # the class methods are rebound in place: the model object stays the same
                res["on" if deep else "off"].append(round(et._window(lambda: et._eval_forward(st, data), seconds), 3))
        patch.uninstall()
    for k in ("off", "on"):
        r = res[k]
        res[k] = dict(ms=r, best=min(r), spread=round((max(r) - min(r)) / min(r), 4))
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=float, default=2.0)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--no-model", action="store_true")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("encoder_down_time needs a CUDA device")
    out = {"gpu": et._gpu_info(), "stages": _stages(a.seconds, a.rounds)}
    if not a.no_model:
        out["eval_forward_1024_all_switches"] = _model(a.seconds, a.rounds)
    s = json.dumps(out)
    print(s)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "encoder_down_time.json"), "w") as f:
            f.write(s + "\n")


if __name__ == "__main__":
    main()
