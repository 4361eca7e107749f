"""Time the RAFT update iterations: the reference's FlowUpdateModule.forward (oracle/_ref: cuDNN and torch elementwise
for the update block) against the same forward with the update block on the fused kernels
(gps_gaussian_b200.update.make_update_forward), and a whole RtStereoHumanModel eval forward with every other switch on
and GPSG_UPDATE off and on.  The method is tools/encoder_time.py's, whose window and eval helpers this tool uses.

    python tools/update_time.py [--seconds 2] [--rounds 3] [--no-model] [--out DIR]

On cuda:0, in one process, with the patch installed (the fused corr build and lookup, GPSG_FLOW_HEAD's upsampling) in
both arms, so that the arms differ only in the update block:
  * FlowUpdateModule.forward at the stage-2 eval shape (1/8 of a 1024^2 pair: [B,96,128,128], 3 iterations, test mode,
    corr "reg_cuda"), B = 2 (one pair) and 4, under no_grad.  The two arms alternate for `--rounds` rounds of
    CUDA-event windows of at least `--seconds`.  Then, in a separate profiled run, the device time per kernel from
    torch.profiler with its FLOPs and bytes from the shapes and the share of its binding roofline (data-sheet fp16
    tensor rate or HBM bandwidth);
  * the eval forward of the reference's RtStereoHumanModel on a synthetic 1024^2 pair, GPSG_UPDATE off / on,
    alternated.
Prints one JSON object with the GPU name, power limit and max SM clock (also written to DIR/update_time.json)."""
import argparse
import json
import os
import re
import sys
import tempfile
import types

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import encoder_time as et  # noqa: E402
from gps_gaussian_b200 import harness, patch, update  # noqa: E402

H = W = 128
ITERS = 3
FMAP_D = 96


def work(B, mask_launches=1):
    """Algorithmic FLOPs (2 per MAC) and HBM bytes per launch of each kernel from the shapes (fp16 intermediates, 2
    bytes; the halo and weight re-reads served by L2 are not counted).  Keys are the profiler's kernel names."""
    px = B * H * W
    return {
        "motion_in": dict(flop=2 * px * 64 * (36 + 98), bytes=px * (36 * 2 + 2 * 4 + 128 * 2 + 4)),
        "uconv<3,64,0>": dict(flop=2 * px * 128 * 576, bytes=px * (128 + 128) * 2),
        "uconv<3,128,0>": dict(flop=2 * px * 126 * 1152, bytes=px * (128 + 126) * 2),
        "uconv<3,192,1>": dict(flop=2 * px * 192 * 2016, bytes=px * (96 + 128 + 192 + 96 + 192) * 2),
        "uconv<3,96,2>": dict(flop=2 * px * 96 * 2016, bytes=px * (96 + 128 + 96 + 96 + 96 + 96) * 2),
        # flow_head.conv1 on every iteration, mask[0] with it on the last (the mean over the launches of a forward)
        "uconv<3,256,0>": dict(flop=2 * px * 256 * 864 * (ITERS + mask_launches) / ITERS,
                               bytes=px * (96 + 256 * (ITERS + mask_launches) / ITERS) * 2),
        "uconv<1,192,3>": dict(flop=2 * px * 576 * 256, bytes=px * (256 + 576) * 2),
        "uconv<3,8,4>": dict(flop=2 * px * 2 * 2304, bytes=px * (256 * 2 + 4 + 8)),
    }


_KERNEL = re.compile(r"(uconv|motion_in|update_pack)<([^>]*)>")


def _per_kernel(prof, calls, B):
    ws = work(B)
    per = {}
    for ev in prof.key_averages():
        m = _KERNEL.search(ev.key)
        if m is None:
            continue
        kind, args = m.group(1), m.group(2).replace(" ", "")
        key = kind if kind in ("motion_in", "update_pack") else f"{kind}<{args}>"
        ms = ev.device_time_total / max(ev.count, 1) / 1e3
        row = dict(ms=round(ms, 4), launches_per_call=round(ev.count / max(calls, 1), 2))
        if key in ws:
            f, b = ws[key]["flop"], ws[key]["bytes"]
            row.update(flop=int(f), bytes=int(b), bound="compute" if f / et.PEAK["fp16"] > b / et.DATASHEET_BW else "memory",
                       share_of_bound=round(max(f / et.PEAK["fp16"], b / et.DATASHEET_BW) / (ms * 1e-3), 3))
        per[key] = row
    return per


def _install(on):
    patch.uninstall()
    os.environ.update(GPSG_FLOW_HEAD="1", GPSG_ENCODER="1", GPSG_ENCODER_DEEP="1", GPSG_GS_HEAD="1", GPSG_DECODER="1",
                      GPSG_UPDATE="1" if on else "0")
    harness.add_reference_to_path()
    patch.install()
    assert patch.update() is on


def _module(seconds, rounds):
    _install(False)
    import core.raft_stereo_human as rsh
    args = types.SimpleNamespace(mixed_precision=True, n_gru_layers=1, slow_fast_gru=None, hidden_dims=[96, 96, 96],
                                 corr_levels=4, corr_radius=4, n_downsample=3, corr_implementation="reg_cuda")
    torch.manual_seed(0)
    m = rsh.FlowUpdateModule(args).cuda().eval()
    orig = rsh.FlowUpdateModule.__dict__["forward"]
    ours = update.make_update_forward(orig)
    res = {}
    for B in (2, 4):
        g = torch.Generator(device="cuda").manual_seed(B)
        f1 = torch.randn(B, FMAP_D, H, W, device="cuda", generator=g).half()
        f2 = torch.randn(B, FMAP_D, H, W, device="cuda", generator=g).half()
        net = torch.tanh(torch.randn(B, 96, H, W, device="cuda", generator=g)).half()
        ctx = torch.randn(B, 288, H, W, device="cuda", generator=g).half()

        def arm(fwd):
            def run():
                with torch.no_grad():
                    return fwd(m, f1, f2, [net], [list(ctx.split(96, 1))], ITERS, None, True)
            return run
        arms = {"module": arm(orig), "kernels": arm(ours)}
        a, b = arms["module"](), arms["kernels"]()
        row = {"flow_mean_abs_diff": float((a - b).abs().mean()), "flow_mean_abs": float(a.abs().mean())}
        times = {k: [] for k in arms}
        for _ in range(rounds):
            for name, fn in arms.items():
                times[name].append(round(et._window(fn, seconds), 4))
        for name, r in times.items():
            row[name] = dict(ms=r, best=min(r), spread=round((max(r) - min(r)) / min(r), 4))
        row["speedup"] = round(row["module"]["best"] / row["kernels"]["best"], 2)
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            for _ in range(10):
                arms["kernels"]()
            torch.cuda.synchronize()
        row["kernels_per_forward"] = _per_kernel(prof, 10, B)
        w = work(B)
        row["flop_per_forward"] = int(sum(v["flop"] for v in w.values()) * ITERS - w["uconv<1,192,3>"]["flop"]
                                      * (ITERS - 1))
        res[f"B{B}"] = row
        del f1, f2, net, ctx
        torch.cuda.empty_cache()
    patch.uninstall()
    return res


def _model(seconds, rounds):
    from gps_gaussian_b200 import synth_dataset
    res = {"off": [], "on": []}
    with tempfile.TemporaryDirectory() as root:
        synth_dataset.write_dataset(root, n_train=1, n_val=1, res=1024, hr=True)
        _install(False)
        _, st, data = et._eval_setup(root)
        for _ in range(rounds):
            for on in (False, True):
                _install(on)        # the class method is rebound in place: the model object stays the same
                res["on" if on else "off"].append(round(et._window(lambda: et._eval_forward(st, data), seconds), 3))
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
        raise SystemExit("update_time needs a CUDA device")
    out = {"gpu": et._gpu_info(), "update_module": _module(a.seconds, a.rounds)}
    if not a.no_model:
        out["eval_forward_1024_all_switches"] = _model(a.seconds, a.rounds)
    s = json.dumps(out)
    print(s)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "update_time.json"), "w") as f:
            f.write(s + "\n")


if __name__ == "__main__":
    main()
