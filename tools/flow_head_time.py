"""Time the disparity head: the reference's op chain (oracle/_ref) against the fused kernels (gps_gaussian_b200.flow_head).

    python tools/flow_head_time.py [--iters 20] [--steps 3] [--no-steps] [--out DIR]

In one process, on cuda:0:
  * convex upsampling at the stage-1 shape (N = 12, fp32 mask) and the stage-2 shape (N = 4, fp16 mask), H = W = 128,
    f = 8: forward and forward + backward, the two implementations alternating, timed with CUDA events; achieved bytes/s
    against the bytes the shapes require (read the mask and flow, write the output; the backward also reads the upstream
    gradient and writes dL/dmask and dL/dflow) and peak max_memory_allocated per call;
  * sequence_loss at [N, 1, 1024, 1024] with 3 fp32 predictions and an fp16 flow_gt (as the training cache stores it),
    forward + backward, timed by the host clock (its host synchronisations are the point);
  * the whole stage-1 step (batch 6) and stage-2 step (batch 2) at src_res 1024 with GPSG_FLOW_HEAD on and off.
Prints one JSON object with the GPU name and power limit (also written to DIR/flow_head_time.json with --out)."""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time
import types

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from gps_gaussian_b200 import flow_head, harness, patch  # noqa: E402

DATASHEET_BW = 3.35e12      # H100 SXM HBM3, NVIDIA data sheet


def _gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                              text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception:
        return torch.cuda.get_device_name()


def _events(fn, iters):
    fn()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / iters, (torch.cuda.max_memory_allocated() - base) / 2 ** 20


def _upsample(iters):
    harness.add_reference_to_path()
    from core.raft_stereo_human import FlowUpdateModule
    ref = lambda fl, m: FlowUpdateModule.upsample_flow(types.SimpleNamespace(args=types.SimpleNamespace(n_downsample=3)), fl, m)
    ours = lambda fl, m: flow_head.convex_upsample(fl, m, 8)
    res = {}
    for stage, N, mdt in ((1, 12, torch.float32), (2, 4, torch.float16)):
        H = W = 128
        flow = (torch.randn(N, 2, H, W, device="cuda") * 8).requires_grad_()
        mask = (torch.randn(N, 576, H, W, device="cuda") * 4).to(mdt).requires_grad_()
        g = torch.randn(N, 2, 8 * H, 8 * W, device="cuda")
        esz = mask.element_size()
        fwd_bytes = N * 576 * H * W * esz + flow.numel() * 4 + g.numel() * 4
        bwd_bytes = fwd_bytes + N * 576 * H * W * esz + flow.numel() * 4 * 2        # + grad_out read, dmask and dflow
        row = {}
        for rnd in range(2):                                # alternate the two implementations
            for name, fn in (("op_chain", ref), ("fused", ours)):
                def fwd():
                    with torch.no_grad():
                        fn(flow, mask)

                def fwdbwd():
                    flow.grad = mask.grad = None
                    fn(flow, mask).backward(g)
                tf, mf = _events(fwd, iters)
                tb, mb = _events(fwdbwd, iters)
                r = row.setdefault(name, {"fwd_ms": [], "fwdbwd_ms": []})
                r["fwd_ms"].append(round(tf, 4))
                r["fwdbwd_ms"].append(round(tb, 4))
                r["fwd_peak_MiB"], r["fwdbwd_peak_MiB"] = round(mf, 1), round(mb, 1)
        for r in row.values():
            r["fwd_TBps"] = round(fwd_bytes / (min(r["fwd_ms"]) * 1e-3) / 1e12, 3)
            r["fwdbwd_TBps"] = round(bwd_bytes / (min(r["fwdbwd_ms"]) * 1e-3) / 1e12, 3)
        row["bytes_fwd"], row["bytes_fwdbwd"] = fwd_bytes, bwd_bytes
        res[f"stage{stage}"] = row
    return res


def _seq_loss(iters):
    harness.add_reference_to_path()
    import lib.loss
    ref = patch.original(lib.loss, "sequence_loss")
    res = {}
    for stage, N in ((1, 12), (2, 4)):
        gt = (torch.rand(N, 1, 1024, 1024, device="cuda") * -40).half()          # the training cache's fp16 flow
        valid = (torch.rand(N, 1, 1024, 1024, device="cuda") > 0.3).float()
        preds = [(gt.float() + torch.randn(gt.shape, device="cuda")).requires_grad_() for _ in range(3)]
        row = {}
        for rnd in range(2):
            for name, fn in (("op_chain", ref), ("fused", flow_head.sequence_loss)):
                def step():
                    loss, _ = fn(preds, gt, valid)
                    loss.backward()
                step()
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                for _ in range(iters):
                    step()
                torch.cuda.synchronize()
                row.setdefault(name, []).append(round((time.perf_counter() - t0) / iters * 1e3, 4))
        res[f"stage{stage}_fwdbwd_ms"] = row
    return res


def _steps(n_steps):
    from gps_gaussian_b200 import synth_dataset
    res = {}
    with tempfile.TemporaryDirectory() as root:
        synth_dataset.write_dataset(root, n_train=6, n_val=1, res=1024, hr=True)
        for stage, bs in ((1, 6), (2, 2)):
            for rnd in range(2):
                for on in (False, True):
                    patch.uninstall()
                    os.environ["GPSG_FLOW_HEAD"] = "1" if on else "0"
                    patch.install()
                    cfg = harness.load_cfg(root, stage=stage, src_res=1024, num_steps=n_steps + 1, batch_size=bs)
                    st = (harness.Stage1State if stage == 1 else harness.C3State)(cfg)
                    data = st.batch(0)
                    step = (lambda: harness.stage1_step(st, data)) if stage == 1 else (lambda: harness.c3_step(st, data))
                    step()
                    torch.cuda.synchronize()
                    torch.cuda.reset_peak_memory_stats()
                    t0 = time.perf_counter()
                    for _ in range(n_steps):
                        step()
                    torch.cuda.synchronize()
                    ms = (time.perf_counter() - t0) / n_steps * 1e3
                    r = res.setdefault(f"stage{stage}_bs{bs}", {}).setdefault("on" if on else "off", {"step_ms": []})
                    r["step_ms"].append(round(ms, 2))
                    r["peak_GiB"] = round(torch.cuda.max_memory_allocated() / 2 ** 30, 2)
                    del st, data
                    torch.cuda.empty_cache()
        patch.uninstall()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--no-steps", action="store_true")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("flow_head_time.py needs a CUDA device")
    if harness.staged_reference() is None:
        raise SystemExit("oracle/_ref is not staged: the op chain to compare against is the reference's own")
    out = {"gpu": _gpu_info(), "datasheet_hbm_TBps": DATASHEET_BW / 1e12, "upsample": _upsample(a.iters),
           "sequence_loss": _seq_loss(a.iters)}
    if not a.no_steps:
        out["steps"] = _steps(a.steps)
    s = json.dumps(out)
    print(s)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "flow_head_time.json"), "w") as f:
            f.write(s + "\n")


if __name__ == "__main__":
    main()
