"""Per-frame time of the real-data loader's rectification, CPU (the reference's own functions) against the GPU route.

    python tools/rectify_time.py [--res 1024] [--iters 10] [--out DIR]

Needs a CUDA device, cv2 and the staged reference (oracle/_ref).  On one synthetic 1024^2 stereo pair it reports, as
the mean over --iters calls:
  cpu_rectify_ms[threads]  StereoHumanDataset.get_rectified_stereo_data (no pts, as get_test_item calls it) at cv2
                           thread counts 1 and os.cpu_count();
  cpu_to_tensor_ms         stereo_to_dict_tensor;
  gpu_upload_ms            the two images and two masks from pageable numpy to the device;
  gpu_kernel_ms            gpsg_rectify_remap (numpy + tensor outputs) on device-resident inputs, CUDA events;
  gpu_download_ms          the numpy contract (two images, two masks) back to the host;
  get_test_item_ms         the whole get_test_item, original and with GPSG_RECTIFY's rebinding;
  cache_samples_per_s      rectified_local/ generation (StereoHumanDataset with use_processed_data=True, pts and
                           flow included), original and rebound.
Prints one JSON object (also written to DIR/rectify_time.json with --out) with the GPU name and power limit."""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from gps_gaussian_b200 import harness, patch, rectify  # noqa: E402
import rectify_cases  # noqa: E402


def _mean_ms(fn, iters, sync=False):
    fn()
    if sync:
        torch.cuda.synchronize()
    t = time.perf_counter()
    for _ in range(iters):
        fn()
    if sync:
        torch.cuda.synchronize()
    return (time.perf_counter() - t) * 1e3 / iters


def _event_ms(fn, iters):
    fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / iters


def _gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception:
        q = torch.cuda.get_device_name()
    return q


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--res", type=int, default=1024)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--samples", type=int, default=2)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import cv2
    harness.add_reference_to_path()
    from lib import human_loader as hl
    S, it = a.res, a.iters
    r = {"gpu": _gpu_info(), "host_cpus": os.cpu_count(), "res": S, "iters": it, "cv2": cv2.__version__}
    views = rectify_cases.pair(5, S, S)
    data = [(img, mask, K, E, None) for img, mask, K, E in views]
    me = types.SimpleNamespace(opt=types.SimpleNamespace(src_res=S))
    orig_rect = hl.StereoHumanDataset.get_rectified_stereo_data
    r["cpu_rectify_ms"] = {}
    for th in (1, os.cpu_count()):
        cv2.setNumThreads(th)
        r["cpu_rectify_ms"][th] = _mean_ms(lambda: orig_rect(me, data[0], data[1]), it)
    cv2.setNumThreads(os.cpu_count())
    st = orig_rect(me, data[0], data[1])
    r["cpu_to_tensor_ms"] = _mean_ms(lambda: hl.StereoHumanDataset.stereo_to_dict_tensor(me, st, "s"), it)

    arrays = [views[k][j] for k in range(2) for j in range(2)]
    r["gpu_upload_ms"] = _mean_ms(lambda: [torch.from_numpy(x).cuda() for x in arrays], it, sync=True)
    dev = [torch.from_numpy(x).cuda() for x in arrays]
    _, cams = rectify.stereo_rectify(data[0], data[1], S)
    run = lambda: rectify.rectify_device([(dev[0], dev[1]), (dev[2], dev[3])], cams, S, numpy_out=True, tensor_out=True)
    r["gpu_kernel_ms"] = _event_ms(run, max(it, 50))
    out = run()
    r["gpu_download_ms"] = _mean_ms(lambda: [o[k].cpu().numpy() for o in out for k in ("img", "mask")], it, sync=True)
    r["gpu_rectify_stereo_ms"] = _mean_ms(lambda: rectify.rectify_stereo(data[0], data[1], S), it, sync=True)
    r["gpu_stereo_item_cuda_ms"] = _mean_ms(lambda: rectify.stereo_item_cuda(data[0], data[1], S, "s"), it, sync=True)

    from gps_gaussian_b200 import synth_dataset
    tmp = tempfile.mkdtemp(prefix="rectify_time_")
    try:
        root = os.path.join(tmp, "data")
        synth_dataset.write_dataset(root, n_train=a.samples, n_val=1, res=S, hr=False)
        cfg = harness.load_cfg(root, src_res=S, use_processed_data=False)
        cfg.defrost()
        cfg.dataset.test_data_root = os.path.join(root, "val")
        cfg.freeze()
        ds = hl.StereoHumanDataset(cfg.dataset, phase="test")
        r["get_test_item_ms"] = {"cpu": _mean_ms(lambda: ds.get_test_item(0, [0, 1]), it)}
        cache = {}
        for on in (False, True):
            patch.uninstall()
            if on:
                os.environ["GPSG_RECTIFY"] = "1"
                patch.install()
                r["get_test_item_ms"]["gpu"] = _mean_ms(lambda: ds.get_test_item(0, [0, 1]), it, sync=True)
            croot = os.path.join(tmp, f"cache{int(on)}")
            shutil.copytree(root, croot)
            ccfg = harness.load_cfg(croot, src_res=S, use_processed_data=True)
            t = time.perf_counter()
            hl.StereoHumanDataset(ccfg.dataset, phase="train")
            torch.cuda.synchronize()
            cache["gpu" if on else "cpu"] = a.samples / (time.perf_counter() - t)
        patch.uninstall()
        r["cache_samples_per_s"] = cache
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    line = json.dumps(r)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "rectify_time.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
