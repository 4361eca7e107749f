"""Time JPEG decoding: Pillow against the GPU route (gps_gaussian_b200.jpeg), and the whole get_test_item with and without
GPSG_DECODE=1 (both with GPSG_RECTIFY=1).

    python tools/jpeg_time.py [--iters 20] [--out DIR]

Per image, at 1024^2 and 2048^2 q95 4:2:0 (the loader's format):
  pillow_ms      file read + np.array(Image.open(f)), host clock
  gpu_e2e_ms     file read + parse + upload + decode + the status read (jpeg.read_img_cuda), host clock
  gpu_kernel_ms  one gpsg_jpeg_decode launch chain on data already on the device, CUDA events
  pair_*         the same for the two source views of a pair decoded in one call
Outputs are checked equal to Pillow's before timing.  Prints one JSON object (also written to DIR/jpeg_time.json with
--out) with the GPU name and power limit."""
import argparse
import ctypes as C
import io
import json
import os
import subprocess
import sys
import tempfile
import shutil
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from gps_gaussian_b200 import _lib, harness, jpeg, patch  # noqa: E402


def _ms(fn, iters, sync=True):
    fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        t = time.perf_counter()
        fn()
        if sync:
            torch.cuda.synchronize()
        ts.append((time.perf_counter() - t) * 1e3)
    return {"median": float(np.median(ts)), "min": float(np.min(ts)), "max": float(np.max(ts))}


def _gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                              text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception:
        return torch.cuda.get_device_name()


def _kernel_call(datas):
    """A closure running gpsg_jpeg_decode on device-resident data with preallocated outputs and workspace."""
    infos = [jpeg.parse(d)[1] for d in datas]
    n = len(datas)
    arr = (jpeg.JpegInfo * n)(*infos)
    blob = torch.from_numpy(np.frombuffer(b"".join(datas), np.uint8).copy()).cuda()
    offs = np.cumsum([0] + [len(d) for d in datas])
    outs = [torch.empty((i.height, i.width, 3), dtype=torch.uint8, device="cuda") for i in infos]
    status = torch.empty(n, dtype=torch.int32, device="cuda")
    wsb = jpeg._L.gpsg_jpeg_decode_workspace_bytes(n, arr)
    ws = torch.empty(wsb + 256, dtype=torch.uint8, device="cuda")
    base = (ws.data_ptr() + 255) // 256 * 256
    dp = (C.c_void_p * n)(*[blob.data_ptr() + int(o) for o in offs[:-1]])
    op = (C.c_void_p * n)(*[o.data_ptr() for o in outs])
    idx, stream = _lib.device_stream(torch.device("cuda"))

    def run():
        _lib.check(jpeg._L.gpsg_jpeg_decode(idx, stream, n, arr, dp, op, status.data_ptr(), base, wsb), "decode")
    return run, outs, status


def _events(fn, iters):
    fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    from PIL import Image
    import importlib.util
    spec = importlib.util.spec_from_file_location("mk", os.path.join(ROOT, "tests", "golden", "make_jpeg_corpus.py"))
    mk = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mk)
    it = a.iters
    r = {"gpu": _gpu_info(), "host_cpus": os.cpu_count(), "iters": it}
    tmp = tempfile.mkdtemp(prefix="jpeg_time_")
    try:
        for S in (1024, 2048):
            paths = []
            for k in range(2):
                p = os.path.join(tmp, f"{S}_{k}.jpg")
                with open(p, "wb") as f:
                    f.write(mk._pil(mk._smooth(S, S, 40 + k), quality=95))
                paths.append(p)
            datas = [open(p, "rb").read() for p in paths]
            want = [np.array(Image.open(p)) for p in paths]
            got = [jpeg.read_img_cuda(p).cpu().numpy() for p in paths]
            assert all(np.array_equal(g, w) for g, w in zip(got, want)), "GPU decode differs from Pillow"
            row = {"bytes": len(datas[0])}
            row["pillow_ms"] = _ms(lambda: np.array(Image.open(paths[0])), it, sync=False)
            row["gpu_e2e_ms"] = _ms(lambda: jpeg.read_img_cuda(paths[0]), it)
            run, _, _ = _kernel_call(datas[:1])
            row["gpu_kernel_ms"] = _events(run, max(it, 50))
            row["pair_pillow_ms"] = _ms(lambda: [np.array(Image.open(p)) for p in paths], it, sync=False)

            def pair_gpu():
                bs = []
                for p in paths:
                    with open(p, "rb") as f:
                        bs.append(f.read())
                jpeg.decode(bs)
            row["pair_gpu_e2e_ms"] = _ms(pair_gpu, it)
            run2, outs, st = _kernel_call(datas)
            row["pair_gpu_kernel_ms"] = _events(run2, max(it, 50))
            torch.cuda.synchronize()
            assert not st.any() and all(np.array_equal(o.cpu().numpy(), w) for o, w in zip(outs, want))
            r[f"{S}"] = row

        harness.add_reference_to_path()
        from lib import human_loader as hl
        from gps_gaussian_b200 import synth_dataset
        root = os.path.join(tmp, "data")
        synth_dataset.write_dataset(root, n_train=1, n_val=1, res=1024, hr=False)
        cfg = harness.load_cfg(root, src_res=1024, use_processed_data=False)
        cfg.defrost()
        cfg.dataset.test_data_root = os.path.join(root, "val")
        cfg.freeze()
        ds = hl.StereoHumanDataset(cfg.dataset, phase="test")
        gti = {}
        os.environ["GPSG_RECTIFY"] = "1"
        for on in (False, True, False, True):                 # alternated, so drift shows as a spread
            patch.uninstall()
            os.environ["GPSG_DECODE"] = "1" if on else "0"
            patch.install()
            t = _ms(lambda: ds.get_test_item(0, [0, 1]), it)
            gti.setdefault("decode" if on else "pillow", []).append(t["median"])
        patch.uninstall()
        r["get_test_item_1024_median_ms"] = gti
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    line = json.dumps(r)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "jpeg_time.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
