"""Time JPEG encoding: cv2.imwrite against the GPSG_ENCODE route (gps_gaussian_b200.jpeg, csrc/jpeg_encode.cu), and the
per-view writes of the unmodified dataset renderer and the per-frame time of the unmodified inference scripts, with and
without GPSG_ENCODE=1.

    python tools/jpeg_encode_time.py [--iters 20] [--out DIR] [--no-render] [--no-inference]

Per image, q95 4:2:0 (cv2's default) of a photo-like BGR frame, at sizes 64^2 .. 2048^2:
  cv2_ms        cv2.imwrite on the host clock (cv2's own threads)
  gpu_ms        the rebound cv2.imwrite: pinned upload + launch chain + size read + download + file write, host clock
  kernel_ms     one gpsg_jpeg_encode launch chain on a device-resident image, CUDA events
Files are checked byte-identical before timing.  render_data.py (the test_mesh_render_gpu scan tree) is run once with and
once without the switch; every cv2.imwrite call is timed per extension inside the script.  test_real_data.py and
test_view_interp.py run on a synthetic 1024^2 dataset with a seeded untrained checkpoint (GPSG_RECTIFY=1 both ways), with
the same per-call timing and the script's wall time per written frame.  Prints one JSON object (also
written to DIR/jpeg_encode_time.json with --out) with the GPU name and power limit."""
import argparse
import ctypes as C
import importlib.util
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from gps_gaussian_b200 import _lib, harness, jpeg, patch  # noqa: E402


def _stats(ts):
    return {"median": float(np.median(ts)), "min": float(np.min(ts)), "max": float(np.max(ts))}


def _gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                              text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception:
        return torch.cuda.get_device_name()


def _frame(n, seed=0):
    """A rendered-view-like BGR frame: smooth shading, a textured disc, a little noise."""
    path = os.path.join(ROOT, "tests", "golden", "jpeg_encode", "make_jpeg_encode_corpus.py")
    spec = importlib.util.spec_from_file_location("make_jpeg_encode_corpus", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod.smooth(n, n, "420", seed)


def _kernel_ms(img, iters):
    t = torch.from_numpy(img).cuda()
    d = jpeg.JpegEncodeDesc(img.shape[1], img.shape[0], 3, jpeg.ORDERS["bgr"], 95, 420, img.shape[1] * 3)
    arr = (jpeg.JpegEncodeDesc * 1)(d)
    out = torch.empty(int(jpeg._L.gpsg_jpeg_encode_max_bytes(C.byref(d))), dtype=torch.uint8, device="cuda")
    sizes = torch.empty(1, dtype=torch.int64, device="cuda")
    wsb = int(jpeg._L.gpsg_jpeg_encode_workspace_bytes(1, arr))
    ws = torch.empty(wsb + 256, dtype=torch.uint8, device="cuda")
    base = (ws.data_ptr() + 255) // 256 * 256
    src_p, out_p = (C.c_void_p * 1)(t.data_ptr()), (C.c_void_p * 1)(out.data_ptr())
    idx, stream = _lib.device_stream(torch.device("cuda"))

    def call():
        _lib.check(jpeg._L.gpsg_jpeg_encode(idx, stream, 1, arr, src_p, out_p, sizes.data_ptr(), base, wsb), "encode")
    call()
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        call()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    return _stats(ts)


def _per_image(iters):
    import cv2
    os.environ["GPSG_ENCODE"] = "1"
    patch.install()
    orig = cv2.imwrite._gpsg_original
    routed = cv2.imwrite
    saved = patch._MIN_NATIVE_PIXELS
    patch._MIN_NATIVE_PIXELS = 0                  # time the GPU route at every size, the threshold's own evidence
    res = {}
    with tempfile.TemporaryDirectory() as tmp:
        fa, fb = os.path.join(tmp, "a.jpg"), os.path.join(tmp, "b.jpg")
        for n in (64, 128, 256, 512, 1024, 2048):
            img = _frame(n)[:, :, ::-1]               # render_data.py's negative-stride view
            orig(fa, img)
            routed(fb, img)
            assert open(fa, "rb").read() == open(fb, "rb").read(), n
            tc, tg = [], []
            for _ in range(iters):                    # alternate the two routes
                t = time.perf_counter()
                orig(fa, img)
                tc.append((time.perf_counter() - t) * 1e3)
                t = time.perf_counter()
                routed(fb, img)
                tg.append((time.perf_counter() - t) * 1e3)
            res[f"{n}x{n}"] = {"cv2_ms": _stats(tc), "gpu_ms": _stats(tg),
                               "kernel_ms": _kernel_ms(np.ascontiguousarray(img), iters),
                               "file_bytes": os.path.getsize(fa)}
    patch._MIN_NATIVE_PIXELS = saved
    patch.uninstall()
    return res


_TIMER = ("import os, runpy, sys, time, json\n"
          "sys.argv = sys.argv[1:]\nsys.path.insert(0, os.path.dirname(sys.argv[0]))\n"
          "import cv2\n"
          "_w, _acc = cv2.imwrite, {}\n"
          "def _timed(f, *a, **k):\n"
          "    t = time.perf_counter(); r = _w(f, *a, **k)\n"
          "    e = os.path.splitext(f)[1]; s = _acc.setdefault(e, [0, 0.0]); s[0] += 1; s[1] += time.perf_counter() - t\n"
          "    return r\n"
          "cv2.imwrite = _timed\n"
          "t0 = time.perf_counter()\n"
          "runpy.run_path(sys.argv[0], run_name='__main__')\n"
          "print('TIMES', json.dumps({'total_s': time.perf_counter() - t0, 'writes': _acc}))\n")


def _render_data():
    if harness.staged_reference() is None:
        return "not measured (oracle/_ref not staged)"
    sys.path.insert(0, os.path.join(ROOT, "tests"))          # test_mesh_render_gpu imports its helpers from there
    spec = importlib.util.spec_from_file_location("_mr", os.path.join(ROOT, "tests", "test_mesh_render_gpu.py"))
    mr = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mr)
    script = os.path.join(harness.staged_reference(), "prepare_data", "render_data.py")
    out = {}
    for on in (False, True):
        with tempfile.TemporaryDirectory() as work:
            mr._scan_tree(work)
            env = harness.script_env(patch=True)
            env.pop("GPSG_ENCODE", None)
            if on:
                env["GPSG_ENCODE"] = "1"
            p = subprocess.run([sys.executable, "-c", _TIMER, script], cwd=work, env=env, text=True,
                               capture_output=True, timeout=3600)
            if p.returncode:
                raise RuntimeError(p.stderr[-4000:])
            r = json.loads([ln for ln in p.stdout.splitlines() if ln.startswith("TIMES")][-1].split(" ", 1)[1])
        views = 2 * 16 * 5
        out["encode_on" if on else "encode_off"] = {
            "total_s": r["total_s"],
            "per_view_ms": {ext: 1e3 * s / views for ext, (n, s) in r["writes"].items()},
            "calls": {ext: n for ext, (n, s) in r["writes"].items()}}
    return out


def _inference():
    if harness.staged_reference() is None:
        return "not measured (oracle/_ref not staged)"
    from gps_gaussian_b200 import synth_dataset
    res = 1024
    out = {}
    with tempfile.TemporaryDirectory() as tmp:
        data = os.path.join(tmp, "data")
        synth_dataset.write_dataset(data, n_train=1, n_val=2, res=res, hr=False)
        cfg = harness.load_cfg(data, src_res=res)
        from lib.network import RtStereoHumanModel
        torch.manual_seed(7)
        ckpt = os.path.join(tmp, "init.pth")
        torch.save({"network": RtStereoHumanModel(cfg, with_gs_render=True).state_dict()}, ckpt)
        # the scripts run from the working copy's root (cwd first on sys.path); their DataLoader iterators are shut down
        # before the interpreter exits, as harness.SCRIPT_RUNNER does
        runner = (_TIMER.replace("sys.path.insert(0, os.path.dirname(sys.argv[0]))\n", "") +
                  "import gc\nfrom torch.utils.data.dataloader import _MultiProcessingDataLoaderIter\n"
                  "for o in gc.get_objects():\n    if isinstance(o, _MultiProcessingDataLoaderIter):\n"
                  "        o._shutdown_workers()\n")
        for script in ("test_real_data.py", "test_view_interp.py"):
            args = ["--test_data_root", os.path.join(data, "val"), "--ckpt_path", ckpt]
            args += ["--src_view", "0", "1"] if script == "test_real_data.py" else ["--novel_view_nums", "4"]
            for on in (False, True):
                work = harness.make_workdir(os.path.join(tmp, f"{script}_{int(on)}"), data, src_res=res)
                env = harness.script_env(patch=True, extra={"GPSG_RECTIFY": "1"})
                env.pop("GPSG_ENCODE", None)
                if on:
                    env["GPSG_ENCODE"] = "1"
                p = subprocess.run([sys.executable, "-c", runner, script] + args, cwd=work, env=env, text=True,
                                   capture_output=True, timeout=1800)
                if p.returncode:
                    raise RuntimeError(p.stderr[-4000:])
                r = json.loads([ln for ln in p.stdout.splitlines() if ln.startswith("TIMES")][-1].split(" ", 1)[1])
                n, t = r["writes"].get(".jpg", [0, 0.0])
                out.setdefault(script, {})["encode_on" if on else "encode_off"] = {
                    "frames": n, "script_s": r["total_s"], "script_ms_per_frame": 1e3 * r["total_s"] / max(n, 1),
                    "jpeg_write_ms_per_frame": 1e3 * t / max(n, 1)}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--out", default=None)
    ap.add_argument("--no-render", action="store_true")
    ap.add_argument("--no-inference", action="store_true")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("jpeg_encode_time.py needs a CUDA device")
    import cv2
    res = {"gpu": _gpu_info(), "cv2": cv2.__version__, "cv2_threads": cv2.getNumThreads(),
           "per_image_q95_420": _per_image(a.iters)}
    res["render_data"] = "not measured (--no-render)" if a.no_render else _render_data()
    res["inference_scripts"] = "not measured (--no-inference)" if a.no_inference else _inference()
    s = json.dumps(res, indent=1)
    print(s)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "jpeg_encode_time.json"), "w") as f:
            f.write(s + "\n")


if __name__ == "__main__":
    main()
