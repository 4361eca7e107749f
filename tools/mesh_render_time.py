"""Per-scan wall time of the dataset renderer (prepare_data/render_data.py through the `taichi_three` stand-in), split into
its stages, on a seeded procedural scan.

    python tools/mesh_render_time.py [--faces 300000] [--tex 2048] [--renders 16] [--seed 0]

A scan of render_data.py is 16 x 5 = 80 `scene.render()` calls, each drawing the 1024^2 camera and the 2048^2 `hr`
camera.  Per stage, this prints the time of one occurrence and the per-scan total it implies:
  readobj   the stand-in's `readobj` of the scan's OBJ (once per scan)
  upload    `StaticModel._init()`: the padded arrays and the fp32 texture to the GPU (once per scan)
  render    `scene.render()` of both cameras, CUDA events around it (80 per scan)
  readback  the four `to_numpy()` reads the script makes per view: zbuf, img, mask at 1024^2 and img at 2048^2
            (80 per scan; the hr image is read for 3 of 5 views, counted for all here)
  encode    `render_data.save`'s cv2 writes: depth PNG, JPEG, mask PNG, and the 2048^2 JPEG for 3 of 5 views
            (80 per scan)
and one render of the 1024^2 camera by the serial CPU oracle (oracle/mesh_oracle.c) for scale.  One JSON line per
measurement, then a summary line, with the card name and its power limit.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "gps-gaussian_b200", "dropin"), os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)


def _card():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        limit = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                               capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        limit = "unknown"
    return name, limit


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--faces", type=int, default=300_000)
    ap.add_argument("--tex", type=int, default=2048)
    ap.add_argument("--renders", type=int, default=16)
    ap.add_argument("--seed", type=int, default=0)
    a = ap.parse_args()

    import cv2
    import torch
    import taichi_three as t3
    import mesh_reference as mr
    from gps_gaussian_b200 import synth_mesh

    card, limit = _card()
    tmp = tempfile.mkdtemp(prefix="mesh_render_time_")
    obj, tex_img = synth_mesh.procedural_scan(a.faces, a.tex, seed=a.seed)
    synth_mesh.write_obj(os.path.join(tmp, "scan.obj"), obj)
    cv2.imwrite(os.path.join(tmp, "material0.jpeg"), tex_img)
    texture = np.ascontiguousarray(cv2.imread(os.path.join(tmp, "material0.jpeg"))[:, :, ::-1]).swapaxes(0, 1)[:, ::-1, :]

    t0 = time.perf_counter()
    obj = t3.readobj(os.path.join(tmp, "scan.obj"), scale=1)
    t_readobj = time.perf_counter() - t0
    n_cap = 2 * max(len(obj["vi"]), len(obj["f"]), len(obj["vt"]))

    scene = t3.Scene()
    model = t3.StaticModel(n_cap, obj=obj, tex=texture)
    scene.add_model(model)
    cams = [t3.Camera(res=(1024, 1024)), t3.Camera(res=(2048, 2048))]
    for c in cams:
        scene.add_camera(c)
    ld, _ = mr.lights(seed=a.seed)
    scene.add_lights(t3.Lights([t3.Light([-float(x) for x in d], color=[1.0, 1.0, 1.0]) for d in ld]))
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    model._init()
    torch.cuda.synchronize()
    t_upload = time.perf_counter() - t0
    model._t3_initialised = True

    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    renders, reads, encodes = [], [], []
    for k in range(a.renders + 2):                  # the first two renders warm up
        ang = 360.0 * k / max(1, a.renders)
        for cam, ref in zip(cams, (mr.ring_camera(ang), mr.ring_camera(ang, hr=True))):
            cam.set_intrinsic(*ref._dev_K)
            cam.set(pos=ref.eye, target=ref.target)
            cam._init()
        torch.cuda.synchronize()
        ev0.record()
        scene.render()
        ev1.record()
        torch.cuda.synchronize()
        t_render = ev0.elapsed_time(ev1) / 1e3
        t0 = time.perf_counter()
        depth = cams[0].zbuf.to_numpy().swapaxes(0, 1)
        img = cams[0].img.to_numpy().swapaxes(0, 1)
        mask = cams[0].mask.to_numpy().swapaxes(0, 1)
        img_hr = cams[1].img.to_numpy().swapaxes(0, 1)
        t_read = time.perf_counter() - t0
        t0 = time.perf_counter()
        cv2.imwrite(os.path.join(tmp, "d.png"), (depth * 2.0 ** 15).astype(np.uint16))
        cv2.imwrite(os.path.join(tmp, "i.jpg"), (np.clip(img, 0, 1) * 255.0 + 0.5).astype(np.uint8)[:, :, ::-1])
        cv2.imwrite(os.path.join(tmp, "m.png"), (np.clip(mask, 0, 1) * 255.0 + 0.5).astype(np.uint8))
        t_enc = time.perf_counter() - t0
        t0 = time.perf_counter()
        cv2.imwrite(os.path.join(tmp, "h.jpg"), (np.clip(img_hr, 0, 1) * 255.0 + 0.5).astype(np.uint8)[:, :, ::-1])
        t_enc_hr = time.perf_counter() - t0
        if k >= 2:
            renders.append(t_render)
            reads.append(t_read)
            encodes.append(t_enc + 0.6 * t_enc_hr)
            print(json.dumps({"render_ms": round(t_render * 1e3, 3), "readback_ms": round(t_read * 1e3, 2),
                              "encode_ms": round((t_enc + 0.6 * t_enc_hr) * 1e3, 2),
                              "covered_px_1024": int((mask[..., 0] > 0).sum())}))

    cam0 = cams[0]
    m = model.render_inputs()
    t0 = time.perf_counter()
    mr.oracle_render(cam0, scene.lights.light_dirs, scene.lights.light_colors, obj["vi"], obj["f"][:, :, 0], obj["vt"],
                     obj["f"][:, :, 1], m["tex"].cpu().numpy())
    t_oracle = time.perf_counter() - t0

    med = lambda v: float(np.median(v))
    per_scan = {"readobj": t_readobj, "upload": t_upload, "render": 80 * med(renders), "readback": 80 * med(reads),
                "encode": 80 * med(encodes)}
    total = sum(per_scan.values())
    print(json.dumps({
        "card": card, "power_limit": limit, "faces": int(len(obj["f"])), "tex": a.tex, "renders_timed": len(renders),
        "render_ms_median": round(med(renders) * 1e3, 3), "render_ms_min": round(min(renders) * 1e3, 3),
        "readback_ms_median": round(med(reads) * 1e3, 2), "encode_ms_median": round(med(encodes) * 1e3, 2),
        "readobj_s": round(t_readobj, 3), "upload_s": round(t_upload, 3),
        "per_scan_s": {k: round(v, 3) for k, v in per_scan.items()}, "per_scan_total_s": round(total, 3),
        "dominant": max(per_scan, key=per_scan.get), "cpu_oracle_1024_s": round(t_oracle, 3)}))


if __name__ == "__main__":
    main()
