#!/usr/bin/env python
"""Per-kernel times of the rasterizer forward + backward on the C2 scene (CUDA events around each launch, serialised on
one stream) -- the quick loop used while tuning kernels:  python tools/stage_times.py [--reps 50] [--seeds 1314 1315]
--deterministic times the deterministic backward (GPSG_BWD_DETERMINISTIC: render_backward_det, render_backward_det_reduce)
instead of the default one and adds its workspace bytes per view.  --aux times aux mode (depth and alpha outputs, and the
backward of all three images) under the same stage names.  --alternate R runs R rounds that alternate default and aux
(same scenes, same process) and prints one line per round and mode.  --antialias times the anti-aliased forward and
backward (GPSG_FWD_ANTIALIAS); with --alternate R the rounds then alternate AA off and on instead.  --empty moves every
Gaussian of the scenes far outside the view and times the sync-free planned forward (the one bench.py measures; the exact
entry point launches no tile sort for an image without pairs): what tile_sort_gather and render_forward cost for empty
tiles alone.  Each line carries the GPU's name and power limit."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from gps_gaussian_b200 import _lib, synth  # noqa: E402
from gps_gaussian_b200.introspect import RasterCall, make_settings, to_device  # noqa: E402
from gps_gaussian_b200.planned import PlannedRasterizer  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--reps", type=int, default=50)
ap.add_argument("--res", type=int, default=1024)
ap.add_argument("--seeds", type=int, nargs="*", default=[1314, 1315, 1316, 1317])
ap.add_argument("--no-backward", action="store_true")
ap.add_argument("--deterministic", action="store_true")
ap.add_argument("--aux", action="store_true")
ap.add_argument("--alternate", type=int, default=0)
ap.add_argument("--antialias", action="store_true")
ap.add_argument("--empty", action="store_true")
a = ap.parse_args()
dev = torch.device("cuda", 0)
scenes = [synth.stereo_pair_scene(a.res, seed=s) for s in a.seeds]
if a.empty:   # every Gaussian 10^4 units away: no pair, every tile empty
    scenes = [dict(sc, means3D=(sc["means3D"] + np.float32(1e4)).astype(np.float32)) for sc in scenes]
calls = [RasterCall(sc, to_device(sc, dev), dev) for sc in scenes]
g = torch.randn(3, a.res, a.res, device=dev)
gD, gA = torch.randn(a.res, a.res, device=dev), torch.randn(a.res, a.res, device=dev)
depth, alpha = torch.empty(a.res, a.res, device=dev), torch.empty(a.res, a.res, device=dev)


def power_limit():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        return "unknown"


POWER = power_limit()


class PlannedCall:
    """The planned forward of one scene, in RasterCall's shape (forward only)."""

    def __init__(self, sc, inp):
        self.sc, self.inp, self.settings = sc, inp, make_settings(sc)
        self.P, self.num_rendered, self.antialiasing = int(inp["means3D"].shape[0]), 0, False
        self.r = PlannedRasterizer(self.P, sc["H"], sc["W"], 1 << 20, device=dev)

    def forward(self, depth=None, alpha=None):
        i = self.inp
        self.r.forward(self.settings, i["means3D"], i["colors"], i["opacity"], i["scales"], i["rots"], depth=depth,
                       alpha=alpha, antialiasing=self.antialiasing)


if a.empty:
    if a.alternate or not a.no_backward:
        ap.error("--empty times the planned forward alone: pass --no-backward, not --alternate")
    calls = [PlannedCall(c.sc, c.inp) for c in calls]


def step(c, aux, aa=False):
    c.antialiasing = aa
    c.forward(*((depth, alpha) if aux else (None, None)))
    if not a.no_backward:
        c.backward(g, deterministic=a.deterministic, **(dict(grad_depth=gD, grad_alpha=gA) if aux else {}))


def run(aux, aa=False):
    for c in calls:
        step(c, aux, aa)
    torch.cuda.synchronize()
    _lib.profile_enable(True)
    _lib.profile_read()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(a.reps):
        for c in calls:
            step(c, aux, aa)
    e1.record()
    torch.cuda.synchronize()
    prof = _lib.profile_read()
    _lib.profile_enable(False)
    out = {k: round(v["ms"] / max(v["calls"], 1) * 1e3, 1) for k, v in prof.items() if v["calls"]}
    out["total_us_per_view"] = round(e0.elapsed_time(e1) * 1e3 / (a.reps * len(calls)), 1)
    out["N_dup_mean"] = sum(c.num_rendered for c in calls) / len(calls)
    flags = _lib.BWD_DETERMINISTIC if a.deterministic else 0
    size = _lib.lib.gpsg_rasterize_backward_workspace_bytes
    out["bwd_workspace_bytes_mean"] = sum(size(c.P, c.num_rendered, flags, int(aux)) for c in calls) / len(calls)
    out["aux"] = aux
    out["empty"] = a.empty
    out["antialias"] = aa
    out["gpu"] = torch.cuda.get_device_name(0)
    out["power_limit"] = POWER
    return out


if a.alternate and a.antialias:
    for r in range(a.alternate):
        for aa in (False, True):
            print(json.dumps(dict(run(a.aux, aa), round=r)))
elif a.alternate:
    for r in range(a.alternate):
        for aux in (False, True):
            print(json.dumps(dict(run(aux), round=r)))
else:
    print(json.dumps(run(a.aux, a.antialias)))
