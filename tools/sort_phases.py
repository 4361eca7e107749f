#!/usr/bin/env python
"""Where the tile sort's time goes, per phase, on the C2 scene:  python tools/sort_phases.py [--reps 20] [--seeds ...]

Builds the library once more with GPSG_SORT_PHASES (raster_binning.cu), into lib/libgpsg_sm90_sortphases.so, and runs the
sync-free planned forward (the one bench.py measures) on it.  In that build thread 0 of every tile-sort CTA adds the
%globaltimer time between CTA barriers to one counter per phase.  Printed per phase: microseconds of one CTA per tile it
sorted (the CTA's 16 warps wait out each phase together), the tiles per view, and the GPU's name and power limit.  The
instrumented kernel runs a little slower than the normal one; compare phases with each other, and time the kernel itself
with tools/stage_times.py."""
import argparse
import ctypes
import importlib.util
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PHASES = ("ticket_range", "load_minmax", "ordering", "fixup_fallback", "gather", "lists")

ap = argparse.ArgumentParser()
ap.add_argument("--reps", type=int, default=20)
ap.add_argument("--res", type=int, default=1024)
ap.add_argument("--seeds", type=int, nargs="*", default=[1314, 1315, 1316, 1317])
a = ap.parse_args()

spec = importlib.util.spec_from_file_location("_gpsg_build", os.path.join(ROOT, "gps-gaussian_b200", "build.py"))
build = importlib.util.module_from_spec(spec)
spec.loader.exec_module(build)
os.environ["GPSG_LIB_PATH"] = build.build(defines=["GPSG_SORT_PHASES"],
                                          out=os.path.join(build.LIBDIR, "libgpsg_sm90_sortphases.so"))

sys.path.insert(0, ROOT)
import torch  # noqa: E402
from gps_gaussian_b200 import _lib, synth  # noqa: E402
from gps_gaussian_b200.introspect import make_settings, to_device  # noqa: E402
from gps_gaussian_b200.planned import PlannedRasterizer  # noqa: E402

read = _lib.lib.gpsg_sort_phases_read
read.restype, read.argtypes = ctypes.c_int, [ctypes.POINTER(ctypes.c_ulonglong)]
words = (ctypes.c_ulonglong * 8)()


def read_phases():
    if read(words) != 0:
        raise _lib.GpsgError(_lib.lib.gpsg_last_error().decode())
    return np.array(words[:], dtype=np.float64)


dev = torch.device("cuda", 0)
views = []
for s in a.seeds:
    sc = synth.stereo_pair_scene(a.res, seed=s)
    inp = to_device(sc, dev)
    views.append((make_settings(sc), inp, PlannedRasterizer(int(inp["means3D"].shape[0]), sc["H"], sc["W"], 1 << 22,
                                                              device=dev)))   # C2 makes ~1.3 M pairs


def forward_all():
    for st, i, r in views:
        r.forward(st, i["means3D"], i["colors"], i["opacity"], i["scales"], i["rots"])


forward_all()
torch.cuda.synchronize()
read_phases()
for _ in range(a.reps):
    forward_all()
torch.cuda.synchronize()
ns = read_phases()
assert all(r.ok() for _, _, r in views), "pair capacity exceeded: the planned forward sorted nothing"
tiles = ns[6]
out = {p: round(ns[k] / tiles / 1e3, 2) for k, p in enumerate(PHASES)}
out["per_tile_us"] = round(ns[:6].sum() / tiles / 1e3, 2)
out["tiles_per_view"] = tiles / (a.reps * len(views))
out["gpu"] = torch.cuda.get_device_name(0)
out["power_limit"] = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                                    capture_output=True, text=True).stdout.strip()
print(json.dumps(out))
