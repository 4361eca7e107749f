#!/usr/bin/env python
"""CPU count of the compositing forward's work on one scene, from the independent numpy restatement of the rasterizer
(oracle/raster_independent.py) and the kernels' own cull box and block layout -- the counts the per-block survivor lists
(raster_binning.cu: build_block_lists, raster_render.cu) were designed from.  No GPU, no timing:

    python tools/forward_work.py [--res 1024] [--seed 1314]

Prints one JSON line: pairs, tiles and empty tiles, tile-length distribution, entries a warp block scans and keeps
(survivors), where a block's last contribution sits in its tile list, and the spread of the blocks' stop positions inside
a 2-block (8x8) and a 4-block (16x8) CTA.  The cull box is restated in fp32 numpy (np.log for __logf), so a survivor
count may differ from the device's by an entry whose box touches a block edge to within an ulp."""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from gps_gaussian_b200 import synth  # noqa: E402
from oracle import raster_independent as ri  # noqa: E402


def cull_box(conic, opacity):
    """slab_entry (raster_binning.cu): half-extents of the region where o*exp(power) can reach 1/255."""
    f = np.float32
    a, b, c = (conic[:, k].astype(f) for k in range(3))
    o = opacity.astype(f)
    ex = np.full(o.shape, f(3.0e38))
    ey = ex.copy()
    det = a * c - b * b
    with np.errstate(all="ignore"):
        tau2 = f(2.0) * np.log(o * f(255.0)).astype(f) * f(1.0005) + f(1e-4)
        bx = np.sqrt(tau2 * c / det) * f(1.0005) + f(0.01)
        by = np.sqrt(tau2 * a / det) * f(1.0005) + f(0.01)
    ok = (det > 0) & (a > 0) & (c > 0) & np.isfinite(bx) & np.isfinite(by)
    ex[ok], ey[ok] = bx[ok], by[ok]
    dead = ~(o * f(255.0) >= f(1.0))
    ex[dead], ey[dead] = f(-3.0e38), f(-3.0e38)
    return ex, ey


def block_origin(tx, ty, k):
    """fwd_block_origin (gpsg_internal.cuh)."""
    return 16 * tx + 8 * ((k >> 1) & 1), 16 * ty + 4 * (2 * (k >> 2) + (k & 1))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--res", type=int, default=1024)
    ap.add_argument("--seed", type=int, default=1314)
    args = ap.parse_args()
    sc = synth.stereo_pair_scene(args.res, seed=args.seed)
    W, H = sc["W"], sc["H"]
    g = ri.project(sc["means3D"], sc["scales"], sc["rots"], sc["opacity"], sc["view"], sc["proj"], sc["tanfovx"],
                   sc["tanfovy"], W, H)
    keys, plist, ranges = ri.bin_tiles(g)
    _, _, n_contrib = ri.composite(g, plist, ranges, sc["colors"], sc["opacity"], sc["bg"], W, H)
    # the device composites the fp32 state: means2D, conic, opacity as fp32
    xy = g["pix"].astype(np.float32)
    ex, ey = cull_box(g["conic"], np.asarray(sc["opacity"], np.float32).reshape(-1))
    lengths = (ranges[:, 1].astype(np.int64) - ranges[:, 0])
    busy = np.nonzero(lengths > 0)[0]
    scanned, kept, stop_frac, pix_frac, spread2, spread4 = [], [], [], [], [], []
    f = np.float32
    for t in busy:
        s, n = int(ranges[t, 0]), int(lengths[t])
        ids = plist[s:s + n]
        x, y, hx, hy = xy[ids, 0], xy[ids, 1], ex[ids], ey[ids]
        tx, ty = int(t) % g["gx"], int(t) // g["gx"]
        stops = []
        for k in range(8):
            bx0, by0 = block_origin(tx, ty, k)
            if bx0 >= W or by0 >= H:
                stops.append(np.nan)
                continue
            hit = (x >= f(bx0) - hx) & (x <= f(bx0 + 7) + hx) & (y >= f(by0) - hy) & (y <= f(by0 + 3) + hy)
            scanned.append(n)
            kept.append(int(hit.sum()))
            nc = n_contrib[by0:min(by0 + 4, H), bx0:min(bx0 + 8, W)].astype(np.int64)
            stops.append(nc.max() / n)
            pix_frac.extend((nc.reshape(-1) / n).tolist())
        stops = np.asarray(stops)
        stop_frac.extend(stops[np.isfinite(stops)].tolist())
        for grp, out in ((2, spread2), (4, spread4)):
            for c0 in range(0, 8, grp):
                v = stops[c0:c0 + grp]
                v = v[np.isfinite(v)]
                if v.size > 1 and v.mean() > 0:
                    out.append(v.max() / v.mean())
    busy_len = lengths[busy]
    res = dict(scene=f"stereo_pair_scene({args.res}, seed={args.seed})", P=int(sc["means3D"].shape[0]),
               P_visible=int(g["visible"].sum()), N=int(keys.size), tiles=int(lengths.size), non_empty_tiles=int(busy.size),
               tiles_1025_1536=int(((busy_len > 1024) & (busy_len <= 1536)).sum()),
               tile_len_median=float(np.median(busy_len)) if busy.size else 0.0, tile_len_max=int(lengths.max()),
               entries_scanned_per_block=float(np.mean(scanned)) if scanned else 0.0,
               survivors_per_block=float(np.mean(kept)) if kept else 0.0,
               survivor_fraction=float(np.sum(kept) / max(np.sum(scanned), 1)),
               list_bytes_written_per_pair=float(4 * np.sum(kept) / max(keys.size, 1)),
               block_stop_fraction_mean=float(np.mean(stop_frac)) if stop_frac else 0.0,
               pixel_stop_fraction_median=float(np.median(pix_frac)) if pix_frac else 0.0,
               stop_spread_max_over_mean_2_blocks=float(np.mean(spread2)) if spread2 else 0.0,
               stop_spread_max_over_mean_4_blocks=float(np.mean(spread4)) if spread4 else 0.0)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
