"""The compositing forward's per-block survivor lists (raster_binning.cu: build_block_lists) on the tile-length classes of
every binning path, on ragged image edges and on an image with no pairs at all.

For each scene the forward must match the fp32 oracle (test_raster_gpu._assert_forward_parity), and the lists the binning
left behind must equal a numpy rebuild from the sorted slabs: for each 8x4 block of each tile, the list positions whose
cull box (slabA centre +- half-extents) meets the block, in list order."""
import os
import subprocess
import sys

import numpy as np
import pytest

from gps_gaussian_b200 import synth
from test_raster_gpu import _assert_forward_parity

pytestmark = pytest.mark.gpu


def _block_window(tile, grid_x, k):
    # fwd_block_origin (gpsg_internal.cuh): blocks 2c, 2c+1 form an 8x8 quarter tile
    tx, ty = tile % grid_x, tile // grid_x
    bx0 = 16 * tx + 8 * ((k >> 1) & 1)
    by0 = 16 * ty + 4 * (2 * (k >> 2) + (k & 1))
    f = np.float32
    return f(bx0), f(bx0 + 7), f(by0), f(by0 + 3)


def _assert_block_lists(st, W):
    grid_x = (W + 15) // 16
    ranges = st["ranges"].cpu().numpy().view(np.uint32).astype(np.int64)
    counts = st["block_counts"].cpu().numpy().view(np.uint32)
    if not (ranges[:, 1] > ranges[:, 0]).any():
        return 0
    A = st["slabA"].cpu().numpy()
    lists = st["block_lists"].cpu().numpy().view(np.uint32)
    checked = 0
    for t in np.nonzero(ranges[:, 1] > ranges[:, 0])[0]:
        s, e = ranges[t]
        n = e - s
        a = A[s:e]
        for k in range(8):
            wx0, wx1, wy0, wy1 = _block_window(int(t), grid_x, k)
            hit = (a[:, 0] >= wx0 - a[:, 2]) & (a[:, 0] <= wx1 + a[:, 2]) & (a[:, 1] >= wy0 - a[:, 3]) & (a[:, 1] <= wy1 + a[:, 3])
            want = np.nonzero(hit)[0].astype(np.uint32)
            assert counts[t, k] == want.size, (int(t), k)
            got = lists[8 * s + k * n: 8 * s + k * n + want.size]
            assert np.array_equal(got, want), (int(t), k)
            checked += 1
    return checked


SCENES = {
    # (res, P, spread, mul, bg, camera overrides)
    "over-4096": (48, 30000, 0.25, 1.0, (0.0, 0.0, 0.0), {}),          # tile lists > 4096: the radix path
    "over-2048": (64, 4500, 0.35, 1.5, (0.0, 0.0, 0.0), {}),           # 2048 < n <= 4096: the big-tile sort kernel
    "ragged": (250, 4000, 0.6, 4.0, (0.3, 0.6, 0.9), {}),              # W, H not multiples of 16
    "ragged-wide": (64, 3000, 0.6, 4.0, (0.3, 0.6, 0.9), dict(width=250, height=40, focal=(240.0, 190.0),
                                                               principal=(118.0, 23.0))),
}


@pytest.mark.parametrize("name", list(SCENES))
def test_block_lists_and_forward(name):
    res, P, spread, mul, bg, cam = SCENES[name]
    sc = synth.random_cube_scene(P, res, spread=spread, scale_mul=mul, bg=bg, seed=11, **cam)
    rc, ref = _assert_forward_parity(sc, tag=f"block-lists-{name}")
    st = rc.state()
    counts = np.diff(st["ranges"].cpu().numpy().view(np.uint32).astype(np.int64), axis=1)
    if name == "over-4096":
        assert counts.max() > 4096
    elif name == "over-2048":
        assert 2048 < counts.max() <= 4096
    assert _assert_block_lists(st, sc["W"]) > 0


def test_all_empty_image():
    """Every Gaussian far outside the view: no pair, every pixel is the background."""
    from test_raster_gpu import _run
    sc = synth.random_cube_scene(2000, 100, bg=(0.2, 0.4, 0.6), seed=5)
    sc = dict(sc, means3D=(sc["means3D"] + np.float32(1e4)).astype(np.float32))
    rc = _run(sc)
    assert rc.num_rendered == 0
    st = rc.state()
    assert (st["final_T"].cpu().numpy() == 1.0).all() and (st["n_contrib"].cpu().numpy() == 0).all()
    img = rc.color.cpu().numpy()
    for c, v in enumerate((0.2, 0.4, 0.6)):
        assert (img[c] == np.float32(v)).all()


def test_block_lists_radix_path():
    """The same scenes with GPSG_BINNING=radix (read once per process: a subprocess), where the lists come from the
    per-tile pass after gather_ranges."""
    env = dict(os.environ, GPSG_BINNING="radix")
    here = os.path.dirname(os.path.abspath(__file__))
    r = subprocess.run([sys.executable, "-m", "pytest", "-q", "-x", "-m", "gpu", os.path.join(here, "test_block_lists_gpu.py"),
                        "-k", "test_block_lists_and_forward or test_all_empty"],
                       env=env, cwd=os.path.dirname(here), capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-4000:] + r.stderr[-4000:]
