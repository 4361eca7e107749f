"""The in-CTA tile sort (tile_sort_gather_kernel) on tile lists that sit on every one of its size-class boundaries.

Each scene puts one tile list of each length 512/513, 1024/1025, 1536/1537 and 2048/2049 (1, 2, 3 and 4 keys per thread,
then the big-tile kernel) into its own tile, plus one 1300-entry tile whose depths span more than 24 bits.  Every tile
also holds two equal-depth runs of 16 (ordered by id in shared memory) or 17 (the full-sort fallback).  On the exact
entry point, keys, point list and ranges must equal the oracle's bit for bit; the planned entry point, which does not
write keys and point list, must render the same image."""
import numpy as np
import pytest
import torch

from gps_gaussian_b200 import synth
from test_raster_gpu import _assert_forward_parity

pytestmark = pytest.mark.gpu

SIZES = (512, 513, 1024, 1025, 1536, 1537, 2048, 2049)
WIDE_N, WIDE_Z = 1300, (0.5, 90.0)      # depth bits 0x3f000000 .. 0x42b40000: a 26-bit window
RES, GRID = 128, 8


def _boundary_scene(run, seed=3):
    cam = synth.random_cube_scene(1, RES, seed=seed)                 # the ring camera only
    K, E = cam["cam"]["K"], cam["cam"]["E"]
    rng = np.random.default_rng(seed)
    lists = [(n, (2.0, 6.0)) for n in SIZES] + [(WIDE_N, WIDE_Z)]
    pos = []
    for t, (n, (z0, z1)) in enumerate(lists):
        m = run - 1                                                   # copies of entries 0 and 1: two runs of `run`
        z = rng.uniform(z0, z1, n - 2 * m)
        z = np.concatenate([z, np.full(m, z[0]), np.full(m, z[1])])
        # pixel within 2 px of the tile centre; with a 3 px radius (below) the splat touches this tile only
        u = 16 * (t % GRID) + 7.5 + rng.uniform(-2, 2, n)
        v = 16 * (t // GRID) + 7.5 + rng.uniform(-2, 2, n)
        u[-2 * m:-m], v[-2 * m:-m] = u[0], v[0]                      # identical positions => identical depth bits
        u[-m:], v[-m:] = u[1], v[1]
        x = (u + 0.5 - K[0, 2]) * z / K[0, 0]
        y = (v + 0.5 - K[1, 2]) * z / K[1, 1]
        pos.append(np.stack([x, y, z], 1))
    p_view = np.concatenate(pos)
    P = p_view.shape[0]
    X = ((p_view - E[:, 3]) @ E[:, :3]).astype(np.float32)
    perm = rng.permutation(P)                                          # interleave the runs in index space
    rot = rng.standard_normal((P, 4)).astype(np.float32)
    rot /= np.linalg.norm(rot, axis=1, keepdims=True)
    scale = np.repeat((0.4 * p_view[:, 2:3] / K[0, 0]).astype(np.float32), 3, axis=1)   # ~0.4 px sigma
    attrs = dict(means3D=X, scales=scale, rots=rot, opacity=rng.uniform(0.2, 1.0, (P, 1)).astype(np.float32),
                 colors=rng.uniform(0.0, 1.0, (P, 3)).astype(np.float32))
    return dict(cam, **{k: np.ascontiguousarray(a[perm]) for k, a in attrs.items()})


@pytest.mark.parametrize("run", [16, 17])
def test_tile_lists_on_size_class_boundaries(run):
    from gps_gaussian_b200.introspect import to_device
    from gps_gaussian_b200.planned import PlannedRasterizer
    sc = _boundary_scene(run)
    rc, ref = _assert_forward_parity(sc, tag=f"tile-sort-boundaries-run{run}")
    rng_ = np.asarray(ref["ranges"]).reshape(-1, 2).astype(np.int64)
    counts = rng_[:, 1] - rng_[:, 0]
    assert list(counts[:len(SIZES) + 1]) == list(SIZES) + [WIDE_N] and not counts[len(SIZES) + 1:].any()
    depth = (np.asarray(ref["keys"]).astype(np.uint64) & np.uint64(0xffffffff)).astype(np.int64)
    for t in range(len(SIZES) + 1):
        assert np.unique(depth[rng_[t, 0]:rng_[t, 1]], return_counts=True)[1].max() == run
    wide = depth[rng_[len(SIZES), 0]:rng_[len(SIZES), 1]]
    assert wide.max() - wide.min() >= 1 << 24
    d = to_device(sc)
    pr = PlannedRasterizer(sc["means3D"].shape[0], RES, RES, capacity_pairs=rc.num_rendered + 1024)
    out = pr.forward(sc, d["means3D"], d["colors"], d["opacity"], d["scales"], d["rots"])
    torch.cuda.synchronize()
    assert pr.ok() and pr.status()["num_rendered"] == rc.num_rendered
    assert torch.equal(out, rc.color) and torch.equal(pr.radii, rc.radii)
