"""The tile sort's counting pass (raster_binning.cu: TileSort::count_sort) on the depth windows and bucket sizes where it
changes behaviour.

A tile of n <= 2048 entries is ordered by bucketing each entry on the top 11 bits of its depth window (shift =
max(0, w - 11), w the bit length of the tile's depth span) and insertion-sorting each bucket; a bucket of more than 32
entries sends the tile to the radix sort instead.  Each scene holds, one tile each:
  * one list on each size-class boundary (512/513, 1024/1025, 1536/1537, 2048/2049), whose depths span [2, 6] (w = 24,
    shift 13) with one cluster of CLUSTER nearly equal depths -- 32 entries (counting path) or 33 (radix path) in one
    bucket -- that holds two runs of equal depths (ordered by Gaussian id);
  * a narrow window (w < 11, shift 0: every bucket is one depth word) with equal-depth runs;
  * all depths equal (w = 0): 20 entries (one bucket, counting path) and 600 (radix path);
  * the widest window a camera produces here (depths 0.25 .. 2e5, w = 28); w = 31 would need a depth span from the near
    plane (0.2) to ~1e38.
On the exact entry point keys, point list and ranges must equal the oracle's bit for bit, slab A must be the sorted
Gaussians' means, and the per-block survivor lists and their counts must equal a rebuild from slab A; the planned entry
point must render the same image bit for bit."""
import numpy as np
import pytest
import torch

from gps_gaussian_b200 import synth
from test_block_lists_gpu import _assert_block_lists
from test_raster_gpu import _assert_forward_parity

pytestmark = pytest.mark.gpu

RES, GRID = 128, 8
SIZES = (512, 513, 1024, 1025, 1536, 1537, 2048, 2049)
BUCKET_BITS, MAX_BUCKET = 11, 32
CLUSTER_Z = 4.002          # mid-bucket for a window starting at depth 2.0 (bucket width 2^13 ulps ~ 3.9e-3 at z = 4)


def _tile_depths(rng, n, cluster):
    """Depths of one size-class tile: anchors at 2 and 6, `cluster` entries within +-3e-4 of CLUSTER_Z (two runs of 8
    equal depths among them), the rest uniform in [2, 6] away from the cluster's bucket."""
    z = rng.uniform(2.0, 6.0, n - 2 - cluster)
    z = np.where(np.abs(z - CLUSTER_Z) < 0.02, z + 0.05, z)
    c = CLUSTER_Z + rng.uniform(-3e-4, 3e-4, cluster)
    return np.concatenate([[2.0, 6.0], z, c]), [(n - cluster, 8), (n - cluster + 8, 8)]


def _scene(cluster, seed=7):
    cam = synth.random_cube_scene(1, RES, seed=seed)                 # the ring camera only
    K, E = cam["cam"]["K"], cam["cam"]["E"]
    rng = np.random.default_rng(seed)
    tiles = [_tile_depths(rng, n, cluster) for n in SIZES]
    tiles.append((4.0 + rng.uniform(0.0, 4e-4, 700), [(0, 12), (12, 5)]))    # ~900 ulps: w = 10
    tiles.append((np.full(20, 3.0), [(0, 20)]))                              # w = 0, one bucket of 20
    tiles.append((np.full(600, 3.0), [(0, 600)]))                            # w = 0, one bucket of 600
    tiles.append((np.concatenate([[0.25, 2e5], np.exp(rng.uniform(np.log(0.25), np.log(2e5), 1298))]), []))
    pos = []
    for t, (z, runs) in enumerate(tiles):
        n = z.size
        # pixel within 2 px of the tile centre; with a ~0.4 px sigma the splat touches this tile only
        u = 16 * (t % GRID) + 7.5 + rng.uniform(-2, 2, n)
        v = 16 * (t // GRID) + 7.5 + rng.uniform(-2, 2, n)
        for s, m in runs:                                             # identical positions => identical depth bits
            z[s:s + m], u[s:s + m], v[s:s + m] = z[s], u[s], v[s]
        x = (u + 0.5 - K[0, 2]) * z / K[0, 0]
        y = (v + 0.5 - K[1, 2]) * z / K[1, 1]
        pos.append(np.stack([x, y, z], 1))
    p_view = np.concatenate(pos)
    P = p_view.shape[0]
    X = ((p_view - E[:, 3]) @ E[:, :3]).astype(np.float32)
    perm = rng.permutation(P)                                          # interleave the tiles and runs in index space
    rot = rng.standard_normal((P, 4)).astype(np.float32)
    rot /= np.linalg.norm(rot, axis=1, keepdims=True)
    scale = np.repeat((0.4 * p_view[:, 2:3] / K[0, 0]).astype(np.float32), 3, axis=1)
    attrs = dict(means3D=X, scales=scale, rots=rot, opacity=rng.uniform(0.2, 1.0, (P, 1)).astype(np.float32),
                 colors=rng.uniform(0.0, 1.0, (P, 3)).astype(np.float32))
    return dict(cam, **{k: np.ascontiguousarray(a[perm]) for k, a in attrs.items()}), [z.size for z, _ in tiles]


def _window(depth_bits):
    """(w, largest bucket, largest equal-depth run) of one tile, as the kernel buckets it."""
    off = depth_bits - depth_bits.min()
    w = int(off.max()).bit_length()
    shift = max(0, w - BUCKET_BITS)
    return w, int(np.bincount(off >> shift).max()), int(np.unique(depth_bits, return_counts=True)[1].max())


@pytest.mark.parametrize("cluster", [MAX_BUCKET, MAX_BUCKET + 1])
def test_counting_pass_windows_and_buckets(cluster):
    from gps_gaussian_b200.introspect import to_device
    from gps_gaussian_b200.planned import PlannedRasterizer
    sc, lengths = _scene(cluster)
    rc, ref = _assert_forward_parity(sc, tag=f"tile-count-sort-cluster{cluster}")
    ranges = np.asarray(ref["ranges"]).reshape(-1, 2).astype(np.int64)
    counts = ranges[:, 1] - ranges[:, 0]
    assert list(counts[:len(lengths)]) == lengths and not counts[len(lengths):].any()
    depth = (np.asarray(ref["keys"]).astype(np.uint64) & np.uint64(0xffffffff)).astype(np.int64)
    win = [_window(depth[s:e]) for s, e in ranges[:len(lengths)]]
    # the scene exercises what it claims to
    for t in range(len(SIZES)):
        assert win[t][0] == 24 and win[t][1] == cluster and win[t][2] >= 8, (t, win[t])
    narrow, one_bucket, flat, wide = win[len(SIZES):]
    assert 0 < narrow[0] < BUCKET_BITS and narrow[2] >= 12 and narrow[1] == narrow[2]
    assert one_bucket == (0, 20, 20) and flat == (0, 600, 600)
    assert wide[0] >= 28
    # slab A follows the point list: its centres are the sorted Gaussians' means
    st = rc.state()
    vals = np.asarray(ref["vals"]).astype(np.int64)
    means = st["means2D"].cpu().numpy()
    assert np.array_equal(st["slabA"].cpu().numpy()[:, :2].view(np.uint32), means[vals].view(np.uint32))
    assert _assert_block_lists(st, sc["W"]) == 8 * len(lengths)
    d = to_device(sc)
    pr = PlannedRasterizer(sc["means3D"].shape[0], RES, RES, capacity_pairs=rc.num_rendered + 1024)
    out = pr.forward(sc, d["means3D"], d["colors"], d["opacity"], d["scales"], d["rots"])
    torch.cuda.synchronize()
    assert pr.ok() and pr.status()["num_rendered"] == rc.num_rendered
    assert torch.equal(out, rc.color) and torch.equal(pr.radii, rc.radii)
