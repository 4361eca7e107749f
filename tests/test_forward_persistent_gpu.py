"""The persistent tile sort (tile_sort_gather_kernel<false>: a grid of as many CTAs as fit on the GPU, each taking tiles
of tile_order with an atomic ticket and stopping at the first empty one) and its survivor-list build (hit masks in shared
memory, two warps per block list), on scenes chosen by how many tiles are non-empty.

The exact entry point must match the fp32 oracle and a numpy rebuild of the lists; the planned (sync-free) entry point
must leave the same image, final_T, n_contrib, ranges, slab A, block counts and block lists, bit for bit, directly, on
CUDA graph replays and on 8 streams at once.  Every output is poisoned with NaN before each forward, so a pixel or tile
that no kernel visits cannot pass."""
import ctypes as C

import numpy as np
import pytest
import torch

from gps_gaussian_b200 import _lib, synth
from test_block_lists_gpu import _assert_block_lists
from test_raster_gpu import _assert_forward_parity, _run

pytestmark = pytest.mark.gpu

BG = (0.3, 0.6, 0.9)


def _tile_scene(counts, res, seed=0, width=None):
    """counts: {tile id: n}.  n splats of ~0.4 px sigma within 2 px of each tile's centre, so each lands in its tile only
    (the ring camera of synth.random_cube_scene, image res x res or width x res)."""
    W = width or res
    cam = synth.random_cube_scene(1, res, seed=seed, bg=BG, width=W, height=res)
    K, E = cam["cam"]["K"], cam["cam"]["E"]
    gx = (W + 15) // 16
    rng = np.random.default_rng(seed)
    pos = []
    for t, n in counts.items():
        z = rng.uniform(2.0, 6.0, n)
        u = 16 * (t % gx) + 7.5 + rng.uniform(-2, 2, n)
        v = 16 * (t // gx) + 7.5 + rng.uniform(-2, 2, n)
        pos.append(np.stack([(u + 0.5 - K[0, 2]) * z / K[0, 0], (v + 0.5 - K[1, 2]) * z / K[1, 1], z], 1))
    p_view = np.concatenate(pos)
    P = p_view.shape[0]
    X = ((p_view - E[:, 3]) @ E[:, :3]).astype(np.float32)
    rot = rng.standard_normal((P, 4)).astype(np.float32)
    rot /= np.linalg.norm(rot, axis=1, keepdims=True)
    attrs = dict(means3D=X, scales=np.repeat((0.4 * p_view[:, 2:3] / K[0, 0]).astype(np.float32), 3, axis=1), rots=rot,
                 opacity=rng.uniform(0.05, 0.6, (P, 1)).astype(np.float32),
                 colors=rng.uniform(0.0, 1.0, (P, 3)).astype(np.float32))
    perm = rng.permutation(P)
    return dict(cam, **{k: np.ascontiguousarray(a[perm]) for k, a in attrs.items()})


def _empty_scene():
    sc = synth.random_cube_scene(3000, 128, bg=BG, seed=5)
    return dict(sc, means3D=(sc["means3D"] + np.float32(1e4)).astype(np.float32))


def _one_tile_scene():
    return _tile_scene({37: 300}, 128, seed=1)


def _all_tiles_scene():
    return _tile_scene({t: 1 + 37 * t for t in range(64)}, 128, seed=2)


def _ragged_count_scene():
    # 601 non-empty tiles of 1024 (prime: a multiple of no multi-CTA grid), lengths spread over every size class
    rng = np.random.default_rng(3)
    tiles = rng.choice(1024, 601, replace=False)
    return _tile_scene({int(t): int(n) for t, n in zip(tiles, rng.integers(1, 1700, 601))}, 512, seed=3)


def _big_mixed_scene():
    # big tiles (2048 < n <= 4096, the big-tile kernel) among short ones, on a non-square image
    counts = {0: 2049, 5: 4096, 17: 3000, 40: 2048, 41: 1537, 42: 700}
    counts.update({t: 1 + 13 * t for t in range(18, 40)})
    return _tile_scene(counts, 96, seed=4, width=160)


SCENES = {"empty": _empty_scene, "one-tile": _one_tile_scene, "all-tiles": _all_tiles_scene,
          "601-tiles": _ragged_count_scene, "big-mixed": _big_mixed_scene}


def _tiles(sc):
    return ((sc["W"] + 15) // 16) * ((sc["H"] + 15) // 16)


def _nonempty(rc):
    r = rc.state()["ranges"].cpu().numpy().view(np.uint32).astype(np.int64)
    return r[:, 1] > r[:, 0]


def _planned(sc, capacity):
    from gps_gaussian_b200.planned import PlannedRasterizer
    return PlannedRasterizer(sc["means3D"].shape[0], sc["H"], sc["W"], capacity_pairs=capacity)


def _args(sc):
    from gps_gaussian_b200.introspect import to_device
    d = to_device(sc)
    return (sc, d["means3D"], d["colors"], d["opacity"], d["scales"], d["rots"])


def _poison(pr, depth=None, alpha=None):
    pr.color.fill_(float("nan"))
    pr.image.fill_(0xff)          # final_T = NaN, n_contrib = ~0, ranges, counts
    pr.binning.fill_(0xff)
    for t in (depth, alpha):
        if t is not None:
            t.fill_(float("nan"))


def _planned_state(pr, sc):
    """final_T, n_contrib, ranges, block counts and, per non-empty tile, slab A and the 8 lists of a planned forward."""
    H, W, tiles = sc["H"], sc["W"], _tiles(sc)
    iv, bv = _lib.ImageView(), _lib.BinningView()
    _lib.check(_lib.lib.gpsg_image_view(C.c_void_p(pr.image.data_ptr()), W, H, C.byref(iv)), "gpsg_image_view")
    _lib.check(_lib.lib.gpsg_binning_view(C.c_void_p(pr.binning.data_ptr()), pr.capacity, C.byref(bv)), "gpsg_binning_view")
    sub = lambda buf, ptr, n: buf[int(ptr) - buf.data_ptr():int(ptr) - buf.data_ptr() + n]
    st = dict(final_T=sub(pr.image, iv.final_T, 4 * H * W).view(torch.float32).view(H, W),
              n_contrib=sub(pr.image, iv.n_contrib, 4 * H * W).view(torch.int32).view(H, W),
              ranges=sub(pr.image, iv.ranges, 8 * tiles).view(torch.int32).view(tiles, 2),
              block_counts=sub(pr.image, iv.block_counts, 32 * tiles).view(torch.int32).view(tiles, 8))
    st["slabA"] = sub(pr.binning, bv.slabA, 16 * pr.capacity).view(torch.float32).view(-1, 4)
    st["block_lists"] = sub(pr.binning, bv.block_lists, 32 * pr.capacity).view(torch.int32)
    return {k: v.cpu().numpy() for k, v in st.items()}


def _assert_same_state(got, want, N):
    """Planned state `got` equals exact state `want` (numpy dicts): images' per-pixel state, ranges, counts, slab A and
    lists of every non-empty tile."""
    for k in ("final_T", "n_contrib", "ranges"):
        assert np.array_equal(got[k].view(np.uint32), want[k].view(np.uint32)), k
    ranges = want["ranges"].view(np.uint32).astype(np.int64)
    live = ranges[:, 1] > ranges[:, 0]
    assert np.array_equal(got["block_counts"][live], want["block_counts"][live])
    if N:
        assert np.array_equal(got["slabA"][:N].view(np.uint32), want["slabA"][:N].view(np.uint32))
    for t in np.nonzero(live)[0]:
        s, e = ranges[t]
        for k in range(8):
            c = int(want["block_counts"][t, k])
            a = 8 * s + k * (e - s)
            assert np.array_equal(got["block_lists"][a:a + c], want["block_lists"][a:a + c]), (int(t), k)


def _exact_state(rc):
    st = rc.state()
    keep = ("final_T", "n_contrib", "ranges", "block_counts", "slabA", "block_lists")
    return {k: st[k].cpu().numpy() for k in keep if k in st}


@pytest.mark.parametrize("name", list(SCENES))
def test_exact_and_planned_forward(name):
    """Oracle parity and list rebuild on the exact entry point; the planned one leaves the same state bit for bit."""
    sc = SCENES[name]()
    if name == "empty":
        rc = _run(sc)
        assert rc.num_rendered == 0
        assert (rc.color.cpu().numpy() == np.asarray(BG, np.float32)[:, None, None]).all()
    else:
        rc, _ = _assert_forward_parity(sc, tag=f"persistent-{name}")
        assert _assert_block_lists(rc.state(), sc["W"]) > 0
    live = _nonempty(rc)
    want_live = {"empty": 0, "one-tile": 1, "all-tiles": _tiles(sc), "601-tiles": 601, "big-mixed": 28}[name]
    assert live.sum() == want_live
    if name == "big-mixed":
        r = rc.state()["ranges"].cpu().numpy().view(np.uint32).astype(np.int64)
        assert ((r[:, 1] - r[:, 0]) > 2048).sum() == 3
    pr = _planned(sc, max(rc.num_rendered, 1) + 512)
    _poison(pr)
    out = pr.forward(*_args(sc))
    torch.cuda.synchronize()
    assert pr.ok() and pr.status()["num_rendered"] == rc.num_rendered
    assert torch.equal(out, rc.color)
    _assert_same_state(_planned_state(pr, sc), _exact_state(rc), rc.num_rendered)


def test_planned_overflow_renders_the_background():
    """Capacity too small: the tile sort does nothing and every pixel gets the background, T = 1, n_contrib = 0."""
    sc = _ragged_count_scene()
    rc = _run(sc)
    pr = _planned(sc, rc.num_rendered // 2)
    _poison(pr)
    out = pr.forward(*_args(sc))
    torch.cuda.synchronize()
    assert not pr.ok()
    assert (out.cpu().numpy() == np.asarray(BG, np.float32)[:, None, None]).all()
    st = _planned_state(pr, sc)
    assert (st["final_T"] == 1.0).all() and (st["n_contrib"] == 0).all()


@pytest.mark.parametrize("name", ["601-tiles", "big-mixed"])
def test_graph_replays_equal_a_direct_call(name):
    """The ticket word is re-zeroed in stream order by every replay: two replays give the direct call's state."""
    sc = SCENES[name]()
    args = _args(sc)
    rc = _run(sc)
    pr = _planned(sc, rc.num_rendered + 512)
    pr.forward(*args)
    torch.cuda.synchronize()
    want = _planned_state(pr, sc)
    img = pr.color.clone()
    pr.capture(*args)
    for _ in range(2):
        _poison(pr)
        pr.replay()
        torch.cuda.synchronize()
        assert pr.ok() and torch.equal(pr.color, img)
        _assert_same_state(_planned_state(pr, sc), want, rc.num_rendered)


def test_eight_streams_equal_serial_views():
    """8 planned rasterizers on 8 streams at once (their persistent grids share the GPU) render what they render one
    after the other."""
    scenes = [_ragged_count_scene(), _big_mixed_scene()] * 4
    args = [_args(sc) for sc in scenes]
    prs = [_planned(sc, 520_000) for sc in scenes]
    want = []
    for pr, a in zip(prs, args):
        _poison(pr)
        pr.forward(*a)
        torch.cuda.synchronize()
        assert pr.ok()
        want.append((pr.color.clone(), _planned_state(pr, a[0])))
    for pr in prs:
        _poison(pr)
    torch.cuda.synchronize()
    streams = [torch.cuda.Stream() for _ in prs]
    for _ in range(3):
        for pr, a, s in zip(prs, args, streams):
            s.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(s):
                pr.forward(*a)
        for s in streams:
            torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    for pr, a, (img, st) in zip(prs, args, want):
        assert pr.ok() and torch.equal(pr.color, img)
        _assert_same_state(_planned_state(pr, a[0]), st, pr.status()["num_rendered"])


@pytest.mark.parametrize("mode", ["aux", "antialias"])
def test_aux_and_antialias_planned_equal_exact(mode):
    from gps_gaussian_b200.introspect import RasterCall
    for sc in (_ragged_count_scene(), _big_mixed_scene(), _empty_scene()):
        H, W = sc["H"], sc["W"]
        aux = mode == "aux"
        rc = RasterCall(sc, antialiasing=not aux)
        rc.color.fill_(float("nan"))
        dd = torch.full((H, W), float("nan"), device="cuda") if aux else None
        da = torch.full((H, W), float("nan"), device="cuda") if aux else None
        rc.forward(dd, da)
        torch.cuda.synchronize()
        pr = _planned(sc, max(rc.num_rendered, 1) + 512)
        pd = torch.empty((H, W), device="cuda") if aux else None
        pa = torch.empty((H, W), device="cuda") if aux else None
        _poison(pr, pd, pa)
        pr.forward(*_args(sc), depth=pd, alpha=pa, antialiasing=not aux)
        torch.cuda.synchronize()
        assert pr.ok() and torch.equal(pr.color, rc.color)
        assert not torch.isnan(rc.color).any()
        if aux:
            assert torch.equal(pd, dd) and torch.equal(pa, da) and not torch.isnan(dd).any()
        _assert_same_state(_planned_state(pr, sc), _exact_state(rc), rc.num_rendered)
