"""Novel-view calibration (closed-form, batched) pinned to the reference's get_novel_calib golden vectors, and the
Gaussian cache across novel views (sync-free map-ingest sweep) against per-ratio get_novel_calib + pts2render."""
import os
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from gps_gaussian_b200 import novel_calib, synth

G = np.load(os.path.join(os.path.dirname(__file__), "golden", "novel_calib_golden.npz"))
OPTS = {"plain": SimpleNamespace(use_hr_img=False, znear=0.01, zfar=100.0, trans=[0.0, 0.0, 0.0], scale=1.0),
        "hr": SimpleNamespace(use_hr_img=True, znear=0.01, zfar=100.0, trans=[0.0, 0.0, 0.0], scale=1.0),
        "shift": SimpleNamespace(use_hr_img=False, znear=0.05, zfar=20.0, trans=[0.1, -0.2, 0.3], scale=1.5)}
KEYS = ("FovX", "FovY", "world_view_transform", "full_proj_transform", "camera_center")


@pytest.mark.parametrize("tag", list(OPTS))
def test_novel_calib_batch_matches_reference_golden(tag):
    """All (sample, ratio) cameras in one vectorised pass == the reference's per-sample scipy/inv/bmm loop (fp32 outputs;
    the reference itself rounds through float32 intermediates, so agreement is to a few ulp of the largest entry)."""
    opt, side = OPTS[tag], int(G[f"{tag}_side"])
    got = novel_calib.novel_calib_batch(G["intr0"], G["intr1"], G["extr0"], G["extr1"], G["ratios"], side, side, opt.znear,
                                        opt.zfar, opt.trans, opt.scale, opt.use_hr_img)
    for k in KEYS:
        ref = G[f"{tag}_{k}"]
        assert got[k].shape == ref.shape and got[k].dtype == np.float32, k
        assert np.abs(got[k] - ref).max() <= 4e-6 * max(1.0, np.abs(ref).max()), (k, np.abs(got[k] - ref).max())


def test_get_novel_calib_mirror_fills_data_like_the_reference():
    bs = G["intr0"].shape[0]
    T = lambda a: torch.tensor(a)
    data = {"lmain": {"intr": T(G["intr0"]), "extr": T(G["extr0"])}, "rmain": {"intr": T(G["intr1"]), "extr": T(G["extr1"])},
            "novel_view": {"width": torch.full((bs,), 1024, dtype=torch.int32), "height": torch.full((bs,), 1024, dtype=torch.int32)}}
    out = novel_calib.get_novel_calib(data, OPTS["plain"], ratio=0.5)
    ri = list(G["ratios"]).index(0.5)
    for k in KEYS:
        ref = G[f"plain_{k}"][:, ri]
        t = out["novel_view"][k]
        assert tuple(t.shape) == ref.shape and t.dtype == torch.float32
        assert np.abs(t.numpy() - ref).max() <= 4e-6 * max(1.0, np.abs(ref).max())
    # rotations stay orthonormal, endpoints reproduce the source cameras
    c = novel_calib.novel_calib_batch(G["intr0"], G["intr1"], G["extr0"], G["extr1"], [0.0, 1.0], 1024, 1024, 0.01, 100.0)
    R = np.swapaxes(c["world_view_transform"][..., :3, :3], -1, -2).astype(np.float64)
    assert np.abs(R @ np.swapaxes(R, -1, -2) - np.eye(3)).max() < 1e-6
    assert np.abs(R[:, 0] - G["extr0"][:, :, :3]).max() < 1e-6 and np.abs(R[:, 1] - G["extr1"][:, :, :3]).max() < 1e-6


def test_synth_novel_camera_agrees_with_batched_calib():
    """The benchmark's camera generator (synth.novel_camera) and the batched closed form are the same function."""
    K0, E0 = synth.ring_camera(-11.25, 512)
    K1, E1 = synth.ring_camera(+11.25, 512)
    for ratio in (0.25, 0.5):
        a = synth.novel_camera(K0, E0, K1, E1, 512, 512, ratio)
        b = novel_calib.novel_calib_batch(K0[None], K1[None], E0[None], E1[None], [ratio], 512, 512, synth.ZNEAR, synth.ZFAR)
        for k in ("world_view_transform", "full_proj_transform", "camera_center"):
            assert np.abs(a[k] - b[k][0, 0]).max() < 2e-6 * max(1.0, np.abs(a[k]).max()), k
        assert abs(a["FovX"] - float(b["FovX"][0, 0])) < 1e-6


def _pair_data(res, seeds, width=None, height=None, fy_scale=1.0):
    """Source maps res x res; the novel view width x height (default res), fy of the source intrinsics scaled by fy_scale."""
    datas = []
    for seed in seeds:
        sc = synth.stereo_pair_scene(res, keep_maps=True, seed=seed)
        d = {"novel_view": {"width": torch.tensor([width or res]), "height": torch.tensor([height or res])}}
        for name, vw in zip(("lmain", "rmain"), sc["views"]):
            T = lambda a: torch.tensor(a).cuda()[None]
            K = vw["K"].copy()
            K[1, 1] *= fy_scale
            d[name] = {"img": T(vw["img"]), "pts_valid": torch.tensor(vw["valid"]).cuda()[None], "xyz": T(vw["xyz"]),
                       "rot_maps": T(vw["rot_maps"]), "scale_maps": T(vw["scale_maps"]), "opacity_maps": T(vw["opacity_maps"]),
                       "intr": torch.tensor(K, dtype=torch.float32).cuda()[None],
                       "extr": torch.tensor(vw["E"], dtype=torch.float32).cuda()[None]}
        datas.append(d)
    data = {"novel_view": {k: torch.cat([d["novel_view"][k] for d in datas]) for k in datas[0]["novel_view"]}}
    for v in ("lmain", "rmain"):
        data[v] = {k: torch.cat([d[v][k] for d in datas]) for k in datas[0][v]}
    return data


@pytest.mark.gpu
@pytest.mark.parametrize("streams,mode,cam", [(1, "compact", {}), (3, "compact", {}), (2, "maps", {}),
                                              (2, "compact", dict(width=160, height=96, fy_scale=1.15)),
                                              (2, "maps", dict(width=96, height=160, fy_scale=0.85))],
                         ids=["1-compact", "3-compact", "2-maps", "2-compact-160x96", "2-maps-96x160"])
def test_cached_novel_view_sweep_equals_per_ratio_calib_plus_pts2render(streams, mode, cam):
    """test_view_interp.py:39-47 restructured: one cache, all ratios, no gather / sync -- bit-identical to the loop.
    Also with a non-square novel view and source intrinsics with fx != fy."""
    from gps_gaussian_b200.GaussianRender import pts2render
    from gps_gaussian_b200.novel_views import NovelViewRenderer
    res, ratios = 128, [0.1, 0.3, 0.5, 0.7, 0.9]
    data = _pair_data(res, (21, 22), **cam)
    opt = OPTS["plain"]
    bg = [0.05, 0.1, 0.2]
    sweep = NovelViewRenderer(data, opt, bg, streams=streams, mode=mode).render(ratios)
    assert sweep.shape == (2, len(ratios), 3, cam.get("height", res), cam.get("width", res))
    for r, ratio in enumerate(ratios):
        d = novel_calib.get_novel_calib(data, opt, ratio=ratio)
        ref = pts2render(d, bg)["novel_view"]["img_pred"]
        assert torch.equal(sweep[:, r], ref), ratio
    assert float((sweep[:, 0] - sweep[:, -1]).abs().max()) > 0.05          # the camera really moved


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["compact", "maps"])
def test_cached_sweep_grows_capacity_on_overflow(mode):
    from gps_gaussian_b200.novel_views import NovelViewRenderer
    res = 96
    data = _pair_data(res, (5,))
    opt = OPTS["plain"]
    big = NovelViewRenderer(data, opt, [0, 0, 0]).render([0.5])
    small = NovelViewRenderer(data, opt, [0, 0, 0], streams=2, capacity_pairs=64, mode=mode)
    out = small.render([0.5, 0.25])
    assert int(small.last_status[0, 2]) == 1                                # the tiny capacity did overflow...
    assert torch.equal(out[:, 0], big[:, 0])                                # ...and the re-render is exact


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["compact", "maps"])
def test_cached_sweep_routes_overlong_tile_lists_through_the_exact_entry_point(mode, monkeypatch):
    """ADVICE r1: an overflow caused by a tile list longer than the in-CTA sort cannot be cured by a larger buffer; such a view
    must go through the exact entry point (radix fallback) instead of growing 8 times and raising.  Forced here by lowering
    the threshold the redo logic compares `status[k,1]` (longest tile list) against; the capacity is sized from `status[k,0]`
    in ONE step otherwise."""
    from gps_gaussian_b200 import novel_views
    from gps_gaussian_b200.novel_views import NovelViewRenderer
    res = 96
    data = _pair_data(res, (6,))
    opt = OPTS["plain"]
    big = NovelViewRenderer(data, opt, [0, 0, 0]).render([0.5, 0.25])
    small = NovelViewRenderer(data, opt, [0, 0, 0], streams=1, capacity_pairs=64, mode=mode)
    out = small.render([0.5, 0.25])
    n_pairs = int(small.last_status[0, 0])
    assert n_pairs > 64 and small.rast[0].capacity < 3 * n_pairs             # one growth step, sized from the job's own count
    assert torch.equal(out, big)
    monkeypatch.setattr(novel_views, "_MAX_TILE_SORT", 8)                     # every overflowed job now counts as "tile too long"
    tiny = NovelViewRenderer(data, opt, [0, 0, 0], streams=2, capacity_pairs=64, mode=mode)
    cap0 = tiny.rast[0].capacity
    out2 = tiny.render([0.5, 0.25])
    assert tiny.rast[0].capacity == cap0                                      # no blind growth ...
    assert torch.equal(out2, big)                                             # ... the exact entry point rendered them
