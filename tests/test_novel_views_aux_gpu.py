"""GPU: aux mode of the novel-view cache -- depth and alpha sweeps beside the image sweep, through the planned forwards'
out_depth / out_alpha (gpsg_rasterize_forward_planned / _maps_planned), including the overflow re-render and the exact
fallback for over-long tile lists."""
import pytest
import torch

from test_novel_views import OPTS, _pair_data

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("streams,mode,cam", [(1, "compact", {}), (3, "compact", {}), (2, "maps", {}),
                                              (2, "maps", dict(width=96, height=160, fy_scale=0.85))],
                         ids=["1-compact", "3-compact", "2-maps", "2-maps-96x160"])
def test_aux_sweep_equals_per_ratio_pts2render_aux(streams, mode, cam):
    """Images, depth and alpha of the cached aux sweep == get_novel_calib + pts2render_aux per ratio, bit for bit; the
    images also equal the sweep without aux."""
    from gps_gaussian_b200 import novel_calib
    from gps_gaussian_b200.GaussianRender import pts2render_aux
    from gps_gaussian_b200.novel_views import NovelViewRenderer, render_novel_views
    res, ratios = 128, [0.1, 0.5, 0.9]
    data = _pair_data(res, (21, 22), **cam)
    opt, bg = OPTS["plain"], [0.05, 0.1, 0.2]
    H, W = cam.get("height", res), cam.get("width", res)
    nvr = NovelViewRenderer(data, opt, bg, streams=streams, mode=mode)
    img, depth, alpha = nvr.render(ratios, aux=True)
    assert depth.shape == (2, len(ratios), 1, H, W) and alpha.shape == depth.shape
    assert torch.equal(img, nvr.render(ratios))
    for r, ratio in enumerate(ratios):
        nv = pts2render_aux(novel_calib.get_novel_calib(data, opt, ratio=ratio), bg)["novel_view"]
        assert torch.equal(img[:, r], nv["img_pred"]) and torch.equal(depth[:, r], nv["depth_pred"]), ratio
        assert torch.equal(alpha[:, r], nv["alpha_pred"]), ratio
    assert float(alpha.max()) > 0.5 and float(depth.max()) > 0.0
    out = render_novel_views(data, opt, ratios, bg, streams=streams, mode=mode, aux=True)["novel_view"]
    for k, t in (("img_pred_sweep", img), ("depth_pred_sweep", depth), ("alpha_pred_sweep", alpha)):
        assert torch.equal(out[k], t), k


@pytest.mark.parametrize("mode", ["compact", "maps"])
def test_aux_sweep_overflow_and_exact_fallback(mode, monkeypatch):
    """A forced overflow (tiny capacity) re-renders the view with a grown buffer, and an overflow counted as an over-long
    tile list goes through the exact aux entry point: both equal the big-capacity aux sweep bit for bit."""
    from gps_gaussian_b200 import novel_views
    from gps_gaussian_b200.novel_views import NovelViewRenderer
    res, ratios = 96, [0.5, 0.25]
    data = _pair_data(res, (6,))
    opt = OPTS["plain"]
    big = NovelViewRenderer(data, opt, [0, 0, 0], mode=mode).render(ratios, aux=True)
    small = NovelViewRenderer(data, opt, [0, 0, 0], streams=2, capacity_pairs=64, mode=mode)
    out = small.render(ratios, aux=True)
    assert int(small.last_status[0, 2]) == 1                                  # the tiny capacity did overflow...
    for a, b in zip(out, big):
        assert torch.equal(a, b)                                              # ...and the re-render is exact
    monkeypatch.setattr(novel_views, "_MAX_TILE_SORT", 8)
    tiny = NovelViewRenderer(data, opt, [0, 0, 0], streams=2, capacity_pairs=64, mode=mode)
    cap0 = tiny.rast[0].capacity
    out2 = tiny.render(ratios, aux=True)
    assert tiny.rast[0].capacity == cap0                                      # the exact entry point rendered them
    for a, b in zip(out2, big):
        assert torch.equal(a, b)
