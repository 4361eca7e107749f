"""The stage-1 preview splat on the GPU (gps_gaussian_b200.point_splat -> csrc/point_splat.cu) against the serial reference
(tests/splat_reference.py, on the C oracle's restatement of lib/TaichiRender.py:13-24): depth and colour equal bit for bit,
untouched pixels and batches included, and reruns give identical bytes."""
import numpy as np
import pytest
import torch

from splat_reference import fresh_buffers, splat_serial

pytestmark = pytest.mark.gpu


def _both(calls, depth0, color0):
    """calls: [(pts, mask, B, N)] in order on the same buffers.  Returns ((gpu depth, colour), (reference depth, colour))."""
    from gps_gaussian_b200.point_splat import point_splat
    d, c = torch.from_numpy(depth0).cuda(), torch.from_numpy(color0).cuda()
    rd, rc = depth0.copy(), color0.copy()
    for pts, mask, B, N in calls:
        point_splat(torch.from_numpy(pts).cuda(), torch.from_numpy(mask).cuda(), d, c, B=B, N=N)
        splat_serial(pts, mask, rd, rc, B=B, N=N)
    torch.cuda.synchronize()
    return (d.cpu().numpy(), c.cpu().numpy()), (rd, rc)


def _assert_bits(got, want, what=""):
    for name, g, w in zip(("depth", "color"), got, want):
        bad = g.view(np.uint32) != w.view(np.uint32)
        assert not bad.any(), (what, name, int(bad.sum()), np.argwhere(bad)[:5].tolist(), g[bad][:5], w[bad][:5])


def _cloud(rng, Bp, Np, res, zlevels=8, off=0.25):
    """Points over [-off*res, (1+off)*res)^2 (off-image ones clamp to the border) with z quantised to a few levels, so
    pixels see many exact ties; some -0, negative z and NaN mask."""
    lo, hi = -off * res, (1 + off) * res
    xy = rng.uniform(lo, hi, (Bp, Np, 2))
    z = rng.integers(-1, zlevels, (Bp, Np, 1)) / 4.0
    rgb = rng.uniform(-1, 1, (Bp, Np, 3))
    pts = np.concatenate([xy, z, rgb], 2).astype(np.float32)
    pts[..., 2][rng.uniform(size=(Bp, Np)) < 0.05] = -0.0
    mask = (rng.uniform(size=(Bp, Np)) > 0.2).astype(np.float32)
    mask[rng.uniform(size=(Bp, Np)) < 0.01] = np.nan
    return pts, mask


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_collisions_two_calls(seed):
    rng = np.random.default_rng(seed)
    res, Np = 24, 6000                                      # ~10 points per pixel
    a, b = _cloud(rng, 2, Np, res), _cloud(rng, 2, Np, res)
    d0, c0 = fresh_buffers(2, res)
    got, want = _both([(a[0], a[1], 2, Np), (b[0], b[1], 2, Np)], d0, c0)
    _assert_bits(got, want, seed)
    assert (want[1] != -1).mean() > 0.5 and (want[1] == -1).any()     # drawn and untouched pixels both present
    # the second call really composes on the first: a fresh second call gives another image
    (_, c_b), _ = _both([(b[0], b[1], 2, Np)], *fresh_buffers(2, res))
    assert not np.array_equal(c_b, got[1])


def test_edge_cases():
    nan, inf = np.float32(np.nan), np.float32(np.inf)
    rows = [
        [1, 1, nan, 1, 1, 1],          # NaN z: skipped
        [nan, 2, 0.5, 2, 2, 2],        # NaN x -> column 0
        [2, nan, 0.5, 3, 3, 3],        # NaN y -> row 0
        [1e10, 1, 0.5, 4, 4, 4],       # saturating cast, clamp to res-1
        [-1e10, -1e10, 0.5, 5, 5, 5],  # -> (0, 0)
        [inf, -inf, 0.5, 6, 6, 6],
        [3, 3, -0.0, 7, 7, 7],         # -0 and +0 tie at (3, 3)
        [3.9, 3.1, 0.0, 8, 8, 8],
        [3, 3, -0.0, 9, 9, 9],
        [4, 4, -0.5, 10, 10, 10],      # negative z
        [5, 5, -inf, 11, 11, 11],
        [6, 6, inf, 12, 12, 12],       # +inf z wins its pixel
        [6, 6, inf, 13, 13, 13],
        [6, 6, 1e30, 14, 14, 14],
        [7, 0, 0.25, 15, 15, 15],      # NaN mask: drawn
        [7, 1, 0.25, 16, 16, 16],      # mask 0.49: skipped
        [7, 2, 0.25, 17, 17, 17],      # mask 0.5: drawn
    ]
    pts = np.array([rows], np.float32)
    mask = np.ones((1, len(rows)), np.float32)
    mask[0, 14], mask[0, 15], mask[0, 16] = np.nan, 0.49, 0.5
    out = {}
    for init in (0.0, -1.0, -0.0, -np.inf, np.nan):         # depth before the call (in/out)
        d0, c0 = fresh_buffers(1, 8)
        d0[...] = init
        got, want = _both([(pts, mask, 1, len(rows))], d0, c0)
        _assert_bits(got, want, init)
        out[repr(init)] = got                                 # repr: -0.0 and 0.0 are one dict key
    # on depth -1 the zeros draw: depth takes the FIRST zero's value (-0), colour the last zero's rgb
    d, c = out["-1.0"]
    assert d[0, 0, 3, 3] == 0 and np.signbit(d[0, 0, 3, 3]) and c[0, 0, 3, 3] == 9
    assert np.signbit(out["-0.0"][0][0, 0, 3, 3]) and out["-0.0"][1][0, 0, 3, 3] == 9   # -0 stays: +0 > -0 is false
    d, c = out["0.0"]
    assert not np.signbit(d[0, 0, 3, 3]) and c[0, 0, 3, 3] == 9 and c[0, 0, 4, 4] == -1
    assert d[0, 0, 6, 6] == np.inf and c[0, 0, 6, 6] == 13 and c[0, 0, 1, 7] == 4 and c[0, 0, 0, 0] == 5
    assert c[0, 0, 0, 7] == 6 and c[0, 0, 2, 0] == 2 and c[0, 0, 0, 2] == 3
    assert (out["nan"][1] == -1).all()                       # nothing is >= NaN
    # same points split into two calls on the same buffers
    d0, c0 = fresh_buffers(1, 8)
    got, want = _both([(pts[:, :9].copy(), mask[:, :9].copy(), 1, 9), (pts[:, 9:].copy(), mask[:, 9:].copy(), 1, 8)], d0, c0)
    _assert_bits(got, want, "split")


def test_loop_domain_smaller_than_buffers():
    rng = np.random.default_rng(7)
    res, Bp, Np, B, N = 16, 3, 4000, 2, 3000
    pts, mask = _cloud(rng, Bp, Np, res)
    d0 = rng.uniform(-0.5, 1.0, (Bp, 1, res, res)).astype(np.float32)    # arbitrary in/out contents
    c0 = rng.uniform(-1, 1, (Bp, 3, res, res)).astype(np.float32)
    got, want = _both([(pts, mask, B, N)], d0, c0)
    _assert_bits(got, want)
    assert got[0][B:].tobytes() == d0[B:].tobytes() and got[1][B:].tobytes() == c0[B:].tobytes()
    # rows >= N are not read: poisoning them changes nothing
    pts2 = pts.copy()
    pts2[:, N:, 2] = 1e9
    got2, _ = _both([(pts2, mask, B, N)], d0, c0)
    _assert_bits(got2, got)


def test_full_resolution_two_views_and_rerun():
    """2 x 1024^2 points at res 1024, as the stage-1 preview at the reference's src_res, twice: identical bytes."""
    rng = np.random.default_rng(11)
    res, Np = 1024, 1024 * 1024
    views = []
    for _ in range(2):
        pts, mask = _cloud(rng, 1, Np, res, zlevels=64, off=0.05)
        views.append((pts, mask, 1, Np))
    d0, c0 = fresh_buffers(1, res)
    got, want = _both(views, d0, c0)
    _assert_bits(got, want)
    again, _ = _both(views, d0, c0)
    assert again[0].tobytes() == got[0].tobytes() and again[1].tobytes() == got[1].tobytes()


def test_rejects_bad_tensors():
    from gps_gaussian_b200.point_splat import point_splat
    pts = torch.zeros(1, 8, 6, device="cuda")
    mask = torch.ones(1, 8, device="cuda")
    d, c = torch.zeros(1, 1, 4, 4, device="cuda"), torch.zeros(1, 3, 4, 4, device="cuda")
    with pytest.raises(TypeError):
        point_splat(pts.cpu(), mask, d, c)
    with pytest.raises(TypeError):
        point_splat(pts, mask.half(), d, c)
    with pytest.raises(TypeError):
        point_splat(pts, mask, d, torch.zeros(1, 4, 4, 3, device="cuda").permute(0, 3, 1, 2))
    with pytest.raises(ValueError):
        point_splat(pts, mask, d, c, B=2)
    with pytest.raises(ValueError):
        point_splat(pts, mask, d, c, res=8)
    with pytest.raises(ValueError):
        point_splat(pts, torch.ones(1, 7, device="cuda"), d, c)


@pytest.mark.skipif(__import__("gps_gaussian_b200.harness", fromlist=["x"]).staged_reference() is None,
                    reason="oracle/_ref not staged")
def test_reference_flow2render_equals_serial_splat(tmp_path):
    """The reference's own TaichiRenderBatch.flow2render (lib/TaichiRender.py:26-60, through the `taichi` stand-in) on a
    stage-1 validation batch equals the serial reference fed with the same points, rebuilt here from the reference's
    flow2depth / depth2pc / perspective on the same tensors."""
    from gps_gaussian_b200 import harness, synth_dataset
    res = 256
    root = str(tmp_path / "data")
    synth_dataset.write_dataset(root, n_train=2, n_val=2, res=res, hr=False)
    st = harness.Stage1State(harness.load_cfg(root, stage=1, src_res=res, num_steps=3, batch_size=2))
    from lib.utils import depth2pc, flow2depth, get_novel_calib_for_show, perspective
    data = st.batch(0)
    st.model.eval()
    with torch.no_grad():
        data, _, _ = st.model(data, is_train=False)
        data = get_novel_calib_for_show(data, ratio=0.5)
        # the points flow2render builds (lib/TaichiRender.py:27-51), before it runs
        calib = torch.matmul(data['novel_view']['intr'], data['novel_view']['extr'])
        B = calib.shape[0]
        inputs = []
        for view in ('lmain', 'rmain'):
            d = data[view]
            depth_pred = flow2depth(d).clone()
            valid = (depth_pred != 0).view(B, -1, 1).squeeze(2)
            pts = depth2pc(depth_pred, d['extr'], d['intr'])
            pv = torch.zeros_like(pts)
            pv[valid] = pts[valid]
            pv = perspective(pv, calib)
            pv[:, :, 2:] = 1.0 / (pv[:, :, 2:] + 1e-8)
            img = torch.zeros_like(pv)
            img[valid] = d['img'].permute(0, 2, 3, 1).reshape(B, -1, 3)[valid]
            inputs.append((torch.cat((pv, img), 2).cpu().numpy(), valid.view(B, -1, 1).float().cpu().numpy()))
        data = st.render.flow2render(data)
    got = data['novel_view']['img_pred'].cpu().numpy()
    rd, rc = fresh_buffers(B, res)
    for pts, mask in inputs:
        splat_serial(pts, mask, rd, rc, B=1, N=res * res)                 # TaichiRenderBatch(bs=1): sample 0 only
    assert B == 2 and got.shape == rc.shape
    assert got.tobytes() == rc.tobytes()
    assert (rc[0] != -1).mean() > 0.05 and (rc[1] == -1).all()
    print(f"flow2render: {int((rc[0, 0] != -1).sum())} of {res * res} pixels drawn, bit-identical to the serial reference")
