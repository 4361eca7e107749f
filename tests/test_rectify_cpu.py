"""Rectification without a GPU: the numpy oracle (oracle/rectify_oracle.py) against cv2 and the goldens, the whole oracle
dict against the reference's own loader functions, and the GPSG_RECTIFY switch of the patch."""
import os
import subprocess
import sys
import types

import numpy as np
import pytest
import torch

from gps_gaussian_b200 import harness, patch
from oracle import rectify_oracle as ro

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import rectify_cases  # noqa: E402

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "rectify_golden.npz")
CASES = ("ring", "wide", "nonsquare", "empty")
needs_ref = pytest.mark.skipif(harness.staged_reference() is None, reason="oracle/_ref not staged")


def _golden(name):
    g = np.load(GOLDEN)
    return {k.split("/", 1)[1]: g[k] for k in g.files if k.startswith(name + "/")}


def _oracle_from_golden(g):
    cams = [(g["K0"], g["R0"], g["P0"][:3, :3]), (g["K1"], g["R1"], g["P1"][:3, :3]), g["Tf_x"]]
    depths = (g["depth0"], g["depth1"]) if "depth0" in g else None
    return ro.rectify_pair(((g["in_img0"], g["in_mask0"]), (g["in_img1"], g["in_mask1"])), cams, int(g["src_res"]), depths)


def _same(a, b):
    """Bit-identical arrays: dtype, shape and bytes (so -0 vs +0 and NaN payloads count)."""
    return a.dtype == b.dtype and a.shape == b.shape and a.tobytes() == b.tobytes()


# ---- rules 1-4 against cv2 ---------------------------------------------------------------------------------------
SWEEP = [(s, res, ang, tilt) for s in range(3) for res, ang, tilt in ((128, 22.5, 0.0), (256, 60.0, 8.0), (512, 22.5, 3.0))]


@pytest.mark.parametrize("seed,res,angle,tilt", SWEEP)
def test_oracle_equals_cv2_rules(seed, res, angle, tilt):
    cv2 = pytest.importorskip("cv2")
    views = rectify_cases.pair(seed, res, res, angle=angle, tilt=tilt)
    R0, R1, P0, P1 = rectify_cases.stereo_rectify(views[0][2], views[0][3], views[1][2], views[1][3], res)
    rng = np.random.default_rng(seed)
    for (img, mask, K, _), R, P in zip(views, (R0, R1), (P0, P1)):
        cx, cy = cv2.initUndistortRectifyMap(K, np.zeros(4), R, P, (res, res), cv2.CV_32FC1)
        ox, oy = ro.rectify_maps(K, R, P[:3, :3], res, res)
        # rule 1: the fixed point that decides every tap is identical; the fp32 maps may differ in rare ulps
        assert np.array_equal(ro.fixed_point(cx), ro.fixed_point(ox)) and np.array_equal(ro.fixed_point(cy), ro.fixed_point(oy))
        assert np.abs(cx.astype(np.float64) - ox).max() <= np.spacing(np.abs(ox).max()) and (cx != ox).mean() < 1e-4
        for C in (1, 3, 4):                                              # rule 2
            src = rng.integers(0, 256, (res, res, C), dtype=np.uint8)
            want = cv2.remap(src, cx, cy, cv2.INTER_LINEAR)
            got = ro.remap_u8(src, cx, cy)
            assert _same(want, got.reshape(want.shape)), C
        d = rng.uniform(0, 3, (res, res)).astype(np.float32)             # rule 3
        assert _same(cv2.remap(d, cx, cy, cv2.INTER_LINEAR), ro.remap_f32(d, cx, cy))
        v = (rng.integers(0, 256, (res, res)) / 255.0).astype(np.float32)  # rule 4
        assert _same(cv2.erode(v, np.ones((3, 3), np.uint8), 1), ro.erode3(v))


def test_remap_f32_order_is_load_bearing():
    """Summing the four products in pairs instead of left to right changes results: the order in rule 3 is needed."""
    rng = np.random.default_rng(3)
    views = rectify_cases.pair(3, 128, 128)
    K, E = views[0][2], views[0][3]
    mx, my = ro.rectify_maps(K, np.eye(3), K, 128, 128)
    mx = mx + rng.uniform(-3, 3, mx.shape).astype(np.float32)
    my = my + rng.uniform(-3, 3, my.shape).astype(np.float32)
    d = rng.uniform(0, 3, (128, 128)).astype(np.float32)
    ax, ay, taps = ro._taps(mx, my, 128, 128)
    f = np.float32
    tx, ty = ax.astype(f) / f(32), ay.astype(f) / f(32)
    w = [(f(1) - ty) * (f(1) - tx), (f(1) - ty) * tx, ty * (f(1) - tx), ty * tx]
    p = [np.where(inside, d[ys, xs], f(0)) * wk for wk, (ys, xs, inside) in zip(w, taps)]
    assert (((p[0] + p[1]) + (p[2] + p[3])) != ro.remap_f32(d, mx, my)).any()


# ---- goldens -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", CASES)
def test_oracle_equals_goldens(name):
    g = _golden(name)
    got = _oracle_from_golden(g)
    for k, v in got.items():
        assert _same(v, g[k]), (name, k)
    assert ("flow0" in got) == ("flow0" in g)
    for k in range(2):
        img_t, mask_t = ro.tensor_contract(got[f"img{k}"], got[f"mask{k}"])
        assert _same(img_t, g[f"img_t{k}"]) and _same(mask_t, g[f"mask_t{k}"]), (name, k)


def test_goldens_cover_the_issue_cases():
    ring, wide, nonsq, empty = (_golden(n) for n in CASES)
    assert not np.array_equal(ring["K0"], ring["K1"])
    for k in range(2):                                               # maps leave the source image: constant-0 border
        assert (wide[f"img{k}"].max(-1) == 0).any()
    assert nonsq["in_img0"].shape[:2] == (96, 160) and nonsq["img0"].shape[:2] == (128, 128)
    m = ring["mask0"][..., 0].astype(np.int64)
    assert ((m > 100) & (m < 150)).any() and ((m > 150) & (m < 190)).any()  # soft edges around 0.5 and 0.66 of 255
    assert (ring["depth0"] < 0.05).any() and (ring["depth0"] > 0.05).any() and (ring["flow0"] != 0).any()
    assert not empty["mask0"].any() and not empty["valid0"].any() and not np.abs(empty["flow0"]).any()


# ---- the whole dict against the reference's own functions ---------------------------------------------------------
@needs_ref
@pytest.mark.parametrize("with_pts", [False, True])
@pytest.mark.parametrize("seed", [21, 22])
def test_oracle_dict_equals_reference(seed, with_pts):
    pytest.importorskip("cv2")
    harness.add_reference_to_path()
    from lib import human_loader as hl
    from gps_gaussian_b200 import rectify
    S = 128
    views = rectify_cases.pair(seed, S, S, angle=22.5 + seed % 3)
    rng = np.random.default_rng(seed)
    data = [(img, mask, K, E, hl.depth2pts(torch.FloatTensor(rectify_cases.inv_depth(S, rng)), torch.FloatTensor(E),
                                          torch.FloatTensor(K)) if with_pts else None) for img, mask, K, E in views]
    me = types.SimpleNamespace(opt=types.SimpleNamespace(src_res=S))
    want = hl.StereoHumanDataset.get_rectified_stereo_data(me, data[0], data[1])
    camera, cams = rectify.stereo_rectify(data[0], data[1], S)
    assert camera.keys() == want["camera"].keys()
    for k in camera:
        assert _same(camera[k], want["camera"][k]), k
    depths = None
    if with_pts:
        depths = [hl.pts2depth(torch.FloatTensor(d[4]), torch.FloatTensor(camera[f"extr{k}"]),
                               torch.FloatTensor(camera[f"intr{k}"])).numpy() for k, d in enumerate(data)]
    got = ro.rectify_pair([(d[0], d[1]) for d in data], [(K, R, P[:3, :3]) for K, R, P in cams] + [camera["Tf_x"]], S,
                          depths)
    assert list(got) == [k for k in want if k != "camera"]
    for k, v in got.items():
        assert _same(v, want[k]), k
    item = hl.StereoHumanDataset.stereo_to_dict_tensor(me, want, "s")
    for k, view in enumerate(("lmain", "rmain")):
        img_t, mask_t = ro.tensor_contract(got[f"img{k}"], got[f"mask{k}"])
        assert _same(img_t, item[view]["img"].contiguous().numpy()) and _same(mask_t, item[view]["mask"].contiguous().numpy())


def test_cpu_torch_divides_uint8_by_255_exactly():
    """stereo_to_dict_tensor's `uint8 tensor / 255.0` is an fp32 division, not a multiply by the reciprocal: the
    device kernel divides (__fdiv_rn) because of this."""
    u = torch.arange(256, dtype=torch.uint8).repeat(64)
    got = (u / 255.0).numpy()
    v = np.tile(np.arange(256, dtype=np.float32), 64)
    assert _same(got, v / np.float32(255))
    assert not _same(got, v * np.float32(1 / 255.0))


# ---- the switch --------------------------------------------------------------------------------------------------
def _fake_loader():
    mod = types.ModuleType("lib.human_loader")

    class StereoHumanDataset:
        def get_rectified_stereo_data(self, main_view_data, ref_view_data):
            return "original rectify"

        def get_test_item(self, index, source_id):
            return "original test item"
    mod.StereoHumanDataset = StereoHumanDataset
    mod.pts2depth = None
    return mod


@pytest.fixture
def clean_patch():
    patch.uninstall()
    yield
    patch.uninstall()


@pytest.mark.parametrize("value", [None, "0", "1"])
def test_switch_binds_only_when_set(monkeypatch, clean_patch, value):
    mod = _fake_loader()
    cls = mod.StereoHumanDataset
    before = dict(cls.__dict__)
    monkeypatch.setitem(sys.modules, "lib.human_loader", mod)
    if value is None:
        monkeypatch.delenv("GPSG_RECTIFY", raising=False)
    else:
        monkeypatch.setenv("GPSG_RECTIFY", value)
    patch.install()
    bound = value == "1"
    assert patch.rectify() is bound
    for attr in ("get_rectified_stereo_data", "get_test_item"):
        assert (cls.__dict__[attr] is before[attr]) is not bound, attr
    patch.uninstall()
    for attr in ("get_rectified_stereo_data", "get_test_item"):
        assert cls.__dict__[attr] is before[attr]


@pytest.mark.parametrize("cuda", [False, True])
def test_switch_falls_back_in_worker_and_without_cuda(monkeypatch, clean_patch, cuda):
    """Inside a DataLoader worker, or without CUDA, the rebound methods call the reference's own."""
    mod = _fake_loader()
    monkeypatch.setitem(sys.modules, "lib.human_loader", mod)
    monkeypatch.setenv("GPSG_RECTIFY", "1")
    patch.install()
    monkeypatch.setattr(torch.cuda, "is_available", lambda: cuda)
    if cuda:                                          # a simulated forked worker: CUDA would be there but must not be used
        monkeypatch.setattr(torch.utils.data, "get_worker_info", lambda: types.SimpleNamespace(id=0, num_workers=2))
    ds = mod.StereoHumanDataset()
    assert ds.get_rectified_stereo_data(None, None) == "original rectify"
    assert ds.get_test_item(0, [0, 1]) == "original test item"


_PROBE = ("import lib.human_loader as h\n"
          "c = h.StereoHumanDataset\n"
          "print(c.get_rectified_stereo_data.__module__, c.get_test_item.__module__, type(h.__spec__.loader).__name__)\n")


@needs_ref
@pytest.mark.parametrize("rectify", [False, True])
def test_unmodified_loader_with_patch_alone(rectify):
    """The route the scripts take (dropin/sitecustomize.py with GPSG_PATCH=1): without GPSG_RECTIFY the reference's
    loader module is neither hooked nor changed; with it, both methods are ours."""
    pytest.importorskip("cv2")
    env = harness.script_env(patch=True, extra={"GPSG_RECTIFY": "1"} if rectify else None)
    if not rectify:
        env.pop("GPSG_RECTIFY", None)
    p = subprocess.run([sys.executable, "-c", _PROBE], cwd=harness.staged_reference(), env=env, text=True,
                       capture_output=True, timeout=300)
    assert p.returncode == 0, p.stderr[-3000:]
    mods = p.stdout.split()
    if rectify:
        assert mods[:2] == ["gps_gaussian_b200.patch"] * 2 and mods[2] == "_PatchingLoader"
    else:
        assert mods[:2] == ["lib.human_loader"] * 2 and mods[2] != "_PatchingLoader"
