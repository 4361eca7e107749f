"""Rectification on the device (csrc/rectify.cu through gps_gaussian_b200.rectify) is bit-identical to the CPU path:
against the goldens, against the numpy oracle on a seeded sweep up to a 1024^2 pair, against the reference's own loader
functions, and end to end through the unmodified test_real_data.py and the rectified_local/ cache with GPSG_RECTIFY=1.
Every output buffer is poisoned (0xAB bytes, NaN for floats) before the launch, so an unwritten pixel cannot pass."""
import filecmp
import glob
import os
import shutil
import subprocess
import sys
import types

import numpy as np
import pytest
import torch

from gps_gaussian_b200 import harness, rectify
from oracle import rectify_oracle as ro

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import rectify_cases  # noqa: E402

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "rectify_golden.npz")
needs_ref = pytest.mark.skipif(harness.staged_reference() is None, reason="oracle/_ref not staged")


@pytest.fixture(autouse=True)
def poisoned(monkeypatch):
    def empty(shape, dtype, device):
        t = torch.empty(shape, dtype=dtype, device=device)
        t.view(torch.uint8).fill_(0xAB) if dtype == torch.uint8 else t.fill_(float("nan"))
        return t
    monkeypatch.setattr(rectify, "_empty", empty)


def _same(a, b):
    return a.dtype == b.dtype and a.shape == b.shape and a.tobytes() == b.tobytes()


def _host(out):
    return [{k: v.cpu().contiguous().numpy() for k, v in o.items()} for o in out]


def _golden(name):
    g = np.load(GOLDEN)
    return {k.split("/", 1)[1]: g[k] for k in g.files if k.startswith(name + "/")}


@pytest.mark.parametrize("name", ["ring", "wide", "nonsquare", "empty"])
def test_device_equals_goldens(name):
    g = _golden(name)
    cams = [(g[f"K{k}"], g[f"R{k}"], g[f"P{k}"]) for k in range(2)]
    depths = (g["depth0"], g["depth1"]) if "depth0" in g else None
    out = _host(rectify.rectify_device([(g[f"in_img{k}"], g[f"in_mask{k}"]) for k in range(2)], cams, int(g["src_res"]),
                                       depths=depths, Tf_x=g["Tf_x"], numpy_out=True, tensor_out=True))
    for k in range(2):
        assert _same(out[k]["img"], g[f"img{k}"]) and _same(out[k]["mask"], g[f"mask{k}"]), (name, k)
        assert _same(out[k]["img_t"], g[f"img_t{k}"]) and _same(out[k]["mask_t"], g[f"mask_t{k}"]), (name, k)
        if depths is not None:
            assert _same(out[k]["flow"], g[f"flow{k}"]) and _same(out[k]["valid"], g[f"valid{k}"]), (name, k)


SWEEP = [(0, 1024, 1024, 1024, 3, 3, 22.5, 0.0), (1, 256, 256, 256, 1, 1, 60.0, 8.0), (2, 200, 320, 256, 4, 4, 22.5, 3.0),
         (3, 256, 256, 192, 3, 1, 30.0, 0.0), (4, 512, 512, 512, 4, 1, 22.5, 0.0)]


@pytest.mark.parametrize("seed,Hin,Win,res,C,Cm,angle,tilt", SWEEP)
def test_device_equals_oracle_sweep(seed, Hin, Win, res, C, Cm, angle, tilt):
    pytest.importorskip("cv2")
    views = rectify_cases.pair(seed, Hin, Win, angle=angle, tilt=tilt, C=C, Cm=Cm)
    R0, R1, P0, P1 = rectify_cases.stereo_rectify(views[0][2], views[0][3], views[1][2], views[1][3], res)
    rng = np.random.default_rng(seed)
    depths = [rng.uniform(-0.1, 3.0, (Hin, Win)).astype(np.float32) for _ in range(2)]
    Tf_x = np.array(-float(P1[0, 0]) * 0.3 * (seed + 1))
    cams = [(views[0][2], R0, P0), (views[1][2], R1, P1)]
    out = _host(rectify.rectify_device([(v[0], v[1]) for v in views], cams, res, depths=depths, Tf_x=Tf_x,
                                       numpy_out=True, tensor_out=True))
    want = ro.rectify_pair([(v[0], v[1]) for v in views], [(c[0], c[1], c[2][:3, :3]) for c in cams] + [Tf_x], res,
                           depths)
    for k in range(2):
        for key in ("img", "mask", "flow", "valid"):
            w = want[f"{key}{k}"]
            assert _same(out[k][key], w.reshape(out[k][key].shape) if w.ndim == 3 and w.shape[2] == 1 else w), (k, key)
        mx, my = ro.rectify_maps(cams[k][0], cams[k][1], cams[k][2][:3, :3], res, res)
        assert _same(out[k]["depth"], ro.remap_f32(depths[k], mx, my)), k
        img_t, mask_t = ro.tensor_contract(want[f"img{k}"].reshape(res, res, C), want[f"mask{k}"].reshape(res, res, Cm))
        assert _same(out[k]["img_t"], img_t) and _same(out[k]["mask_t"], mask_t), k
    # the wide / tilted cameras leave the source: the border pixels are the constant 0
    if angle >= 60:
        assert (out[0]["img"] == 0).any() or (out[1]["img"] == 0).any()


def _reference_pair(hl, seed, S, with_pts):
    views = rectify_cases.pair(seed, S, S, angle=22.5)
    rng = np.random.default_rng(seed)
    return [(img, mask, K, E, hl.depth2pts(torch.FloatTensor(rectify_cases.inv_depth(S, rng)), torch.FloatTensor(E),
                                          torch.FloatTensor(K)) if with_pts else None) for img, mask, K, E in views]


@needs_ref
@pytest.mark.parametrize("with_pts", [False, True])
def test_numpy_and_tensor_contract_equal_reference(with_pts):
    pytest.importorskip("cv2")
    harness.add_reference_to_path()
    from lib import human_loader as hl
    S = 256
    data = _reference_pair(hl, 31, S, with_pts)
    me = types.SimpleNamespace(opt=types.SimpleNamespace(src_res=S))
    want = hl.StereoHumanDataset.get_rectified_stereo_data(me, data[0], data[1])
    got = rectify.rectify_stereo(data[0], data[1], S, pts2depth=hl.pts2depth)
    assert list(got) == list(want)
    for k, v in want.items():
        if k == "camera":
            assert all(_same(got[k][c], v[c]) for c in v)
        else:
            assert _same(got[k], v), k
    want_t = hl.StereoHumanDataset.stereo_to_dict_tensor(me, want, "s")
    got_t = rectify.stereo_item_cuda(data[0], data[1], S, "s", pts2depth=hl.pts2depth)
    assert got_t["name"] == "s"
    for view in ("lmain", "rmain"):
        assert list(got_t[view]) == list(want_t[view])
        for key, w in want_t[view].items():
            g = got_t[view][key]
            assert g.is_cuda == (key in ("img", "mask")), key
            assert g.dtype == w.dtype and g.shape == w.shape and g.stride() == w.stride(), key
            assert _same(g.cpu().numpy(), w.numpy()), (view, key)


RES = 128


@pytest.fixture(scope="module")
def dataset(tmp_path_factory):
    from gps_gaussian_b200 import synth_dataset
    root = str(tmp_path_factory.mktemp("rectifydata"))
    synth_dataset.write_dataset(root, n_train=2, n_val=2, res=RES, hr=True)
    return root


def _run(work, args, rectify_on):
    env = harness.script_env(patch=True, extra={"GPSG_RECTIFY": "1"} if rectify_on else None)
    if not rectify_on:
        env.pop("GPSG_RECTIFY", None)
    return subprocess.run([sys.executable, "-c", harness.SCRIPT_RUNNER] + args, cwd=work, env=env, text=True,
                          capture_output=True, timeout=900)


@needs_ref
def test_real_data_script_jpegs_identical_with_switch(dataset, tmp_path):
    """test_real_data.py, unmodified, with GPSG_PATCH=1 and with GPSG_PATCH=1 GPSG_RECTIFY=1: the same JPEG bytes.  The
    checkpoint is a freshly initialised model (seeded), saved as train_stage2.py saves one."""
    pytest.importorskip("cv2")
    cfg = harness.load_cfg(dataset, src_res=RES)
    from lib.network import RtStereoHumanModel
    torch.manual_seed(7)
    ckpt = str(tmp_path / "init.pth")
    torch.save({"network": RtStereoHumanModel(cfg, with_gs_render=True).state_dict()}, ckpt)
    outs = {}
    for on in (False, True):
        work = harness.make_workdir(str(tmp_path / f"work{int(on)}"), dataset, src_res=RES)
        p = _run(work, ["test_real_data.py", "--test_data_root", os.path.join(dataset, "val"), "--ckpt_path", ckpt,
                        "--src_view", "0", "1"], on)
        assert p.returncode == 0, p.stdout[-3000:] + p.stderr[-6000:]
        outs[on] = sorted(glob.glob(os.path.join(work, "test_out", "*_novel.jpg")))
        assert len(outs[on]) == 2, outs[on]
    for a, b in zip(outs[False], outs[True]):
        assert os.path.basename(a) == os.path.basename(b)
        assert filecmp.cmp(a, b, shallow=False), (a, b)


_CACHE = ("from config.stereo_human_config import ConfigStereoHuman\n"
          "from lib.human_loader import StereoHumanDataset\n"
          "c = ConfigStereoHuman(); c.load('config/stage2.yaml'); c = c.get_cfg()\n"
          "StereoHumanDataset(c.dataset, phase='train')\n")


@needs_ref
def test_rectified_cache_identical_with_switch(dataset, tmp_path):
    """StereoHumanDataset(..., use_processed_data=True) writes rectified_local/: byte-identical files either way."""
    pytest.importorskip("cv2")
    trees = {}
    for on in (False, True):
        root = str(tmp_path / f"data{int(on)}")
        shutil.copytree(dataset, root)
        work = harness.make_workdir(str(tmp_path / f"cwork{int(on)}"), root, src_res=RES, use_processed_data=True)
        with open(os.path.join(work, "make_cache.py"), "w") as f:
            f.write(_CACHE)
        p = _run(work, ["make_cache.py"], on)
        assert p.returncode == 0, p.stdout[-3000:] + p.stderr[-6000:]
        base = os.path.join(root, "rectified_local")
        trees[on] = {os.path.relpath(f, base): f for f in glob.glob(os.path.join(base, "**", "*"), recursive=True)
                     if os.path.isfile(f)}
    assert sorted(trees[False]) == sorted(trees[True]) and len(trees[False]) >= 2 * 9
    for rel, f in trees[False].items():
        assert filecmp.cmp(f, trees[True][rel], shallow=False), rel
