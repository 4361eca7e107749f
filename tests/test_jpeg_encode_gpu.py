"""GPU: the JPEG encoder (csrc/jpeg_encode.cu) writes the committed cv2 files byte for byte through the raw ABI (poisoned
outputs framed by guard bytes, one image per call and mixed batches, reruns identical); large sizes, pitched inputs and
both channel orders against the serial oracle; our decoder reads every file back as Pillow does; the unmodified
dataset renderer and inference scripts write identical files with and without GPSG_ENCODE=1."""
import ctypes as C
import filecmp
import glob
import hashlib
import importlib.util
import io
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from gps_gaussian_b200 import harness, jpeg
from oracle import jpeg_encode_oracle as oracle

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
GUARD = 64


def _corpus():
    path = os.path.join(HERE, "golden", "jpeg_encode", "make_jpeg_encode_corpus.py")
    spec = importlib.util.spec_from_file_location("make_jpeg_encode_corpus", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


K = _corpus()
MANIFEST = K.manifest()
NAMES = sorted(K.cases())


def _sha(data):
    return hashlib.sha256(data).hexdigest()


def _dev(img):
    return torch.from_numpy(np.ascontiguousarray(img)).cuda()


def _raw(items):
    """gpsg_jpeg_encode over [(device image, quality, sampling, order)] in one call, each output poisoned and framed by
    guard bytes; returns the files after checking that nothing outside them was written."""
    n = len(items)
    descs, srcs = [], []
    for t, q, s, order in items:
        t = t.contiguous()
        nc = 1 if t.dim() == 2 else 3
        descs.append(jpeg.JpegEncodeDesc(t.shape[1], t.shape[0], nc, jpeg.ORDERS[order], q, int(s), t.shape[1] * nc))
        srcs.append(t)
    arr = (jpeg.JpegEncodeDesc * n)(*descs)
    caps = [int(jpeg._L.gpsg_jpeg_encode_max_bytes(C.byref(d))) for d in descs]
    offs = np.cumsum([0] + [c + 2 * GUARD for c in caps])
    blob = torch.full((int(offs[-1]),), 0xCD, dtype=torch.uint8, device="cuda")
    for i in range(n):
        blob[int(offs[i]):int(offs[i]) + GUARD] = 0xA5
        blob[int(offs[i + 1]) - GUARD:int(offs[i + 1])] = 0xA5
    sizes = torch.full((n,), -1, dtype=torch.int64, device="cuda")
    wsb = int(jpeg._L.gpsg_jpeg_encode_workspace_bytes(n, arr))
    ws = torch.full((wsb + 256,), 0xEE, dtype=torch.uint8, device="cuda")
    base = (ws.data_ptr() + 255) // 256 * 256
    src_p = (C.c_void_p * n)(*[t.data_ptr() for t in srcs])
    out_p = (C.c_void_p * n)(*[blob.data_ptr() + int(offs[i]) + GUARD for i in range(n)])
    idx, stream = jpeg._lib.device_stream(torch.device("cuda"))
    rc = jpeg._L.gpsg_jpeg_encode(idx, stream, n, arr, src_p, out_p, sizes.data_ptr(), base, wsb)
    assert rc == 0, jpeg._L.gpsg_last_error()
    torch.cuda.synchronize()
    host, got = blob.cpu().numpy(), sizes.cpu().tolist()
    files = []
    for i in range(n):
        o = int(offs[i])
        assert 0 < got[i] <= caps[i]
        assert (host[o:o + GUARD] == 0xA5).all() and (host[int(offs[i + 1]) - GUARD:int(offs[i + 1])] == 0xA5).all()
        assert (host[o + GUARD + got[i]:int(offs[i + 1]) - GUARD] == 0xCD).all()      # nothing past the file
        files.append(host[o + GUARD:o + GUARD + got[i]].tobytes())
    return files


def _fixture_item(name):
    q, s = K.params(name)
    return _dev(K.image(name)), q, s, "bgr"


def test_fixtures_one_image_per_call():
    for name in NAMES:
        got, = _raw([_fixture_item(name)])
        assert _sha(got) == MANIFEST["files"][name], name


def test_fixtures_as_mixed_batches_and_reruns_identical():
    rng = np.random.default_rng(0)
    order = [NAMES[i] for i in rng.permutation(len(NAMES))]
    for chunk in (order[:64], order[64:]):
        items = [_fixture_item(n) for n in chunk]
        first = _raw(items)
        assert [_sha(f) for f in first] == [MANIFEST["files"][n] for n in chunk]
        assert _raw(items) == first


@pytest.mark.parametrize("hw", [(1024, 1024), (2048, 2048), (1023, 1025), (2047, 2049)])
def test_large_sizes(hw):
    h, w = hw
    items = []
    for lay in K.LAYOUTS:
        img = K.smooth(h, w, lay, 12) if lay != "420" else K.noise(h, w, lay, 13)
        items.append((img, 95 if lay != "444" else 100, "420" if lay == "gray" else lay))
    got = _raw([(_dev(img), q, s, "bgr") for img, q, s in items])
    for (img, q, s), data in zip(items, got):
        assert data == oracle.encode(img, q, s, order="bgr"), (hw, s)
    if K.versions() == MANIFEST["versions"]:
        img, q, s = items[3]
        assert got[3] == K.cv2_encode(img, q, s)


def test_pitched_inputs_and_both_orders():
    img = K.noise(45, 70, "420", 21)
    wide = torch.zeros(45, 96, 3, dtype=torch.uint8, device="cuda")
    wide[:, 13:83] = _dev(img)
    view = wide[:, 13:83]                         # row pitch 288 bytes, not 210
    assert view.stride(0) == 288
    for s in ("444", "422", "420"):
        want = oracle.encode(img, 90, s, order="bgr")
        assert jpeg.encode(view, 90, s, order="bgr") == want
        assert jpeg.encode(_dev(img[:, :, ::-1]), 90, s) == want                 # order='rgb' is the default
    gray = torch.zeros(33, 50, dtype=torch.uint8, device="cuda")
    gray[:, 3:40] = _dev(K.noise(33, 37, "gray", 2))
    assert jpeg.encode(gray[:, 3:40], 75) == oracle.encode(K.noise(33, 37, "gray", 2), 75)
    assert jpeg.encode(gray[:, 3:40, None], 75) == oracle.encode(K.noise(33, 37, "gray", 2), 75)
    transposed = _dev(img).transpose(0, 1)        # non-unit inner strides: made contiguous first
    assert jpeg.encode(transposed, 90, order="bgr") == oracle.encode(img.transpose(1, 0, 2), 90, order="bgr")


def test_public_encode_lists_counts_and_imwrite(tmp_path):
    jpeg.reset_encode_counts()
    items = [_fixture_item(n) for n in NAMES[:70]]
    got = jpeg.encode([t for t, _, _, _ in items], 95, "420", order="bgr")        # two batches of <= 64
    for (t, _, _, _), data in zip(items, got):
        assert data == oracle.encode(t.cpu().numpy(), 95, "420", order="bgr")
    assert jpeg.encode_counts() == {"native": 70, "fallback": 0}
    img = K.smooth(64, 80, "444", 1)
    path = str(tmp_path / "x.jpg")
    assert jpeg.imwrite_cuda(path, _dev(img[:, :, ::-1]), quality=88, subsampling="422")
    assert open(path, "rb").read() == oracle.encode(img, 88, "422", order="bgr")
    assert jpeg.encode_host(img[:, :, ::-1], 88, "422", order="rgb") == oracle.encode(img, 88, "422", order="bgr")


def test_rebound_imwrite_from_threads_writes_each_threads_image(tmp_path, monkeypatch):
    """Two threads write different images through the rebound cv2.imwrite at once (cv2 releases the GIL, and so does
    the GPU route while it waits); every file must be cv2's file of that thread's image."""
    import threading
    cv2 = pytest.importorskip("cv2")
    from gps_gaussian_b200 import patch
    monkeypatch.setenv("GPSG_ENCODE", "1")
    patch.uninstall()
    patch.install()
    try:
        orig = cv2.imwrite._gpsg_original
        imgs = [K.smooth(600, 640, "420", 30 + k)[:, :, ::-1] for k in range(2)]
        want = [oracle.encode(im, 95, "420", order="bgr") for im in imgs]
        jpeg.reset_encode_counts()
        errors = []

        def writer(k):
            try:
                for i in range(12):
                    assert cv2.imwrite(str(tmp_path / f"t{k}_{i}.jpg"), imgs[k]) is True
            except Exception as e:   # noqa: BLE001 -- reported below
                errors.append(e)
        threads = [threading.Thread(target=writer, args=(k,)) for k in range(2)]
        for t in threads:
            t.start()
        for t in threads:
            t.join()
        assert not errors, errors
        assert jpeg.encode_counts()["native"] == 24
        for k in range(2):
            for i in range(12):
                assert open(tmp_path / f"t{k}_{i}.jpg", "rb").read() == want[k], (k, i)
        assert orig is not cv2.imwrite
    finally:
        patch.uninstall()


def test_round_trip_through_our_decoder():
    from PIL import Image
    names = [n for n in NAMES if not n.startswith("size_1023")] + ["size_1023x1025_420"]
    files = [_raw([_fixture_item(n)])[0] for n in names]
    for name, data, img in zip(names, files, jpeg.decode(files)):
        assert np.array_equal(img.cpu().numpy(), np.array(Image.open(io.BytesIO(data)))), name


# ---- the unmodified scripts --------------------------------------------------------------------------------------------
needs_ref = pytest.mark.skipif(harness.staged_reference() is None, reason="oracle/_ref not staged")
_COUNT = ("\nm = sys.modules.get('gps_gaussian_b200.jpeg')\n"
          "print('ENCODE_COUNTS', m.encode_counts() if m else None)\n")


def _test_mesh_render_gpu():
    spec = importlib.util.spec_from_file_location("_mesh_render_gpu", os.path.join(HERE, "test_mesh_render_gpu.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _counts(stdout):
    line = [ln for ln in stdout.splitlines() if ln.startswith("ENCODE_COUNTS")][-1]
    return eval(line.split(" ", 1)[1])


@needs_ref
def test_render_data_identical_with_and_without_encode(tmp_path):
    """render_data.py as `python render_data.py` runs it (its directory first on sys.path), with the test_mesh_render_gpu
    scan tree; every JPEG (2 scans x 16 poses x (5 views + 3 _hr views)) takes the native route with the switch."""
    pytest.importorskip("cv2")
    mr = _test_mesh_render_gpu()
    script = os.path.join(harness.staged_reference(), "prepare_data", "render_data.py")
    runner = ("import os, runpy, sys\nsys.argv = sys.argv[1:]\nsys.path.insert(0, os.path.dirname(sys.argv[0]))\n"
              "runpy.run_path(sys.argv[0], run_name='__main__')\n") + _COUNT
    trees = {}
    for on in (False, True):
        work = str(tmp_path / f"work{int(on)}")
        mr._scan_tree(work)
        env = harness.script_env(patch=True)
        env.pop("GPSG_ENCODE", None)
        if on:
            env["GPSG_ENCODE"] = "1"
        p = subprocess.run([sys.executable, "-c", runner, script], cwd=work, env=env, text=True, capture_output=True,
                           timeout=1800)
        assert p.returncode == 0, p.stdout[-3000:] + p.stderr[-6000:]
        counts = _counts(p.stdout)
        if on:
            assert counts["native"] == 2 * 16 * (5 + 3), counts
        else:
            assert counts is None or counts["native"] == 0, counts
        trees[on] = os.path.join(work, "PATH", "TO", "SAVE", "RENDERED", "DATA")
    files = sorted(os.path.relpath(os.path.join(d, f), trees[False]) for d, _, fs in os.walk(trees[False]) for f in fs)
    assert len(files) == 2 * 16 * (8 + 5 + 5 + 10)
    for rel in files:
        assert filecmp.cmp(os.path.join(trees[False], rel), os.path.join(trees[True], rel), shallow=False), rel


RES = 128
_NO_THRESHOLD = "import gps_gaussian_b200.patch as _p\n_p._MIN_NATIVE_PIXELS = 0\n"


@pytest.fixture(scope="module")
def dataset(tmp_path_factory):
    from gps_gaussian_b200 import synth_dataset
    root = str(tmp_path_factory.mktemp("encdata"))
    synth_dataset.write_dataset(root, n_train=2, n_val=2, res=RES, hr=True)
    return root


@needs_ref
@pytest.mark.parametrize("script", ["test_real_data.py", "test_view_interp.py"])
def test_inference_scripts_identical_with_and_without_encode(dataset, tmp_path, script):
    pytest.importorskip("cv2")
    cfg = harness.load_cfg(dataset, src_res=RES)
    from lib.network import RtStereoHumanModel
    torch.manual_seed(7)
    ckpt = str(tmp_path / "init.pth")
    torch.save({"network": RtStereoHumanModel(cfg, with_gs_render=True).state_dict()}, ckpt)
    args = ["--test_data_root", os.path.join(dataset, "val"), "--ckpt_path", ckpt]
    args += ["--src_view", "0", "1"] if script == "test_real_data.py" else ["--novel_view_nums", "2"]
    outs = {}
    for on in (False, True):
        work = harness.make_workdir(str(tmp_path / f"work{int(on)}"), dataset, src_res=RES)
        env = harness.script_env(patch=True, extra={"GPSG_RECTIFY": "1"})
        env.pop("GPSG_ENCODE", None)
        if on:
            env["GPSG_ENCODE"] = "1"
        # the test frames (RES^2) are below the size threshold: lower it in the script's process so they take the route
        runner = _NO_THRESHOLD + harness.SCRIPT_RUNNER + _COUNT
        p = subprocess.run([sys.executable, "-c", runner, script] + args, cwd=work, env=env,
                           text=True, capture_output=True, timeout=900)
        assert p.returncode == 0, p.stdout[-3000:] + p.stderr[-6000:]
        out_dir = "test_out" if script == "test_real_data.py" else "interp_out"
        outs[on] = sorted(glob.glob(os.path.join(work, out_dir, "*.jpg")))
        assert len(outs[on]) >= 2, outs[on]
        counts = _counts(p.stdout)
        if on:
            assert counts["native"] == len(outs[on]), counts
        else:
            assert counts is None or counts["native"] == 0, counts
    assert [os.path.basename(a) for a in outs[False]] == [os.path.basename(b) for b in outs[True]]
    for a, b in zip(outs[False], outs[True]):
        assert filecmp.cmp(a, b, shallow=False), (a, b)
