"""CPU: the serial JPEG encoder oracle against the committed cv2 files, live cv2 and Pillow byte for byte; the quantiser
the kernels rely on; the ABI's refusals; the GPSG_ENCODE switch and its routing rules against a fake encoder."""
import ctypes as C
import hashlib
import importlib.util
import io
import os
import sys

import numpy as np
import pytest

from gps_gaussian_b200 import jpeg, patch
from oracle import jpeg_encode_oracle as oracle

cv2 = pytest.importorskip("cv2")
Image = pytest.importorskip("PIL.Image")
HERE = os.path.dirname(os.path.abspath(__file__))


def _corpus():
    path = os.path.join(HERE, "golden", "jpeg_encode", "make_jpeg_encode_corpus.py")
    spec = importlib.util.spec_from_file_location("make_jpeg_encode_corpus", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


K = _corpus()
MANIFEST = K.manifest()
LIVE = K.versions() == MANIFEST["versions"]
PIL_SUBSAMPLING = {"444": 0, "422": 1, "420": 2}


def _sha(data):
    return hashlib.sha256(data).hexdigest()


def _pil(rgb, quality, subsampling):
    """Pillow's file; a gray image gets Pillow's default subsampling (an explicit one would be written into its SOF0)."""
    b = io.BytesIO()
    kw = {} if rgb.ndim == 2 else dict(subsampling=PIL_SUBSAMPLING[subsampling])
    Image.fromarray(rgb).save(b, "JPEG", quality=quality, **kw)
    return b.getvalue()


# ---- the oracle against cv2 --------------------------------------------------------------------------------------------
def test_fixtures_are_pinned():
    names = sorted(K.cases())
    assert sorted(MANIFEST["files"]) == names
    for name in names:
        if K.committed(name):
            assert _sha(K.load(name)) == MANIFEST["files"][name], name


@pytest.mark.parametrize("name", sorted(K.cases()))
def test_oracle_equals_committed_files(name):
    got = oracle.encode(K.image(name), *K.params(name), order="bgr")
    assert _sha(got) == MANIFEST["files"][name]


@pytest.mark.skipif(not LIVE, reason="the installed cv2 / libjpeg-turbo is not the one the fixtures came from")
@pytest.mark.parametrize("kind", ["noise", "smooth"])
@pytest.mark.parametrize("layout", K.LAYOUTS)
def test_oracle_equals_live_cv2_every_quality(kind, layout):
    img = K.KINDS[kind](19, 27, layout, 11)
    sub = "420" if layout == "gray" else layout
    for q in range(1, 101):
        assert oracle.encode(img, q, sub, order="bgr") == K.cv2_encode(img, q, sub), q


@pytest.mark.skipif(not LIVE, reason="the installed cv2 / libjpeg-turbo is not the one the fixtures came from")
@pytest.mark.parametrize("seed", range(4))
def test_oracle_equals_live_cv2_random_sizes(seed):
    rng = np.random.default_rng(100 + seed)
    for _ in range(12):
        h, w = (int(v) for v in rng.integers(1, 70, 2))
        layout = K.LAYOUTS[int(rng.integers(0, 4))]
        q = int(rng.integers(1, 101))
        img = K.noise(h, w, layout, int(rng.integers(1 << 30)))
        sub = "420" if layout == "gray" else layout
        assert oracle.encode(img, q, sub, order="bgr") == K.cv2_encode(img, q, sub), (h, w, layout, q)


@pytest.mark.parametrize("name", [n for n in sorted(K.cases()) if not n.startswith("size_1023")])
def test_pillow_writes_the_same_bytes(name):
    img = K.image(name)
    q, sub = K.params(name)
    rgb = img if img.ndim == 2 else np.ascontiguousarray(img[:, :, ::-1])
    assert _pil(rgb, q, sub) == oracle.encode(rgb, q, sub, order="rgb") == oracle.encode(img, q, sub, order="bgr")


def test_orders_and_strides():
    img = K.noise(21, 30, "420", 4)
    want = oracle.encode(img, 90, "422", order="bgr")
    assert oracle.encode(img[:, :, ::-1], 90, "422", order="rgb") == want
    big = np.zeros((21, 40, 3), np.uint8)
    big[:, 5:35] = img
    assert oracle.encode(big[:, 5:35], 90, "422", order="bgr") == want


# ---- extremes ----------------------------------------------------------------------------------------------------------
def _parse_huffman(data):
    """{(class, id): {symbol: code length}} from the DHT segments of a file, and the offset of its scan data."""
    tables, i = {}, 2
    while True:
        m, ln = data[i + 1], (data[i + 2] << 8) | data[i + 3]
        if m == 0xC4:
            seg = data[i + 4:i + 2 + ln]
            counts, syms = seg[1:17], seg[17:]
            lens, k = {}, 0
            for L, n in enumerate(counts, 1):
                for _ in range(n):
                    lens[syms[k]] = L
                    k += 1
            tables[(seg[0] >> 4, seg[0] & 15)] = lens
        if m == 0xDA:
            return tables, i + 2 + ln
        i += 2 + ln


def _scan_bits(data, coef, nc, bpm, comp_of_block):
    """Bits of the entropy-coded segment, counted from the coefficients and the file's own code lengths."""
    tables, _ = _parse_huffman(data)
    cat = lambda v: int(abs(int(v))).bit_length()
    pred, bits = [0, 0, 0], 0
    for b, z in enumerate(coef):
        c = comp_of_block[b % bpm]
        dc, ac = tables[(0, min(c, 1))], tables[(1, min(c, 1))]
        s = cat(z[0] - pred[c])
        pred[c] = int(z[0])
        bits += dc[s] + s
        run = 0
        for v in z[1:]:
            if v == 0:
                run += 1
                continue
            while run > 15:
                bits += ac[0xF0]
                run -= 16
            bits += ac[run << 4 | cat(v)] + cat(v)
            run = 0
        if run:
            bits += ac[0]
    return bits


def test_padded_last_byte_is_stuffed():
    img = K.image("ffpad_gray")
    data, _, coef = oracle.encode(img, 95, stages=True)
    assert data == K.load("ffpad_gray")
    assert data[-4:] == b"\xff\x00\xff\xd9"
    bits = _scan_bits(data, coef, 1, 1, [0])
    assert bits % 8 != 0                      # the final 0xFF is partly padding
    _, start = _parse_huffman(data)
    assert len(data) - 2 - start - data[start:-2].count(b"\xff\x00") == (bits + 7) // 8


def _longest_run_before_a_coefficient(coef):
    runs = [np.diff(np.concatenate([[-1], np.flatnonzero(z[1:])])) - 1 for z in coef]
    return max(int(r.max()) for r in runs if len(r))


def test_dc_category_11_zrl_runs_and_ac_category_10():
    _, _, coef = oracle.encode(K.image("blocks_q100_gray"), 100, stages=True)
    dc = coef[:, 0].astype(np.int64)
    assert np.abs(np.diff(np.concatenate([[0], dc]))).max() >= 1024            # DC category 11
    _, _, coef = oracle.encode(K.image("checker_q100_gray"), 100, stages=True)
    assert max(int(np.abs(z[1:]).max()).bit_length() for z in coef) == 10     # the largest AC category
    for name in ("noise_q10_gray", "noise_q1_444", "smooth_q95_444"):
        _, _, coef = oracle.encode(K.image(name), *K.params(name), order="bgr", stages=True)
        assert _longest_run_before_a_coefficient(coef) >= 32, name            # two ZRLs before a coefficient


def test_stages_match_the_layout():
    img = K.noise(17, 9, "420", 2)
    data, planes, coef = oracle.encode(img, 75, "420", order="bgr", stages=True)
    hmax, vmax, mx, my, bpm = oracle.geometry(17, 9, 3, "420")
    assert coef.shape == (mx * my * bpm, 64) and planes.shape == (3, 8 * my * vmax, 8 * mx * hmax)
    b, g, r = (img[..., i].astype(np.int64) for i in range(3))
    y = (19595 * r + 38470 * g + 7471 * b + 32768) >> 16
    assert np.array_equal(planes[0, :17, :9], y)
    assert np.array_equal(planes[0, 17:32, :9], np.repeat(y[-1:], 15, 0))     # the last row repeated
    # the last MCU row of 17 rows 4:2:0 holds one block row of Y (height 3 blocks): its lower Y blocks are dummies
    last = coef[(my - 1) * mx * bpm:][:, 1:]
    assert not last[[2, 3]].any()


def test_max_bytes_bounds_the_worst_case():
    for lay in K.LAYOUTS:
        img = K.noise(64, 64, lay, 1) if lay != "gray" else K.checker(64, 64, lay, 0)
        sub = "420" if lay == "gray" else lay
        n = len(oracle.encode(img, 100, sub))
        d = jpeg.JpegEncodeDesc(64, 64, 1 if lay == "gray" else 3, 0, 100, int(sub), 64 * (1 if lay == "gray" else 3))
        assert n <= jpeg._L.gpsg_jpeg_encode_max_bytes(C.byref(d))


# ---- quantisation ------------------------------------------------------------------------------------------------------
def _reciprocal_quantise(x, d):
    """libjpeg-turbo's quantiser with a 16-bit DCTELEM: a reciprocal, a rounding correction and a shift chosen per
    divisor, applied to |x| (the SIMD build's arithmetic)."""
    b = d.bit_length() - 1
    r = 16 + b
    fq, fr = divmod(1 << r, d)
    c = d // 2
    if fr == 0:
        fq >>= 1
        r -= 1
    elif fr <= d // 2:
        c += 1
    else:
        fq += 1
    a = np.abs(x).astype(np.uint64)
    q = (((a + c) * fq) & 0xFFFFFFFF) >> r
    return np.where(x < 0, -q.astype(np.int64), q.astype(np.int64))


def test_quantiser_is_round_half_up_division():
    x = np.arange(-16383, 16384, dtype=np.int64)
    for qv in range(1, 256):
        d = 8 * qv
        want = np.sign(x) * ((np.abs(x) + d // 2) // d)
        assert np.array_equal(_reciprocal_quantise(x, d), want), d


# ---- the ABI -----------------------------------------------------------------------------------------------------------
def _desc(**kw):
    f = dict(width=40, height=24, channels=3, order=0, quality=90, sampling=420, pitch=120)
    f.update(kw)
    return jpeg.JpegEncodeDesc(**f)


@pytest.mark.parametrize("bad", [dict(width=0), dict(height=0), dict(width=65501), dict(height=65501), dict(pitch=119),
                                 dict(channels=2), dict(channels=4), dict(quality=0), dict(quality=101),
                                 dict(sampling=411), dict(sampling=0), dict(order=2), dict(order=-1)])
def test_abi_refuses_bad_descriptors(bad):
    L = jpeg._L
    d = _desc(**bad)
    assert L.gpsg_jpeg_encode_max_bytes(C.byref(d)) == 0
    descs = (jpeg.JpegEncodeDesc * 1)(d)
    assert L.gpsg_jpeg_encode_workspace_bytes(1, descs) == 0
    p = (C.c_void_p * 1)(256)
    assert L.gpsg_jpeg_encode(0, None, 1, descs, p, p, 256, 256, 1 << 20) == -1


def test_abi_refuses_bad_calls():
    L = jpeg._L
    good = (jpeg.JpegEncodeDesc * 1)(_desc())
    assert L.gpsg_jpeg_encode_max_bytes(None) == 0
    assert L.gpsg_jpeg_encode_workspace_bytes(0, good) == 0
    assert L.gpsg_jpeg_encode_workspace_bytes(65, (jpeg.JpegEncodeDesc * 65)(*[_desc()] * 65)) == 0
    ws = L.gpsg_jpeg_encode_workspace_bytes(1, good)
    assert ws > 0 and L.gpsg_jpeg_encode_max_bytes(good) > 40 * 24 * 3 // 4
    assert L.gpsg_jpeg_encode_workspace_bytes(1, (jpeg.JpegEncodeDesc * 1)(_desc(channels=1, pitch=40))) > 0
    p, z = (C.c_void_p * 1)(256), (C.c_void_p * 1)(None)
    for args in ((0, good, p, p, 256, 256, ws), (65, good, p, p, 256, 256, ws), (1, None, p, p, 256, 256, ws),
                 (1, good, None, p, 256, 256, ws), (1, good, p, None, 256, 256, ws), (1, good, z, p, 256, 256, ws),
                 (1, good, p, z, 256, 256, ws), (1, good, p, p, None, 256, ws), (1, good, p, p, 256, None, ws),
                 (1, good, p, p, 256, 256, ws - 1), (1, good, p, p, 256, 257, ws)):
        assert L.gpsg_jpeg_encode(0, None, *args) == -1, args


def test_encode_refuses_host_tensors_and_bad_arguments():
    import torch
    with pytest.raises(ValueError):
        jpeg.encode(torch.zeros(8, 8, 3, dtype=torch.uint8))
    with pytest.raises(ValueError):
        jpeg.encode([torch.zeros(8, 8, dtype=torch.uint8)], quality=0)
    with pytest.raises(ValueError):
        jpeg.encode([torch.zeros(8, 8, dtype=torch.uint8)], subsampling="411")
    with pytest.raises(ValueError):
        jpeg.encode([torch.zeros(8, 8, dtype=torch.uint8)], order="yuv")


# ---- the switch --------------------------------------------------------------------------------------------------------
@pytest.fixture
def clean_patch():
    patch.uninstall()
    yield
    patch.uninstall()


@pytest.mark.parametrize("value", [None, "0", "1"])
def test_encode_switch_is_read_once_and_uninstall_restores(monkeypatch, clean_patch, value):
    original = cv2.imwrite
    if value is None:
        monkeypatch.delenv("GPSG_ENCODE", raising=False)
    else:
        monkeypatch.setenv("GPSG_ENCODE", value)
    patch.install()
    assert patch.encode() is (value == "1")
    assert ("cv2" in patch._targets()) is (value == "1")
    assert (cv2.imwrite is original) is (value != "1")
    monkeypatch.setenv("GPSG_ENCODE", "0" if value == "1" else "1")      # read at install() only
    assert patch.encode() is (value == "1")
    assert (cv2.imwrite is original) is (value != "1")
    monkeypatch.setenv("GPSG_ENCODE", value or "")
    patch.install()                                                     # idempotent: never wraps the wrapper
    if value != "1":
        assert cv2.imwrite is original
    else:
        assert cv2.imwrite._gpsg_original is original
    patch.uninstall()
    assert cv2.imwrite is original


def test_cv2_imported_after_install_is_hooked(tmp_path):
    """A fresh interpreter: install() first, then `import cv2` (the scripts' order) gets the rebound imwrite."""
    import subprocess
    code = ("import os, sys; sys.path.insert(0, %r); from gps_gaussian_b200 import patch; patch.install(); "
            "assert 'cv2' not in sys.modules; import cv2; w = cv2.imwrite; assert hasattr(w, '_gpsg_original'), w; "
            "n = getattr(cv2, '_native', cv2); assert hasattr(n.imwrite, '_gpsg_original'); "
            "patch.uninstall(); assert cv2.imwrite is w._gpsg_original; "
            "assert n.imwrite is w._gpsg_original, n.imwrite; print('ok')") % os.path.dirname(HERE)
    env = dict(os.environ, GPSG_ENCODE="1")
    env.pop("GPSG_PATCH", None)
    out = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, cwd=str(tmp_path))
    assert out.returncode == 0 and out.stdout.strip().endswith("ok"), out.stderr


@pytest.fixture
def routed(monkeypatch, tmp_path):
    """cv2.imwrite as GPSG_ENCODE=1 rebinds it, over a recording fake encoder and a recording 'cv2' original."""
    native, fallback = [], []

    def fake_encode_host(arr, quality, subsampling, order):
        native.append((np.array(arr), quality, subsampling, order))
        return b"native"

    def fake_orig(*args, **kwargs):
        fallback.append((args, kwargs))
        return "cv2's result"
    monkeypatch.setattr(jpeg, "encode_host", fake_encode_host)
    monkeypatch.setattr(patch, "_on_device", lambda: True)
    monkeypatch.setattr(patch, "_MIN_NATIVE_PIXELS", 64)
    return patch._make_imwrite(fake_orig), native, fallback, tmp_path


IMG = K.noise(12, 10, "420", 3)


def test_routing_native_calls(routed):
    imwrite, native, fallback, tmp = routed
    Q, S = cv2.IMWRITE_JPEG_QUALITY, cv2.IMWRITE_JPEG_SAMPLING_FACTOR
    calls = [((str(tmp / "a.jpg"), IMG), {}, 95, "420"),
             ((str(tmp / "b.JPEG"), IMG[:, :, ::-1]), {}, 95, "420"),                      # negative strides
             ((str(tmp / "c.Jpe"), IMG[:, :, 1]), {}, 95, "420"),
             ((str(tmp / "d.jpg"), IMG[:, :, :1]), {}, 95, "420"),
             ((str(tmp / "e.jpg"), IMG, [Q, 80]), {}, 80, "420"),
             ((str(tmp / "f.jpg"), IMG, [Q, 0, S, cv2.IMWRITE_JPEG_SAMPLING_FACTOR_444]), {}, 1, "444"),
             ((str(tmp / "g.jpg"), IMG, (S, cv2.IMWRITE_JPEG_SAMPLING_FACTOR_422, Q, 100)), {}, 100, "422"),
             ((str(tmp / "h.jpg"), IMG, [Q, 50, Q, 70]), {}, 70, "420"),
             ((str(tmp / "i.jpg"),), dict(img=IMG, params=[Q, np.int64(60)]), 60, "420"),
             ((), dict(filename=str(tmp / "j.jpg"), img=IMG), 95, "420")]
    for args, kwargs, q, s in calls:
        assert imwrite(*args, **kwargs) is True
        arr, got_q, got_s, order = native[-1]
        assert (got_q, got_s, order) == (q, s, "bgr")
        src = kwargs.get("img", args[1] if len(args) > 1 else None)
        assert np.array_equal(arr, src)
        name = kwargs.get("filename", args[0] if args else None)
        assert open(name, "rb").read() == b"native"
    assert len(native) == len(calls) and not fallback


def test_routing_cv2_calls(routed):
    imwrite, native, fallback, tmp = routed
    Q, S = cv2.IMWRITE_JPEG_QUALITY, cv2.IMWRITE_JPEG_SAMPLING_FACTOR
    f = str(tmp / "x.jpg")
    calls = [((str(tmp / "x.png"), IMG), {}),
             ((str(tmp / "x.jpg2"), IMG), {}),
             ((f, IMG.astype(np.uint16)), {}),
             ((f, np.zeros((12, 10, 4), np.uint8)), {}),
             ((f, np.zeros((12, 10, 2), np.uint8)), {}),
             ((f, np.zeros((12, 10, 3, 1), np.uint8)), {}),
             ((f, np.zeros((0, 10, 3), np.uint8)), {}),
             ((f, np.zeros((4, 4, 3), np.uint8)), {}),                                        # below the threshold
             ((f, IMG.tolist()), {}),
             ((f, IMG, [cv2.IMWRITE_JPEG_OPTIMIZE, 1]), {}),
             ((f, IMG, [cv2.IMWRITE_JPEG_PROGRESSIVE, 1]), {}),
             ((f, IMG, [cv2.IMWRITE_JPEG_RST_INTERVAL, 4]), {}),
             ((f, IMG, [cv2.IMWRITE_JPEG_LUMA_QUALITY, 50]), {}),
             ((f, IMG, [Q, 101]), {}),
             ((f, IMG, [Q, -1]), {}),
             ((f, IMG, [Q, 90.0]), {}),
             ((f, IMG, [Q, True]), {}),
             ((f, IMG, [Q]), {}),
             ((f, IMG, [S, cv2.IMWRITE_JPEG_SAMPLING_FACTOR_411]), {}),
             ((f, IMG, [S, cv2.IMWRITE_JPEG_SAMPLING_FACTOR_440]), {}),
             ((f, IMG, np.array([Q, 90])), {}),
             ((str(tmp / "missing" / "x.jpg"), IMG), {}),
             ((tmp / "x.jpg", IMG), {}),
             ((f, IMG, [Q, 90], 1), {}),
             ((f,), dict(img=IMG, quality=90))]
    for args, kwargs in calls:
        assert imwrite(*args, **kwargs) == "cv2's result"
        assert fallback[-1][1] == kwargs and len(fallback[-1][0]) == len(args)
        assert all(a is b for a, b in zip(fallback[-1][0], args))
    assert not native and len(fallback) == len(calls)


def test_routing_without_cuda_or_in_a_worker(routed, monkeypatch):
    imwrite, native, fallback, tmp = routed
    monkeypatch.setattr(patch, "_on_device", lambda: False)
    assert imwrite(str(tmp / "a.jpg"), IMG) == "cv2's result"
    assert not native and len(fallback) == 1


def test_missing_directory_returns_what_cv2_returns(tmp_path):
    assert cv2.imwrite(str(tmp_path / "missing" / "x.jpg"), IMG) is False


def test_images_too_large_for_one_call_go_to_cv2(routed):
    imwrite, native, fallback, tmp = routed
    huge = np.broadcast_to(np.zeros((1, 1, 3), np.uint8), (21000, 21000, 3))      # above 2^30 bit words at 4:4:4
    S = cv2.IMWRITE_JPEG_SAMPLING_FACTOR
    assert not jpeg.fits_one_call(21000, 21000, 3, "444") and jpeg.fits_one_call(2048, 2048, 3, "444")
    assert imwrite(str(tmp / "huge.jpg"), huge, [S, cv2.IMWRITE_JPEG_SAMPLING_FACTOR_444]) == "cv2's result"
    assert not native and len(fallback) == 1


def test_device_out_of_memory_goes_to_cv2(routed, monkeypatch):
    import torch
    imwrite, native, fallback, tmp = routed

    def oom(*args, **kwargs):
        raise torch.cuda.OutOfMemoryError("CUDA out of memory")
    monkeypatch.setattr(jpeg, "encode_host", oom)
    assert imwrite(str(tmp / "a.jpg"), IMG) == "cv2's result"
    assert len(fallback) == 1 and fallback[0][0][1] is IMG


def test_child_processes_go_to_cv2(routed, monkeypatch):
    """A multiprocessing child (a Pool of writers, forked after the parent used CUDA) never takes the GPU route."""
    import multiprocessing
    imwrite, native, fallback, tmp = routed
    monkeypatch.setattr(multiprocessing, "parent_process", lambda: object())
    assert imwrite(str(tmp / "a.jpg"), IMG) == "cv2's result"
    assert not native and len(fallback) == 1


def test_staging_is_locked_across_threads(monkeypatch):
    """encode_host holds its lock from filling the pinned buffer until encode() returns: a second thread waits."""
    import threading
    import torch
    inside, order = threading.Event(), []

    class FakeTensor:
        def __init__(self, n):
            self.a = np.zeros(n, np.uint8)

        def numel(self):
            return self.a.size

        def __getitem__(self, k):
            t = FakeTensor(0)
            t.a = self.a[k]
            return t

        def numpy(self):
            return self.a

        def copy_(self, other, non_blocking=False):
            self.a[:] = other.a

        def view(self, shape):
            return self.a.reshape(shape).copy()

    def fake_encode(d, quality, subsampling, order_):
        order.append(("start", int(d.flat[0])))
        inside.set()
        threading.Event().wait(0.2)
        order.append(("end", int(d.flat[0])))
        return bytes([int(d.flat[0])])
    dev = torch.device("cuda", 0)
    monkeypatch.setattr(jpeg, "_STAGING", {dev: (FakeTensor(1 << 20), FakeTensor(1 << 20))})
    monkeypatch.setattr(jpeg, "encode", fake_encode)
    monkeypatch.setattr(torch.cuda, "device", lambda d: __import__("contextlib").nullcontext())
    got = {}
    t1 = threading.Thread(target=lambda: got.setdefault(1, jpeg.encode_host(np.full((8, 8, 3), 1, np.uint8), device=dev)))
    t1.start()
    inside.wait(5)
    t2 = threading.Thread(target=lambda: got.setdefault(2, jpeg.encode_host(np.full((8, 8, 3), 2, np.uint8), device=dev)))
    t2.start()
    t1.join()
    t2.join()
    assert got == {1: b"\x01", 2: b"\x02"}
    assert order == [("start", 1), ("end", 1), ("start", 2), ("end", 2)]
