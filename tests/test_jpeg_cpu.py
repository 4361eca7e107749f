"""CPU: the JPEG marker parser and its refusals, the serial oracle against Pillow byte for byte, the GPSG_DECODE switch
and the Pillow fallback of gps_gaussian_b200.jpeg."""
import ctypes as C
import importlib.util
import io
import json
import os
import sys
import types

import numpy as np
import pytest
import torch

from gps_gaussian_b200 import jpeg, patch
from oracle import jpeg_oracle

Image = pytest.importorskip("PIL.Image")
HERE = os.path.dirname(os.path.abspath(__file__))
CORPUS = os.path.join(HERE, "golden", "jpeg")


def _corpus():
    with open(os.path.join(CORPUS, "sha256.json")) as f:
        sha = json.load(f)
    return {k: open(os.path.join(CORPUS, k), "rb").read() for k in sha}, sha


def _maker():
    spec = importlib.util.spec_from_file_location("make_jpeg_corpus", os.path.join(HERE, "golden", "make_jpeg_corpus.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _pillow(data):
    return np.array(Image.open(io.BytesIO(data)))


def _pil(img, **kw):
    b = io.BytesIO()
    Image.fromarray(img).save(b, format="JPEG", **kw)
    return b.getvalue()


def _marker(data, m):
    """Offset of the first marker 0xFF m in the header (walks the segments)."""
    i = 2
    while i + 4 <= len(data):
        if data[i + 1] == m:
            return i
        i += 2 + ((data[i + 2] << 8) | data[i + 3])
    raise KeyError(hex(m))


BASE = np.random.default_rng(0).integers(0, 256, (24, 40, 3), dtype=np.uint8)


# ---- the corpus ---------------------------------------------------------------------------------------------------
def test_corpus_is_what_pillow_decodes():
    files, sha = _corpus()
    mk = _maker()
    assert len(files) >= 40
    for name, data in files.items():
        assert mk.pillow_sha256(data) == sha[name], name


def test_oracle_equals_pillow_on_corpus():
    files, _ = _corpus()
    for name, data in files.items():
        st, img = jpeg_oracle.decode(data)
        assert st == 0, (name, st)
        assert np.array_equal(img, _pillow(data)), name


@pytest.mark.parametrize("seed", range(4))
def test_oracle_equals_pillow_random_sweep(seed):
    rng = np.random.default_rng(100 + seed)
    mk = _maker()
    for _ in range(12):
        h, w = (int(v) for v in rng.integers(1, 70, 2))
        img = mk._smooth(h, w, int(rng.integers(1 << 30)))
        kw = dict(quality=int(rng.choice([50, 75, 90, 95, 100])), subsampling=int(rng.integers(3)))
        if rng.random() < 0.3:
            kw["optimize"] = True
        if rng.random() < 0.3:
            kw["restart_marker_blocks"] = int(rng.integers(1, 9))
        data = _pil(img[:, :, 0] if rng.random() < 0.2 else img, **kw)
        st, got = jpeg_oracle.decode(data)
        assert st == 0 and np.array_equal(got, _pillow(data)), (h, w, kw)


def test_oracle_stages_are_consistent():
    """The coefficient and plane stages: a flat image has only DC coefficients and flat planes."""
    data = _pil(np.full((16, 16, 3), 128, np.uint8), quality=95, subsampling=2)
    st, img, coef, planes = jpeg_oracle.decode(data, stages=True)
    assert st == 0 and coef.shape == (6, 64) and planes.shape == (3, 16, 16)
    assert not coef[:, 1:].any()
    assert np.array_equal(img, _pillow(data))


# ---- the parser ---------------------------------------------------------------------------------------------------
def test_parser_fills_the_info():
    files, _ = _corpus()
    for name, data in files.items():
        code, info = jpeg.parse(data)
        rc, (W, H, nc, ri) = jpeg_oracle.parse(data)
        assert code == 0 == rc, name
        assert (info.width, info.height, info.num_components, info.restart_interval) == (W, H, nc, ri), name
        assert data[info.ecs_offset + info.ecs_length:][:1] == b"\xff", name
        assert jpeg.supported(data)
    _, info = jpeg.parse(files["q95_420.jpg"])
    assert tuple(info.h_samp) == (2, 1, 1) and tuple(info.v_samp) == (2, 1, 1)
    _, info = jpeg.parse(files["q95_422.jpg"])
    assert tuple(info.h_samp) == (2, 1, 1) and tuple(info.v_samp) == (1, 1, 1)


def _with_sof(data, fn):
    d = bytearray(data)
    fn(d, _marker(data, 0xC0))
    return bytes(d)


def _with_dc_table(data, extra_len, extra_sym):
    """`data` with one more code of length `extra_len` and symbol `extra_sym` in its DC table 0."""
    i = 2
    while True:
        ln = (data[i + 2] << 8) | data[i + 3]
        if data[i + 1] == 0xC4 and data[i + 4] == 0x00:
            break
        i += 2 + ln
    bits = bytearray(data[i + 5:i + 21])
    n = sum(bits)
    vals = data[i + 21:i + 21 + n]
    rest = data[i + 21 + n:i + 2 + ln]             # further tables of the same DHT segment
    bits[extra_len - 1] += 1
    order = [sum(bits[:l]) for l in range(16)]     # new symbol goes last among the codes of its length
    pos = order[extra_len - 1] + bits[extra_len - 1] - 1
    vals = vals[:pos] + bytes([extra_sym]) + vals[pos:]
    seg = b"\x00" + bytes(bits) + vals + rest
    return data[:i] + b"\xff\xc4" + (len(seg) + 2).to_bytes(2, "big") + seg + data[i + 2 + ln:]


def _refusals():
    base = _pil(BASE, quality=90, subsampling=2)
    gray = _pil(BASE[:, :, 0], quality=90)
    cmyk = io.BytesIO()
    Image.fromarray(np.zeros((8, 8, 4), np.uint8), "CMYK").save(cmyk, format="JPEG")
    adobe_rgb = base[:2] + b"\xff\xee\x00\x0eAdobe\x00\x64\x00\x00\x00\x00\x00" + base[2:]
    adobe_rgb = adobe_rgb.replace(b"JFIF\x00", b"JFIX\x00", 1)
    sos = _marker(base, 0xDA)
    two_scans = base[:-2] + base[sos:]
    return {
        "progressive": (_pil(BASE, quality=90, progressive=True), 3),
        "lossless": (_with_sof(base, lambda d, i: d.__setitem__(i + 1, 0xC3)), 5),
        "arithmetic": (_with_sof(base, lambda d, i: d.__setitem__(i + 1, 0xC9)), 4),
        "hierarchical": (_with_sof(base, lambda d, i: d.__setitem__(i + 1, 0xC5)), 6),
        "12-bit": (_with_sof(base, lambda d, i: d.__setitem__(i + 4, 12)), 7),
        "cmyk": (cmyk.getvalue(), 8),
        "adobe-rgb": (adobe_rgb, 8),
        "sampling-4:4:0": (_with_sof(_pil(BASE, quality=90, subsampling=0), lambda d, i: d.__setitem__(i + 11, 0x12)), 9),
        "chroma-2x2": (_with_sof(base, lambda d, i: d.__setitem__(i + 14, 0x22)), 9),
        "two-scans": (two_scans, 10),
        "dnl-height-0": (_with_sof(base, lambda d, i: (d.__setitem__(i + 5, 0), d.__setitem__(i + 6, 0))), 11),
        "truncated": (base[: len(base) // 2], 1),
        "no-eoi": (base[:-2], 1),
        "length-past-end": (base[:sos + 2] + b"\xff\xff", 1),
        "not-jpeg": (b"\x89PNG\r\n\x1a\n" + bytes(32), 2),
        "zero-length": (base[:2] + b"\xff\xe0\x00\x01" + base[2:], 2),
        "sos-before-sof": (base[:2] + base[sos:], 2),
        # Huffman tables libjpeg-turbo refuses when it builds them (Pillow: "broken data stream")
        "dc-all-ones-code": (_with_dc_table(gray, 9, 0), 2),
        "dc-symbol-above-15": (_with_dc_table(gray, 16, 200), 2),
    }


@pytest.mark.parametrize("case", list(_refusals()))
def test_parser_refusals(case):
    data, code = _refusals()[case]
    got, _ = jpeg.parse(data)
    assert got == code, (case, got)
    assert jpeg_oracle.parse(data)[0] == code
    assert not jpeg.supported(data)


@pytest.mark.parametrize("case", ["dc-all-ones-code", "dc-symbol-above-15"])
def test_bad_tables_raise_what_pillow_raises(case):
    """The public call on a refused table: Pillow's exception, not an image."""
    data, _ = _refusals()[case]
    with pytest.raises(OSError) as want:
        _pillow(data)
    with pytest.raises(type(want.value)):
        jpeg.decode(data, device="cpu")


def test_a_full_but_valid_table_is_still_accepted():
    """The code-space check is libjpeg's `code >= 1 << length`: one code short of full is a valid table."""
    data = _with_dc_table(_pil(BASE[:, :, 0], quality=90), 16, 3)
    assert jpeg.parse(data)[0] == 0 == jpeg_oracle.parse(data)[0]
    st, img = jpeg_oracle.decode(data)
    assert st == 0 and np.array_equal(img, _pillow(data))


def test_out_of_range_coefficients_are_flagged():
    """A DC quantiser raised after encoding: dequantised coefficients beyond +-1024 set GPSG_JPEG_ST_COEF in the oracle
    (the kernel flags the same blocks), so the image goes to Pillow."""
    data = bytearray(_pil(BASE, quality=90, subsampling=0))
    i = _marker(bytes(data), 0xDB)
    data[i + 5] = 255                                      # table 0, entry 0 (DC), 8-bit precision
    st, img = jpeg_oracle.decode(bytes(data))
    assert st == 32 and img is None


def test_parser_never_reads_past_the_buffer():
    """Each parser is given the whole file but told its size is a prefix: a parser that read past `size` would find the
    rest of a valid file there and accept it.  Every proper prefix must be refused, with the code the prefix alone gets."""
    data = _pil(BASE, quality=90, subsampling=1, restart_marker_blocks=2)
    whole = C.create_string_buffer(data, len(data))
    info, dims = jpeg.JpegInfo(), (C.c_int * 4)()
    for n in range(0, len(data)):
        alone = jpeg.parse(data[:n])[0]
        assert alone != 0, n
        assert jpeg._L.gpsg_jpeg_parse(whole, n, C.byref(info)) == alone, n
        assert jpeg_oracle._lib().oracle_jpeg_parse(whole, n, dims) == alone == jpeg_oracle.parse(data[:n])[0], n
    assert jpeg._L.gpsg_jpeg_parse(whole, len(data), C.byref(info)) == 0


def test_abi_refusals():
    L = jpeg._L
    info = (jpeg.JpegInfo * 1)()
    assert L.gpsg_jpeg_decode_workspace_bytes(0, info) == 0
    assert L.gpsg_jpeg_decode_workspace_bytes(1, info) == 0                # an info the parser does not produce
    assert L.gpsg_jpeg_parse(None, 0, C.byref(info[0])) == -1
    _, good = jpeg.parse(_pil(BASE, quality=90))
    infos = (jpeg.JpegInfo * 1)(good)
    ws = L.gpsg_jpeg_decode_workspace_bytes(1, infos)
    assert ws > 0
    p = (C.c_void_p * 1)(256)
    for args in ((0, infos, p, p, 256, 256, ws), (65, infos, p, p, 256, 256, ws), (1, infos, None, p, 256, 256, ws),
                 (1, infos, p, p, None, 256, ws), (1, infos, p, p, 256, 256, ws - 1), (1, infos, p, p, 256, 257, ws),
                 (1, info, p, p, 256, 256, ws)):
        assert L.gpsg_jpeg_decode(0, None, *args) == -1, args


# ---- the public call's fallback -----------------------------------------------------------------------------------
def test_fallback_is_pillow_and_counted():
    data = _pil(BASE, quality=90, progressive=True)
    jpeg.reset_counts()
    got = jpeg.decode([data, data], device="cpu")
    assert all(torch.equal(g, torch.from_numpy(_pillow(data))) for g in got)
    assert jpeg.counts() == {"native": 0, "fallback": 2}
    with pytest.raises(jpeg.JpegError):
        jpeg.decode(data, device="cpu", fallback=False)
    with pytest.raises(Exception):                         # Pillow's own exception reaches the caller
        jpeg.decode(b"\xff\xd8\xff\xdb", device="cpu")


def test_native_route_needs_a_cuda_device():
    data = _pil(BASE, quality=90)
    with pytest.raises(ValueError):
        jpeg.decode(data, device="cpu")
    with pytest.raises(ValueError):
        jpeg.decode([_pil(BASE, quality=90, progressive=True), data], device="cpu")


def test_limits_route_to_pillow(monkeypatch):
    """Above Pillow's decompression-bomb limit Pillow warns or raises, so such an image is Pillow's; so is a scan of
    GPSG_JPEG_MAX_SCAN_BYTES or more, which no single call takes."""
    data = _pil(BASE, quality=90)                          # 40 x 24 = 960 pixels
    assert jpeg.supported(data)
    monkeypatch.setattr(Image, "MAX_IMAGE_PIXELS", 400)
    assert not jpeg.supported(data)
    with pytest.raises(Image.DecompressionBombError):      # more than twice the limit: Pillow raises
        jpeg.decode(data, device="cpu")
    monkeypatch.setattr(Image, "MAX_IMAGE_PIXELS", None)
    assert jpeg.supported(data)
    monkeypatch.setattr(jpeg, "MAX_SCAN_BYTES", jpeg.parse(data)[1].ecs_length)
    assert not jpeg.supported(data)
    jpeg.reset_counts()
    assert torch.equal(jpeg.decode(data, device="cpu"), torch.from_numpy(_pillow(data)))
    assert jpeg.counts() == {"native": 0, "fallback": 1}


# ---- the switch ---------------------------------------------------------------------------------------------------
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


@pytest.mark.parametrize("rectify,decode", [(None, "1"), ("1", None), ("1", "0"), ("1", "1")])
def test_decode_switch_and_uninstall(monkeypatch, clean_patch, rectify, decode):
    mod = _fake_loader()
    cls = mod.StereoHumanDataset
    before = dict(cls.__dict__)
    monkeypatch.setitem(sys.modules, "lib.human_loader", mod)
    for k, v in (("GPSG_RECTIFY", rectify), ("GPSG_DECODE", decode)):
        if v is None:
            monkeypatch.delenv(k, raising=False)
        else:
            monkeypatch.setenv(k, v)
    patch.install()
    assert patch.decode() is (decode == "1")
    assert (cls.__dict__["get_test_item"] is before["get_test_item"]) is (rectify != "1")
    monkeypatch.setattr(torch.cuda, "is_available", lambda: False)      # without CUDA: the original path
    assert cls().get_test_item(0, [0, 1]) == "original test item"
    patch.uninstall()
    assert cls.__dict__["get_test_item"] is before["get_test_item"]

