"""GPU: gpsg_jpeg_decode byte for byte against Pillow (the corpus, its large sizes, mixed batches), with poisoned
outputs and guard bytes; streams malformed in a bounded way set the status word and the public call still returns
Pillow's result; the unmodified inference scripts write identical files with and without GPSG_DECODE=1."""
import ctypes as C
import filecmp
import glob
import importlib.util
import io
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from gps_gaussian_b200 import _lib, harness, jpeg  # noqa: E402

Image = pytest.importorskip("PIL.Image")
HERE = os.path.dirname(os.path.abspath(__file__))
CORPUS = os.path.join(HERE, "golden", "jpeg")
GUARD, POISON = 64, 0xA5


def _corpus():
    with open(os.path.join(CORPUS, "sha256.json")) as f:
        names = sorted(json.load(f))
    return {k: open(os.path.join(CORPUS, k), "rb").read() for k in names}


def _maker():
    spec = importlib.util.spec_from_file_location("make_jpeg_corpus", os.path.join(HERE, "golden", "make_jpeg_corpus.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _pillow(data):
    return np.array(Image.open(io.BytesIO(data)))


def _raw(datas):
    """The ABI on a batch: every output poisoned and framed by guard bytes.  Returns (images, status, guards intact)."""
    infos = []
    for d in datas:
        code, info = jpeg.parse(d)
        assert code == 0
        infos.append(info)
    n = len(datas)
    arr = (jpeg.JpegInfo * n)(*infos)
    blob = torch.from_numpy(np.frombuffer(b"".join(datas), np.uint8).copy()).cuda()
    offs = np.cumsum([0] + [len(d) for d in datas])
    bufs, outs = [], []
    for info in infos:
        size = info.width * info.height * info.num_components
        b = torch.full((size + 2 * GUARD,), POISON, dtype=torch.uint8, device="cuda")
        bufs.append(b)
        outs.append(b[GUARD:GUARD + size])
    status = torch.full((n,), -1, dtype=torch.int32, device="cuda")
    wsb = jpeg._L.gpsg_jpeg_decode_workspace_bytes(n, arr)
    ws = torch.full((wsb + 256,), 0x5A, dtype=torch.uint8, device="cuda")
    base = (ws.data_ptr() + 255) // 256 * 256
    idx, stream = _lib.device_stream(torch.device("cuda"))
    rc = jpeg._L.gpsg_jpeg_decode(idx, stream, n, arr, (C.c_void_p * n)(*[blob.data_ptr() + int(o) for o in offs[:-1]]),
                                  (C.c_void_p * n)(*[o.data_ptr() for o in outs]), status.data_ptr(), base, wsb)
    _lib.check(rc, "gpsg_jpeg_decode")
    torch.cuda.synchronize()
    guards = all(bool((b[:GUARD] == POISON).all()) and bool((b[-GUARD:] == POISON).all()) for b in bufs)
    imgs = []
    for info, o in zip(infos, outs):
        shape = (info.height, info.width) if info.num_components == 1 else (info.height, info.width, 3)
        imgs.append(o.view(shape).cpu().numpy())
    return imgs, status.cpu().numpy(), guards


def _check_equal(datas, names):
    imgs, st, guards = _raw(datas)
    assert guards
    for name, d, img, s in zip(names, datas, imgs, st):
        assert s == 0, (name, hex(int(s)))
        assert np.array_equal(img, _pillow(d)), name
    return imgs


def test_corpus_one_image_per_call():
    for name, d in _corpus().items():
        _check_equal([d], [name])


def test_corpus_as_one_mixed_batch_and_reruns_identical():
    c = _corpus()
    names = list(c)
    first = _check_equal([c[k] for k in names], names)
    again = _check_equal([c[k] for k in names], names)
    assert all(np.array_equal(a, b) for a, b in zip(first, again))


def test_large_sizes():
    big = _maker().corpus(large=True)
    for name, d in big.items():
        _check_equal([d], [name])
    names = list(big)
    _check_equal([big[k] for k in names], names)                      # the pair-sized batch, mixed sizes / layouts


def test_random_batches_of_mixed_formats():
    rng = np.random.default_rng(7)
    mk = _maker()
    for _ in range(6):
        datas, names = [], []
        for _ in range(int(rng.integers(2, 7))):
            h, w = (int(v) for v in rng.integers(1, 300, 2))
            img = mk._smooth(h, w, int(rng.integers(1 << 30)))
            kw = dict(quality=int(rng.choice([50, 75, 95, 100])), subsampling=int(rng.integers(3)))
            if rng.random() < 0.3:
                kw["restart_marker_blocks"] = int(rng.integers(1, 9))
            if rng.random() < 0.3:
                kw["optimize"] = True
            datas.append(mk._pil(img[:, :, 0] if rng.random() < 0.25 else img, **kw))
            names.append((h, w, kw))
        _check_equal(datas, names)


def _ecs(data):
    _, info = jpeg.parse(data)
    return info.ecs_offset, info.ecs_offset + info.ecs_length


def _malformed():
    mk = _maker()
    img = mk._smooth(64, 96, 11)
    plain = mk._pil(img, quality=90, subsampling=2)
    rst = mk._pil(img, quality=90, subsampling=2, restart_marker_blocks=2)
    a, b = _ecs(plain)
    truncated = plain[:a + (b - a) // 2] + plain[b:]                       # the scan cut short, EOI kept
    mid = a + (b - a) // 3
    bad_code = plain[:mid] + b"\xff\x00" * 4 + plain[mid + 8:]             # 32 one bits: no Huffman code is that long
    ra, rb = _ecs(rst)
    i = rst.index(b"\xff\xd0", ra)
    j = rst.index(b"\xff\xd1", ra)
    wrong_rst = bytearray(rst)
    wrong_rst[i + 1], wrong_rst[j + 1] = 0xD1, 0xD0
    extra = plain[:b] + bytes(range(1, 40)) + plain[b:]                    # entropy data past the last MCU
    return {"truncated": bytes(truncated), "bad_code": bytes(bad_code), "wrong_rst": bytes(wrong_rst),
            "extra_data": bytes(extra)}, plain


@pytest.mark.parametrize("case", ["truncated", "bad_code", "wrong_rst", "extra_data"])
def test_malformed_stream_sets_status_and_public_call_is_pillow(case):
    cases, _ = _malformed()
    d = cases[case]
    assert jpeg.supported(d)
    imgs, st, guards = _raw([d])
    assert guards and st[0] != 0, case
    jpeg.reset_counts()
    try:
        want = _pillow(d)
    except Exception as e:                                                 # Pillow's exception, or its image
        with pytest.raises(type(e)):
            jpeg.decode(d)
    else:
        assert np.array_equal(jpeg.decode(d).cpu().numpy(), want)
    assert jpeg.counts()["native"] == 0
    with pytest.raises(jpeg.JpegError):
        jpeg.decode(d, fallback=False)


def test_data_after_eoi_is_ignored_as_pillow_does():
    _, plain = _malformed()
    d = plain + b"trailing bytes after EOI \xff\xd9\x00"
    imgs, st, guards = _raw([d])
    assert guards and st[0] == 0 and np.array_equal(imgs[0], _pillow(d))


def _cpu_tests():
    spec = importlib.util.spec_from_file_location("_jpeg_cpu_cases", os.path.join(HERE, "test_jpeg_cpu.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


@pytest.mark.parametrize("case", ["dc-all-ones-code", "dc-symbol-above-15"])
def test_bad_tables_raise_what_pillow_raises_on_cuda(case):
    data, _ = _cpu_tests()._refusals()[case]
    with pytest.raises(OSError) as want:
        _pillow(data)
    jpeg.reset_counts()
    with pytest.raises(type(want.value)):
        jpeg.decode(data)
    assert jpeg.counts()["native"] == 0


def test_out_of_range_coefficients_set_status_and_public_call_is_pillow():
    t = _cpu_tests()
    data = bytearray(t._pil(t.BASE, quality=90, subsampling=0))
    data[t._marker(bytes(data), 0xDB) + 5] = 255               # the DC quantiser, raised after encoding
    data = bytes(data)
    imgs, st, guards = _raw([data])
    assert guards and st[0] & 32, hex(int(st[0]))
    jpeg.reset_counts()
    assert np.array_equal(jpeg.decode(data).cpu().numpy(), _pillow(data))
    assert jpeg.counts() == {"native": 0, "fallback": 1}


def test_batches_split_at_the_scan_size_limit(monkeypatch):
    c = _corpus()
    names = list(c)
    biggest = max(jpeg.parse(c[k])[1].ecs_length for k in names)
    monkeypatch.setattr(jpeg, "MAX_SCAN_BYTES", biggest + 1)      # at most a few images per call
    jpeg.reset_counts()
    got = jpeg.decode([c[k] for k in names])
    assert jpeg.counts() == {"native": len(names), "fallback": 0}
    for k, g in zip(names, got):
        assert np.array_equal(g.cpu().numpy(), _pillow(c[k])), k


def test_public_decode_counts_routes():
    c = _corpus()
    prog = io.BytesIO()
    Image.fromarray(_pillow(c["q95_420.jpg"])).save(prog, format="JPEG", progressive=True)
    jpeg.reset_counts()
    got = jpeg.decode([c["q95_420.jpg"], prog.getvalue(), c["q75_gray.jpg"]])
    assert jpeg.counts() == {"native": 2, "fallback": 1}
    for g, d in zip(got, [c["q95_420.jpg"], prog.getvalue(), c["q75_gray.jpg"]]):
        assert g.is_cuda and g.dtype == torch.uint8 and np.array_equal(g.cpu().numpy(), _pillow(d))


# ---- the unmodified inference scripts --------------------------------------------------------------------------------
needs_ref = pytest.mark.skipif(harness.staged_reference() is None, reason="oracle/_ref not staged")
RES = 128
_COUNT = ("\nm = sys.modules.get('gps_gaussian_b200.jpeg')\n"
          "print('JPEG_COUNTS', m.counts() if m else None)\n")


@pytest.fixture(scope="module")
def dataset(tmp_path_factory):
    from gps_gaussian_b200 import synth_dataset
    root = str(tmp_path_factory.mktemp("jpegdata"))
    synth_dataset.write_dataset(root, n_train=2, n_val=2, res=RES, hr=True)
    return root


@needs_ref
@pytest.mark.parametrize("script", ["test_real_data.py", "test_view_interp.py"])
def test_scripts_identical_with_and_without_decode(dataset, tmp_path, script):
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
        env.pop("GPSG_DECODE", None)
        if on:
            env["GPSG_DECODE"] = "1"
        p = subprocess.run([sys.executable, "-c", harness.SCRIPT_RUNNER + _COUNT, script] + args, cwd=work, env=env,
                           text=True, capture_output=True, timeout=900)
        assert p.returncode == 0, p.stdout[-3000:] + p.stderr[-6000:]
        line = [ln for ln in p.stdout.splitlines() if ln.startswith("JPEG_COUNTS")][-1]
        if on:
            counts = eval(line.split(" ", 1)[1])
            assert counts["native"] >= 2 and counts["fallback"] == 0, line
        else:
            assert line == "JPEG_COUNTS None", line
        out_dir = "test_out" if script == "test_real_data.py" else "interp_out"
        outs[on] = sorted(glob.glob(os.path.join(work, out_dir, "*.jpg")))
        assert len(outs[on]) >= 2, outs[on]
    assert [os.path.basename(a) for a in outs[False]] == [os.path.basename(b) for b in outs[True]]
    for a, b in zip(outs[False], outs[True]):
        assert filecmp.cmp(a, b, shallow=False), (a, b)
