"""JPEG corpus of the decoder tests: encoded with Pillow and cv2, plus the SHA-256 of Pillow's decode of each file.

    python tests/golden/make_jpeg_corpus.py      # writes tests/golden/jpeg/*.jpg and tests/golden/jpeg/sha256.json

The small files are committed.  The 1023x1025, 1024^2 and 2048^2 images are not (they would weigh megabytes): `corpus(
large=True)` makes them from the same seeded content at test time.  Everything here is seeded.
"""
import hashlib
import io
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "jpeg")


def _smooth(h, w, seed):
    """A photo-like frame: gradients, a disc, texture and mild noise."""
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[:h, :w].astype(np.float32)
    r = np.hypot(y - h * 0.45, x - w * 0.55) < min(h, w) * 0.3
    img = np.stack([x / max(w, 1) * 200 + 30, y / max(h, 1) * 180 + 40, (np.sin(x / 7) * np.cos(y / 11) + 1) * 90], -1)
    img[r] = img[r] * 0.4 + np.array([200, 60, 90]) * 0.6
    img += rng.normal(0, 6, img.shape)
    return np.clip(img, 0, 255).astype(np.uint8)


def _pil(img, **kw):
    from PIL import Image
    b = io.BytesIO()
    Image.fromarray(img).save(b, format="JPEG", **kw)
    return b.getvalue()


def _cv2(img, q=95, rst=0):
    import cv2
    ok, buf = cv2.imencode(".jpg", img[:, :, ::-1] if img.ndim == 3 else img,
                           [cv2.IMWRITE_JPEG_QUALITY, q] + ([cv2.IMWRITE_JPEG_RST_INTERVAL, rst] if rst else []))
    assert ok
    return buf.tobytes()


def _mesh_frame():
    """A frame of the project's mesh renderer (its serial oracle, which the kernel matches bit for bit), converted and
    encoded as prepare_data/render_data.py does: clip, *255 + 0.5, BGR, cv2.imwrite's defaults."""
    sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
    from gps_gaussian_b200 import synth_mesh
    from oracle import mesh_oracle
    v, fc, uv = synth_mesh.uv_sphere((0.0, 0.0, 3.0), 1.0, 24, 48)
    tex = np.random.default_rng(3).uniform(0, 1, (32, 16, 3)).astype(np.float32)
    img, _, _ = mesh_oracle.render((96, 80), (70.0, 70.0, 48.0, 40.0), (0.0, 0.0, 0.0), np.diag([-1.0, -1.0, 1.0]),
                                   np.array([[0.3, -0.5, -0.8]], np.float32), np.ones((1, 3), np.float32), v, fc, uv, fc,
                                   tex)
    img = np.ascontiguousarray(img.swapaxes(0, 1))
    img = (np.clip(img, 0, 1) * 255.0 + 0.5).astype(np.uint8)[:, :, ::-1]
    import cv2
    ok, buf = cv2.imencode(".jpg", img)
    assert ok
    return buf.tobytes()


def corpus(large=False):
    """{name: JPEG bytes}.  large=True: only the large sizes."""
    if large:
        return {"q95_420_1023x1025.jpg": _pil(_smooth(1025, 1023, 20), quality=95),
                "q95_420_1024.jpg": _pil(_smooth(1024, 1024, 21), quality=95),
                "cv2_q95_1024.jpg": _cv2(_smooth(1024, 1024, 22)),
                "q95_420_2048.jpg": _pil(_smooth(2048, 2048, 23), quality=95),
                "q95_444_rst_1024.jpg": _pil(_smooth(1024, 1024, 24), quality=95, subsampling=0,
                                             restart_marker_blocks=7)}
    c = {}
    base = _smooth(72, 88, 1)
    for q in (50, 75, 95, 100):
        for sub, tag in ((0, "444"), (1, "422"), (2, "420")):
            c[f"q{q}_{tag}.jpg"] = _pil(base, quality=q, subsampling=sub)
        c[f"q{q}_gray.jpg"] = _pil(base[:, :, 1], quality=q)
    for sub, tag in ((0, "444"), (1, "422"), (2, "420")):
        c[f"opt_{tag}.jpg"] = _pil(base, quality=90, subsampling=sub, optimize=True)
        c[f"rst_pil_{tag}.jpg"] = _pil(base, quality=90, subsampling=sub, restart_marker_blocks=5)
    c["rst_pil_gray.jpg"] = _pil(base[:, :, 0], quality=90, restart_marker_blocks=3)
    c["rst_cv2_1.jpg"] = _cv2(base, rst=1)
    c["rst_cv2_3.jpg"] = _cv2(base, q=80, rst=3)
    for h, w in ((1, 1), (9, 7), (1, 17), (17, 1)):
        img = _smooth(h, w, h * 100 + w)
        for sub, tag in ((0, "444"), (1, "422"), (2, "420")):
            c[f"size_{w}x{h}_{tag}.jpg"] = _pil(img, quality=90, subsampling=sub)
        c[f"size_{w}x{h}_gray.jpg"] = _pil(img[:, :, 2], quality=90)
    noise = np.random.default_rng(5).integers(0, 256, (40, 56, 3), dtype=np.uint8)
    c["noise_q100_444.jpg"] = _pil(noise, quality=100, subsampling=0)
    c["noise_q100_420.jpg"] = _pil(noise, quality=100, subsampling=2)
    c["noise_q100_gray.jpg"] = _pil(noise[:, :, 0], quality=100)
    c["flat_420.jpg"] = _pil(np.full((48, 64, 3), 90, np.uint8), quality=95)
    c["flat_gray.jpg"] = _pil(np.full((33, 31), 200, np.uint8), quality=75)
    c["mesh_frame.jpg"] = _mesh_frame()
    return c


def pillow_sha256(data):
    from PIL import Image
    a = np.array(Image.open(io.BytesIO(data)))
    return hashlib.sha256(a.tobytes() + repr(a.shape).encode()).hexdigest()


if __name__ == "__main__":
    os.makedirs(OUT, exist_ok=True)
    c = corpus()
    for name, data in c.items():
        with open(os.path.join(OUT, name), "wb") as f:
            f.write(data)
    with open(os.path.join(OUT, "sha256.json"), "w") as f:
        json.dump({k: pillow_sha256(v) for k, v in sorted(c.items())}, f, indent=1, sort_keys=True)
    print(len(c), "files,", sum(map(len, c.values())), "bytes")
