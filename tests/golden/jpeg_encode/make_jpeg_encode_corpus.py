"""Fixtures of the JPEG encoder tests: cv2.imencode('.jpg') of seeded numpy images, and their SHA-256.

    python tests/golden/jpeg_encode/make_jpeg_encode_corpus.py   # writes tests/golden/jpeg_encode/*.jpg + sha256.json

Only the encoded files are committed, and of the 1023x1025 ones only the hash (`committed(name)` is False for them);
`image(name)` rebuilds each input from its seed.  The arrays are cv2's (BGR for
three channels).  sha256.json records the cv2 and libjpeg-turbo versions the files came from: where the installed cv2
is the same, the tests also compare against it live.
"""
import hashlib
import json
import os
import re

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
LAYOUTS = ("gray", "444", "422", "420")
SAMPLING = {"444": 0x111111, "422": 0x211111, "420": 0x221111}   # cv2.IMWRITE_JPEG_SAMPLING_FACTOR_*
SIZES = ((1, 1), (1, 17), (17, 1), (7, 9), (8, 8), (15, 15), (16, 16), (17, 17), (33, 65))


def noise(h, w, layout, seed):
    rng = np.random.default_rng(seed)
    return rng.integers(0, 256, (h, w) if layout == "gray" else (h, w, 3), np.uint8)


def smooth(h, w, layout, seed):
    """Gradients, a disc and mild noise: a photo-like frame that compresses as photos do."""
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[:h, :w].astype(np.float32)
    disc = np.hypot(y - h * 0.45, x - w * 0.55) < min(h, w) * 0.3
    img = np.stack([x / w * 200 + 30, y / h * 180 + 40, (np.sin(x / 7) * np.cos(y / 11) + 1) * 90], -1)
    img[disc] = img[disc] * 0.4 + np.array([90, 60, 200]) * 0.6
    img = np.clip(img + rng.normal(0, 4, img.shape), 0, 255).astype(np.uint8)
    return img[:, :, 1].copy() if layout == "gray" else img


def flat(h, w, layout, value):
    return np.full((h, w) if layout == "gray" else (h, w, 3), value, np.uint8)


def blocks(h, w, layout, seed):
    """8x8 blocks of black and white: DC differences of category 11 at q100."""
    rng = np.random.default_rng(seed)
    b = rng.integers(0, 2, (-(-h // 8), -(-w // 8))).astype(np.uint8) * 255
    img = np.kron(b, np.ones((8, 8), np.uint8))[:h, :w]
    return img if layout == "gray" else np.repeat(img[:, :, None], 3, 2)


def checker(h, w, layout, seed):
    """A one-pixel checkerboard: the largest AC categories, and long ZRL runs at q100."""
    img = ((np.add.outer(np.arange(h), np.arange(w)) & 1) * 255).astype(np.uint8)
    return img if layout == "gray" else np.repeat(img[:, :, None], 3, 2)


KINDS = {"noise": noise, "smooth": smooth, "flat": flat, "blocks": blocks, "checker": checker}


def cases():
    """name -> (kind, h, w, layout, seed or value, quality)."""
    c = {}
    for q in (1, 10, 50, 75, 95, 100):
        for lay in LAYOUTS:
            c[f"noise_q{q}_{lay}"] = ("noise", 23, 37, lay, 5, q)
            c[f"smooth_q{q}_{lay}"] = ("smooth", 40, 56, lay, 6, q)
    for h, w in SIZES:
        for lay in LAYOUTS:
            c[f"size_{h}x{w}_{lay}"] = ("noise", h, w, lay, 7, 95)
    for lay in LAYOUTS:
        c[f"size_1023x1025_{lay}"] = ("smooth", 1023, 1025, lay, 8, 95)
        for v in (0, 128, 255):
            c[f"flat{v}_{lay}"] = ("flat", 24, 40, lay, v, 95)
        c[f"blocks_q100_{lay}"] = ("blocks", 32, 48, lay, 9, 100)
        c[f"checker_q100_{lay}"] = ("checker", 16, 24, lay, 0, 100)
    c["ffpad_gray"] = ("noise", 8, 8, "gray", FFPAD_SEED, 95)   # the padded last byte is 0xFF, stuffed with 0x00
    return c


FFPAD_SEED = 3


def image(name):
    kind, h, w, lay, s, _ = cases()[name]
    return KINDS[kind](h, w, lay, s)


def params(name):
    """(quality, subsampling) of a fixture ('420' for gray, where cv2 ignores it)."""
    _, _, _, lay, _, q = cases()[name]
    return q, "420" if lay == "gray" else lay


def cv2_encode(img, quality=95, subsampling="420"):
    import cv2
    ok, buf = cv2.imencode(".jpg", img, [cv2.IMWRITE_JPEG_QUALITY, quality, cv2.IMWRITE_JPEG_SAMPLING_FACTOR,
                                         SAMPLING[subsampling]])
    assert ok
    return buf.tobytes()


def versions():
    import cv2
    m = re.search(r"JPEG:\s+\S*libjpeg-turbo \(ver ([^)]+)\)", cv2.getBuildInformation())
    return {"cv2": cv2.__version__, "libjpeg-turbo": m.group(1) if m else "unknown"}


def committed(name):
    _, h, w, _, _, _ = cases()[name]
    return h * w <= 1 << 16


def load(name):
    with open(os.path.join(HERE, name + ".jpg"), "rb") as f:
        return f.read()


def manifest():
    with open(os.path.join(HERE, "sha256.json")) as f:
        return json.load(f)


def main():
    out = {"versions": versions(), "files": {}}
    for name in cases():
        data = cv2_encode(image(name), *params(name))
        if committed(name):
            with open(os.path.join(HERE, name + ".jpg"), "wb") as f:
                f.write(data)
        out["files"][name] = hashlib.sha256(data).hexdigest()
    with open(os.path.join(HERE, "sha256.json"), "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
        f.write("\n")


if __name__ == "__main__":
    main()
