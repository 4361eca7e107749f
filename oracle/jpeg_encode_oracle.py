"""ctypes wrapper of oracle/jpeg_encode_oracle.c, the serial restatement of the baseline JPEG encoder (test
infrastructure, not product).

Built like oracle/jpeg_oracle.py (the decoder's, beside which it sits): gcc -O2 into oracle/_build/, or into the system
temporary directory when the tree is read-only, under a name that carries a hash of the source; `build()` (called by
`__graft_entry__.build()`) does the same ahead of time.
"""
import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "jpeg_encode_oracle.c")
_LIB = None
SAMPLINGS = ("444", "422", "420")


def _target():
    with open(SRC, "rb") as f:
        tag = hashlib.sha256(f.read()).hexdigest()[:16]
    name = f"libjpeg_encode_oracle_{tag}.so"
    out = os.path.join(HERE, "_build")
    try:
        os.makedirs(out, exist_ok=True)
        if os.access(out, os.W_OK):
            return os.path.join(out, name)
    except OSError:
        pass
    return os.path.join(tempfile.gettempdir(), name)


def build():
    """Compile the oracle if its source changed; returns the library path."""
    dst = _target()
    if not os.path.exists(dst):
        tmp = f"{dst}.{os.getpid()}.tmp"
        subprocess.check_call(["gcc", "-O2", "-fPIC", "-shared", "-std=c11", "-Wall", SRC, "-o", tmp])
        os.replace(tmp, dst)
    return dst


def _lib():
    global _LIB
    if _LIB is None:
        _LIB = C.CDLL(build())
        _LIB.oracle_jpeg_encode_max_bytes.restype = C.c_long
        _LIB.oracle_jpeg_encode_max_bytes.argtypes = [C.c_int] * 4
        _LIB.oracle_jpeg_encode.restype = C.c_long
        _LIB.oracle_jpeg_encode.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_long, C.c_int, C.c_int, C.c_int,
                                            C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_long]
    return _LIB


def geometry(H, W, nc, subsampling="420"):
    """(hmax, vmax, MCU columns, MCU rows, blocks per MCU) of an image."""
    hmax = 2 if nc == 3 and subsampling != "444" else 1
    vmax = 2 if nc == 3 and subsampling == "420" else 1
    mx, my = -(-W // (8 * hmax)), -(-H // (8 * vmax))
    return hmax, vmax, mx, my, (hmax * vmax + 2 if nc == 3 else 1)


def encode(img, quality=95, subsampling="420", order="rgb", stages=False):
    """The JPEG file of a uint8 [H, W] or [H, W, 3] array (any strides), as bytes: what cv2.imencode('.jpg') writes for
    the BGR array (order='bgr' takes the array as cv2 does).  stages=True returns (file, planes [nc, ph, pw] uint8,
    coef [blocks, 64] int16 in zigzag order, MCU order, DC before prediction)."""
    img = np.asarray(img)
    if img.dtype != np.uint8 or img.ndim not in (2, 3) or (img.ndim == 3 and img.shape[2] != 3):
        raise ValueError("encode: uint8 [H, W] or [H, W, 3]")
    if subsampling not in SAMPLINGS or order not in ("rgb", "bgr"):
        raise ValueError("encode: subsampling in 444/422/420, order in rgb/bgr")
    H, W = img.shape[:2]
    nc = 1 if img.ndim == 2 else 3
    a = np.ascontiguousarray(img)
    cap = int(_lib().oracle_jpeg_encode_max_bytes(W, H, nc, int(subsampling)))
    out = np.empty(cap, np.uint8)
    planes = coef = None
    pw = 0
    if stages:
        hmax, vmax, mx, my, bpm = geometry(H, W, nc, subsampling)
        pw = 8 * mx * hmax
        planes = np.zeros((nc, 8 * my * vmax, pw), np.uint8)
        coef = np.zeros((mx * my * bpm, 64), np.int16)
    n = _lib().oracle_jpeg_encode(a.ctypes.data, W, H, nc, W * nc, int(order == "bgr"), int(quality), int(subsampling),
                                  None if planes is None else planes.ctypes.data, pw,
                                  None if coef is None else coef.ctypes.data, out.ctypes.data, cap)
    if n < 0:
        raise ValueError("encode: refused")
    data = out[:n].tobytes()
    return (data, planes, coef) if stages else data


def max_bytes(H, W, nc, subsampling="420"):
    return int(_lib().oracle_jpeg_encode_max_bytes(W, H, nc, int(subsampling)))
