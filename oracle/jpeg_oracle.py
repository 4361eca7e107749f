"""ctypes wrapper of oracle/jpeg_oracle.c, the serial restatement of the baseline JPEG decoder (test infrastructure, not
product).

The shared library is compiled on first use with the oracle's flags (gcc -O2 -ffp-contract=off -fno-fast-math) into
oracle/_build/, or into the system temporary directory when the tree is read-only; `build()` (called by
`__graft_entry__.build()`) does the same ahead of time.  As with oracle/mesh_oracle.py, the recipe sits beside
oracle/build.py rather than in its SRCS, which stays as it is; the library name carries a hash of the source, so a stale
build is never loaded.
"""
import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "jpeg_oracle.c")
_LIB = None


def _target():
    with open(SRC, "rb") as f:
        tag = hashlib.sha256(f.read()).hexdigest()[:16]
    name = f"libjpeg_oracle_{tag}.so"
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
        subprocess.check_call(["gcc", "-O2", "-fPIC", "-shared", "-std=c11", "-ffp-contract=off", "-fno-fast-math", "-Wall",
                               SRC, "-o", tmp])
        os.replace(tmp, dst)
    return dst


def _lib():
    global _LIB
    if _LIB is None:
        _LIB = C.CDLL(build())
        _LIB.oracle_jpeg_parse.restype = C.c_int
        _LIB.oracle_jpeg_parse.argtypes = [C.c_char_p, C.c_size_t, C.POINTER(C.c_int)]
        _LIB.oracle_jpeg_decode.restype = C.c_int
        _LIB.oracle_jpeg_decode.argtypes = [C.c_char_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int]
    return _LIB


def parse(data):
    """(refusal code, (W, H, ncomp, restart interval)); code 0 = decoded natively (GPSG_JPEG_E_* in include/gpsg.h)."""
    dims = (C.c_int * 4)()
    rc = _lib().oracle_jpeg_parse(bytes(data), len(data), dims)
    return rc, tuple(dims)


def decode(data, stages=False):
    """Decode one JPEG.  Returns (status, image) with image shaped like np.array(Image.open(f)) ([H, W] or [H, W, 3]
    uint8); status is 0, -refusal code, or the GPSG_JPEG_ST_* bits of the first decode error (image None then).
    stages=True: returns (status, image, coef [blocks, 64] int16 in MCU order, planes [ncomp, ph, pw] uint8)."""
    data = bytes(data)
    rc, (W, H, nc, _) = parse(data)
    if rc:
        return (-rc, None, None, None) if stages else (-rc, None)
    out = np.empty((H, W, nc) if nc == 3 else (H, W), np.uint8)
    coef = planes = None
    pw = 0
    if stages:
        hmax, vmax = _sampling(data)
        mx, my = -(-W // (8 * hmax)), -(-H // (8 * vmax))
        bpm = hmax * vmax + (nc - 1)
        coef = np.zeros((mx * my * bpm, 64), np.int16)
        pw = mx * hmax * 8
        planes = np.zeros((nc, my * vmax * 8, pw), np.uint8)
    st = _lib().oracle_jpeg_decode(data, len(data), out.ctypes.data, None if coef is None else coef.ctypes.data,
                                   None if planes is None else planes.ctypes.data, pw)
    if st:
        out = None
    return (st, out, coef, planes) if stages else (st, out)


def _sampling(data):
    """Luma (H, V) sampling factors of the frame header."""
    i = 2
    while i + 4 <= len(data):
        m, ln = data[i + 1], (data[i + 2] << 8) | data[i + 3]
        if m in (0xC0, 0xC1):
            s = data[i + 4 + 7]
            return s >> 4, s & 15
        i += 2 + ln
    raise ValueError("no SOF0/SOF1 header")
