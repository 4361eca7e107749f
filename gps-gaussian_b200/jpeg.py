"""Baseline JPEG decoding on the GPU (gpsg_jpeg_parse / gpsg_jpeg_decode, csrc/jpeg_decode.cu).

The result is always exactly what `np.array(Image.open(f))` returns, as a CUDA uint8 tensor: [H, W] for one component,
[H, W, 3] for YCbCr.  Baseline (SOF0 / SOF1) 8-bit Huffman JPEGs with 4:4:4, 4:2:2 or 4:2:0 chroma, or grayscale, are
decoded natively (DESIGN.md §2, "JPEG decoding"); anything else, and any image whose decode sets its status word
(a corrupt stream), is decoded by Pillow and uploaded, unless fallback=False, which raises JpegError instead.  So are
images above Pillow's decompression-bomb limit (`Image.MAX_IMAGE_PIXELS`, read at each call: Pillow then warns or raises
as it would) and scans of GPSG_JPEG_MAX_SCAN_BYTES or more.  The native route needs a CUDA device.

  decode(data | [data, ...], device=None, fallback=True) -> tensor | [tensor, ...]   one launch chain per call
  read_img_cuda(path, device=None)                       -> lib/human_loader.py's read_img, on the GPU
  supported(data)                                        -> whether `data` is decoded natively
  counts() / reset_counts()                              -> {'native': n, 'fallback': m} decodes so far
"""
import ctypes as C
import io
import os

import numpy as np
import torch

from . import _lib

MAX_BATCH = 64            # GPSG_JPEG_MAX_BATCH (include/gpsg.h)
MAX_SCAN_BYTES = 1 << 28  # GPSG_JPEG_MAX_SCAN_BYTES (include/gpsg.h): entropy-coded bytes of one call


class JpegInfo(C.Structure):
    """GpsgJpegInfo (include/gpsg.h)."""
    _fields_ = [("width", C.c_int32), ("height", C.c_int32), ("num_components", C.c_int32),
                ("restart_interval", C.c_int32), ("h_samp", C.c_int32 * 3), ("v_samp", C.c_int32 * 3),
                ("quant_id", C.c_int32 * 3), ("dc_id", C.c_int32 * 3), ("ac_id", C.c_int32 * 3),
                ("quant", (C.c_uint16 * 64) * 4), ("dc_bits", (C.c_uint8 * 16) * 4), ("ac_bits", (C.c_uint8 * 16) * 4),
                ("dc_vals", (C.c_uint8 * 256) * 4), ("ac_vals", (C.c_uint8 * 256) * 4), ("ecs_offset", C.c_int64),
                ("ecs_length", C.c_int64)]


_L = _lib.lib
_L.gpsg_jpeg_parse.restype = C.c_int
_L.gpsg_jpeg_parse.argtypes = [C.c_char_p, C.c_size_t, C.POINTER(JpegInfo)]
_L.gpsg_jpeg_decode_workspace_bytes.restype = C.c_size_t
_L.gpsg_jpeg_decode_workspace_bytes.argtypes = [C.c_int, C.POINTER(JpegInfo)]
_L.gpsg_jpeg_decode.restype = C.c_int
_L.gpsg_jpeg_decode.argtypes = [C.c_int, C.c_void_p, C.c_int, C.POINTER(JpegInfo), C.POINTER(C.c_void_p),
                                C.POINTER(C.c_void_p), C.c_void_p, C.c_void_p, C.c_size_t]

_COUNTS = {"native": 0, "fallback": 0}


class JpegError(ValueError):
    """An image that is not decoded natively, with fallback=False."""


def parse(data):
    """(code, JpegInfo): code 0 when decoded natively, else the GPSG_JPEG_E_* refusal."""
    info = JpegInfo()
    return int(_L.gpsg_jpeg_parse(bytes(data), len(data), C.byref(info))), info


def _native(data):
    """(decoded natively?, refusal code, JpegInfo)."""
    code, info = parse(data)
    if code:
        return False, code, info
    from PIL import Image
    limit = Image.MAX_IMAGE_PIXELS
    ok = info.ecs_length < MAX_SCAN_BYTES and (limit is None or info.width * info.height <= limit)
    return ok, code, info


def supported(data):
    """Whether `data` (the bytes of a JPEG file) is decoded natively."""
    return _native(data)[0]


def counts():
    return dict(_COUNTS)


def reset_counts():
    for k in _COUNTS:
        _COUNTS[k] = 0


def _pillow(data, device):
    from PIL import Image
    _COUNTS["fallback"] += 1
    return torch.from_numpy(np.array(Image.open(io.BytesIO(bytes(data))))).to(device)


def decode(data, device=None, fallback=True):
    """Decode one JPEG (bytes-like) or a list of them (one launch chain per GPSG_JPEG_MAX_BATCH images); returns uint8
    tensors on `device` (default: the current CUDA device) shaped like Pillow's array.  A non-CUDA device is refused
    (ValueError) when an image would take the native route."""
    single = isinstance(data, (bytes, bytearray, memoryview))
    items = [bytes(data)] if single else [bytes(d) for d in data]
    device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
    out = [None] * len(items)
    native = []
    for k, d in enumerate(items):
        ok, code, info = _native(d)
        if ok:
            native.append((k, info, d))
        elif not fallback:
            raise JpegError(f"jpeg: not decoded natively (GPSG_JPEG_E code {code})" if code else
                            "jpeg: not decoded natively (above the pixel or scan-size limit)")
    if native and device.type != "cuda":
        raise ValueError(f"jpeg.decode: the native route needs a CUDA device, got {device}")
    on_gpu = {k for k, _, _ in native}
    for k, d in enumerate(items):
        if k not in on_gpu:
            out[k] = _pillow(d, device)
    batch, size = [], 0
    for item in native:                       # batches within GPSG_JPEG_MAX_BATCH and GPSG_JPEG_MAX_SCAN_BYTES
        if batch and (len(batch) == MAX_BATCH or size + item[1].ecs_length >= MAX_SCAN_BYTES):
            _decode_batch(batch, out, device, fallback)
            batch, size = [], 0
        batch.append(item)
        size += item[1].ecs_length
    if batch:
        _decode_batch(batch, out, device, fallback)
    return out[0] if single else out


def _decode_batch(batch, out, device, fallback):
    n = len(batch)
    infos = (JpegInfo * n)(*[info for _, info, _ in batch])
    offs = np.cumsum([0] + [len(d) for _, _, d in batch])
    blob = torch.from_numpy(np.frombuffer(b"".join(d for _, _, d in batch), np.uint8).copy()).to(device)
    imgs = []
    for _, info, _ in batch:
        shape = (info.height, info.width) if info.num_components == 1 else (info.height, info.width, 3)
        imgs.append(torch.empty(shape, dtype=torch.uint8, device=device))
    status = torch.empty(n, dtype=torch.int32, device=device)
    wsb = int(_L.gpsg_jpeg_decode_workspace_bytes(n, infos))
    if wsb == 0:
        raise _lib.GpsgError("gpsg_jpeg_decode_workspace_bytes refused a parsed batch")
    ws = torch.empty(wsb + 256, dtype=torch.uint8, device=device)
    base = (ws.data_ptr() + 255) // 256 * 256
    data_p = (C.c_void_p * n)(*[blob.data_ptr() + int(offs[i]) for i in range(n)])
    out_p = (C.c_void_p * n)(*[t.data_ptr() for t in imgs])
    idx, stream = _lib.device_stream(device)
    with torch.cuda.device(device):
        rc = _L.gpsg_jpeg_decode(idx, stream, n, infos, data_p, out_p, status.data_ptr(), base, wsb)
    _lib.check(rc, "gpsg_jpeg_decode")
    st = status.cpu().numpy()            # the one host synchronisation of the batch
    for (k, _, d), t, s in zip(batch, imgs, st):
        if s == 0:
            out[k] = t
            _COUNTS["native"] += 1
        elif not fallback:
            raise JpegError(f"jpeg: the stream is not decodable (GPSG_JPEG_ST bits {int(s):#x})")
        else:
            out[k] = _pillow(d, device)


def read_img_cuda(path, device=None):
    """lib/human_loader.py's read_img (np.array(Image.open(path))) as a CUDA tensor; a list of paths is decoded in one
    call and gives a list."""
    single = isinstance(path, (str, bytes, os.PathLike))
    datas = []
    for p in [path] if single else path:
        with open(p, "rb") as f:
            datas.append(f.read())
    got = decode(datas, device)
    return got[0] if single else got
