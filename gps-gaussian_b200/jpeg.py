"""Baseline JPEG decoding and encoding on the GPU (gpsg_jpeg_parse / gpsg_jpeg_decode, csrc/jpeg_decode.cu;
gpsg_jpeg_encode, csrc/jpeg_encode.cu).

Decoding:

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

Encoding writes exactly the file `cv2.imencode('.jpg', bgr, [IMWRITE_JPEG_QUALITY, q, IMWRITE_JPEG_SAMPLING_FACTOR, s])`
and Pillow's `save(f, 'JPEG', quality=q, subsampling=s)` write (DESIGN.md §2, "JPEG encoding"):

  encode(img | [img, ...], quality=95, subsampling='420', order='rgb') -> bytes | [bytes]   one launch chain per batch
  imwrite_cuda(path, img, quality=95, subsampling='420', order='rgb')  -> True, the file written
  encode_host(arr, quality, subsampling, order)  -> bytes of a host array, uploaded through a reused pinned buffer
  encode_counts() / reset_encode_counts()         -> {'native': n, 'fallback': m}: files encoded here, and cv2.imwrite
                                                     calls the GPSG_ENCODE route (patch.py) left to cv2
"""
import ctypes as C
import io
import os
import threading

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
_ENC_COUNTS = {"native": 0, "fallback": 0}


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


# ---- encoding ----------------------------------------------------------------------------------------------------------
ORDERS = {"rgb": 0, "bgr": 1}                 # GPSG_JPEG_ORDER_* (include/gpsg.h)
SAMPLINGS = {"444": 444, "422": 422, "420": 420}
MAX_CALL_BYTES = 1 << 30                      # output bound of one launch chain; larger lists are split


class JpegEncodeDesc(C.Structure):
    """GpsgJpegEncodeDesc (include/gpsg.h)."""
    _fields_ = [("width", C.c_int32), ("height", C.c_int32), ("channels", C.c_int32), ("order", C.c_int32),
                ("quality", C.c_int32), ("sampling", C.c_int32), ("pitch", C.c_int64)]


_L.gpsg_jpeg_encode_max_bytes.restype = C.c_size_t
_L.gpsg_jpeg_encode_max_bytes.argtypes = [C.POINTER(JpegEncodeDesc)]
_L.gpsg_jpeg_encode_workspace_bytes.restype = C.c_size_t
_L.gpsg_jpeg_encode_workspace_bytes.argtypes = [C.c_int, C.POINTER(JpegEncodeDesc)]
_L.gpsg_jpeg_encode.restype = C.c_int
_L.gpsg_jpeg_encode.argtypes = [C.c_int, C.c_void_p, C.c_int, C.POINTER(JpegEncodeDesc), C.POINTER(C.c_void_p),
                                C.POINTER(C.c_void_p), C.c_void_p, C.c_void_p, C.c_size_t]


def encode_counts():
    return dict(_ENC_COUNTS)


def reset_encode_counts():
    for k in _ENC_COUNTS:
        _ENC_COUNTS[k] = 0


def _sampling(subsampling):
    s = SAMPLINGS.get(str(subsampling))
    if s is None:
        raise ValueError(f"jpeg.encode: subsampling must be one of {sorted(SAMPLINGS)}, got {subsampling!r}")
    return s


def _prepare(img, quality, sampling, order):
    """(uint8 CUDA tensor whose rows are the image's, descriptor)."""
    if not isinstance(img, torch.Tensor) or img.device.type != "cuda" or img.dtype != torch.uint8:
        raise ValueError("jpeg.encode: images must be CUDA uint8 tensors")
    if img.dim() == 3 and img.shape[2] == 1:
        img = img[:, :, 0]
    if not (img.dim() == 2 or (img.dim() == 3 and img.shape[2] == 3)):
        raise ValueError(f"jpeg.encode: expected [H, W] or [H, W, 3], got {tuple(img.shape)}")
    H, W = int(img.shape[0]), int(img.shape[1])
    if not (1 <= H <= 65500 and 1 <= W <= 65500):
        raise ValueError(f"jpeg.encode: sizes must lie in 1..65500, got {H}x{W}")
    nc = 1 if img.dim() == 2 else 3
    inner = (img.stride(1) == 1) if nc == 1 else (img.stride(2) == 1 and img.stride(1) == 3)
    if not inner or (H > 1 and img.stride(0) < W * nc):
        img = img.contiguous()
    pitch = img.stride(0) if H > 1 else W * nc
    d = JpegEncodeDesc(W, H, nc, ORDERS[order], int(quality), sampling, pitch)
    if _L.gpsg_jpeg_encode_max_bytes(C.byref(d)) == 0:
        raise ValueError(f"jpeg.encode: refused descriptor (quality {quality})")
    return img, d


def encode(img, quality=95, subsampling="420", order="rgb"):
    """Encode one CUDA uint8 image ([H, W] gray, [H, W, 1] or [H, W, 3], any row pitch) or a list of them as JPEG files;
    returns bytes (a list for a list).  order='rgb' gives cv2.imencode('.jpg', img[..., ::-1]) of the host array, 'bgr'
    cv2.imencode('.jpg', img).  Gray images ignore `subsampling`.  Per batch of at most GPSG_JPEG_MAX_BATCH images: one
    launch chain and two host synchronisations (the file sizes, then the downloads of exactly those bytes)."""
    single = isinstance(img, torch.Tensor)
    items = [img] if single else list(img)
    if order not in ORDERS:
        raise ValueError(f"jpeg.encode: order must be 'rgb' or 'bgr', got {order!r}")
    if isinstance(quality, bool) or int(quality) != quality or not 1 <= quality <= 100:
        raise ValueError(f"jpeg.encode: quality must be an integer in 1..100, got {quality!r}")
    sampling = _sampling(subsampling)
    prepared = [_prepare(t, quality, sampling, order) for t in items]
    out = []
    batch, size = [], 0
    for p in prepared:
        mb = int(_L.gpsg_jpeg_encode_max_bytes(C.byref(p[1])))
        if batch and (len(batch) == MAX_BATCH or size + mb > MAX_CALL_BYTES):
            out += _encode_batch(batch)
            batch, size = [], 0
        batch.append(p)
        size += mb
    if batch:
        out += _encode_batch(batch)
    return out[0] if single else out


def _encode_batch(batch):
    n = len(batch)
    device = batch[0][0].device
    if any(t.device != device for t, _ in batch):
        raise ValueError("jpeg.encode: the images of one call must share a device")
    descs = (JpegEncodeDesc * n)(*[d for _, d in batch])
    caps = [int(_L.gpsg_jpeg_encode_max_bytes(C.byref(d))) for _, d in batch]
    wsb = int(_L.gpsg_jpeg_encode_workspace_bytes(n, descs))
    if wsb == 0:
        raise ValueError("jpeg.encode: batch too large for one call")
    offs = np.cumsum([0] + caps)
    blob = torch.empty(int(offs[-1]), dtype=torch.uint8, device=device)
    sizes = torch.empty(n, dtype=torch.int64, device=device)
    ws = torch.empty(wsb + 256, dtype=torch.uint8, device=device)
    base = (ws.data_ptr() + 255) // 256 * 256
    src_p = (C.c_void_p * n)(*[t.data_ptr() for t, _ in batch])
    out_p = (C.c_void_p * n)(*[blob.data_ptr() + int(offs[i]) for i in range(n)])
    idx, stream = _lib.device_stream(device)
    with torch.cuda.device(device):
        rc = _L.gpsg_jpeg_encode(idx, stream, n, descs, src_p, out_p, sizes.data_ptr(), base, wsb)
    _lib.check(rc, "gpsg_jpeg_encode")
    got = sizes.cpu().tolist()               # host synchronisation 1 of the batch: the file sizes
    host = torch.empty(max(sum(got), 1), dtype=torch.uint8, pin_memory=True)
    ends = np.cumsum([0] + got)
    with torch.cuda.device(device):
        for i in range(n):                   # only the files come down, all on the stream, into pinned memory
            host[int(ends[i]):int(ends[i + 1])].copy_(blob[int(offs[i]):int(offs[i]) + got[i]], non_blocking=True)
        torch.cuda.current_stream(device).synchronize()   # host synchronisation 2: every download
    buf = host.numpy()
    files = [buf[int(ends[i]):int(ends[i + 1])].tobytes() for i in range(n)]
    _ENC_COUNTS["native"] += n
    return files


def fits_one_call(H, W, channels, subsampling="420"):
    """Whether one image of this shape fits one gpsg_jpeg_encode launch chain (else encode() refuses it)."""
    d = (JpegEncodeDesc * 1)(JpegEncodeDesc(W, H, channels, 0, 95, _sampling(subsampling), W * channels))
    return _L.gpsg_jpeg_encode_workspace_bytes(1, d) != 0


def imwrite_cuda(path, img, quality=95, subsampling="420", order="rgb"):
    """Write `encode(img, ...)` to `path`; returns True."""
    data = encode(img, quality, subsampling, order)
    with open(path, "wb") as f:
        f.write(data)
    return True


_STAGING = {}   # device -> (pinned host buffer, device buffer), grown as needed and reused
_STAGING_LOCK = threading.Lock()   # one caller at a time fills, uploads and encodes from the staging buffers


def encode_host(arr, quality=95, subsampling="420", order="rgb", device=None):
    """encode() of a host uint8 array ([H, W], [H, W, 1] or [H, W, 3], any strides, negative ones included): copied once
    into a reused pinned buffer, uploaded, encoded; only the file comes back.  Safe from several threads: the copy, the
    upload and the encode of one call hold a lock, so no call overwrites the staging buffers another has not finished
    with (cv2.imwrite releases the GIL, and a thread pool of writers is a common pattern)."""
    device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
    arr = np.asarray(arr)
    if arr.ndim == 3 and arr.shape[2] == 1:
        arr = arr[:, :, 0]
    n = arr.size
    with _STAGING_LOCK:
        host, dev = _STAGING.get(device, (None, None))
        if host is None or host.numel() < n:
            host = torch.empty(max(n, 1 << 20), dtype=torch.uint8, pin_memory=True)
            dev = torch.empty(host.numel(), dtype=torch.uint8, device=device)
            _STAGING[device] = (host, dev)
        np.copyto(host[:n].numpy().reshape(arr.shape), arr)
        d = dev[:n]
        with torch.cuda.device(device):
            d.copy_(host[:n], non_blocking=True)    # on the stream encode() launches on, and waits for
            return encode(d.view(arr.shape), quality, subsampling, order)
