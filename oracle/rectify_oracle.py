"""numpy restatement of the stereo rectification of the real-data loader (reference lib/human_loader.py:245-366): the
zero-distortion rectify maps, cv2.remap INTER_LINEAR / BORDER_CONSTANT 0 on uint8 and float32 planes, the ground-truth
flow, the eroded valid mask and the tensor contract of stereo_to_dict_tensor.  No cv2 at run time: the device kernels
(csrc/rectify.cu) are checked against this file where cv2 is absent, and this file is checked against cv2 where it is
present (tests/test_rectify_cpu.py).

The rules (DESIGN.md §2, "Rectification"):
  1. maps: iR = inv(P[:3,:3] @ R) by the adjugate in fp64 (the op order of `inv_pr`), (X, Y, Z) = iR @ (u, v, 1),
     map = fp32(fx * (X / Z) + cx), fp32(fy * (Y / Z) + cy) with fx, fy, cx, cy from the SOURCE K.
  2. uint8: X = cvRound(mapx * 32), x0 = X >> 5, ax = X & 31 (same for y); weights (32-ax)(32-ay)*32, ax(32-ay)*32,
     (32-ax)ay*32, ax*ay*32 (sum 2^15); out = sat_u8((sum w*v + 2^14) >> 15); neighbours outside the source add 0.
  3. float32: the same quantised weights as floats, (1 - ax/32) * (1 - ay/32) etc., summed strictly left to right
     ((p00 + p01) + p10) + p11 in fp32, no FMA.
  4. erode 3x3 on float32 = 3x3 minimum with +inf outside.
  5. flow is fp64: offset - (-depth * Tf_x) (Tf_x -> -Tf_x for view 1), 0 where depth < 0.05, times valid.
"""
import numpy as np

INT_MIN = -(2 ** 31)


def inv_pr(P3, R):
    """iR = inv(P3 @ R) in fp64: the product with left-to-right sums, then adjugate / determinant.  Python floats, so
    every op is one IEEE double op in the written order (the device launcher computes the same expressions)."""
    P = [[float(P3[i][j]) for j in range(3)] for i in range(3)]
    Rm = [[float(R[i][j]) for j in range(3)] for i in range(3)]
    M = [[(P[i][0] * Rm[0][j] + P[i][1] * Rm[1][j]) + P[i][2] * Rm[2][j] for j in range(3)] for i in range(3)]
    c00 = M[1][1] * M[2][2] - M[1][2] * M[2][1]
    c01 = M[0][2] * M[2][1] - M[0][1] * M[2][2]
    c02 = M[0][1] * M[1][2] - M[0][2] * M[1][1]
    c10 = M[1][2] * M[2][0] - M[1][0] * M[2][2]
    c11 = M[0][0] * M[2][2] - M[0][2] * M[2][0]
    c12 = M[0][2] * M[1][0] - M[0][0] * M[1][2]
    c20 = M[1][0] * M[2][1] - M[1][1] * M[2][0]
    c21 = M[0][1] * M[2][0] - M[0][0] * M[2][1]
    c22 = M[0][0] * M[1][1] - M[0][1] * M[1][0]
    det = (M[0][0] * c00 + M[0][1] * c10) + M[0][2] * c20
    adj = [[c00, c01, c02], [c10, c11, c12], [c20, c21, c22]]
    return [[adj[i][j] / det for j in range(3)] for i in range(3)]


def rectify_maps(K, R, P3, H, W):
    """(mapx, mapy) float32 [H, W]: cv2.initUndistortRectifyMap(K, 0, R, P, (W, H), CV_32FC1) by rule 1."""
    iR = inv_pr(P3, R)
    u = np.arange(W, dtype=np.float64)[None, :]
    v = np.arange(H, dtype=np.float64)[:, None]
    X = (iR[0][0] * u + iR[0][1] * v) + iR[0][2]
    Y = (iR[1][0] * u + iR[1][1] * v) + iR[1][2]
    Z = (iR[2][0] * u + iR[2][1] * v) + iR[2][2]
    fx, fy, cx, cy = float(K[0][0]), float(K[1][1]), float(K[0][2]), float(K[1][2])
    with np.errstate(divide="ignore", invalid="ignore"):
        mapx = (fx * (X / Z) + cx).astype(np.float32)
        mapy = (fy * (Y / Z) + cy).astype(np.float32)
    return mapx, mapy


def fixed_point(m):
    """cvRound(m * 32) as int64, with cvRound's x86 result (INT_MIN) for NaN and out-of-range values."""
    s = m.astype(np.float32) * np.float32(32)
    ok = np.isfinite(s) & (s >= -2.0 ** 31) & (s < 2.0 ** 31)
    r = np.full(s.shape, INT_MIN, dtype=np.int64)
    r[ok] = np.rint(s[ok]).astype(np.int64)
    return r


def _taps(mapx, mapy, Hin, Win):
    X, Y = fixed_point(mapx), fixed_point(mapy)
    x0, y0, ax, ay = X >> 5, Y >> 5, X & 31, Y & 31
    taps = []
    for dy, dx in ((0, 0), (0, 1), (1, 0), (1, 1)):
        xs, ys = x0 + dx, y0 + dy
        inside = (xs >= 0) & (xs < Win) & (ys >= 0) & (ys < Hin)
        taps.append((np.where(inside, ys, 0), np.where(inside, xs, 0), inside))
    return ax, ay, taps


def remap_u8(src, mapx, mapy):
    """cv2.remap(src uint8 [Hin, Win(, C)], mapx, mapy, INTER_LINEAR) by rule 2."""
    Hin, Win = src.shape[:2]
    ax, ay, taps = _taps(mapx, mapy, Hin, Win)
    w = [(32 - ax) * (32 - ay) * 32, ax * (32 - ay) * 32, (32 - ax) * ay * 32, ax * ay * 32]
    acc = np.zeros(mapx.shape + src.shape[2:], dtype=np.int64)
    for wk, (ys, xs, inside) in zip(w, taps):
        v = src[ys, xs].astype(np.int64)
        if src.ndim == 3:
            wk, inside = wk[..., None], inside[..., None]
        acc += np.where(inside, wk * v, 0)
    return np.clip((acc + (1 << 14)) >> 15, 0, 255).astype(np.uint8)


def remap_f32(src, mapx, mapy):
    """cv2.remap(src float32 [Hin, Win], mapx, mapy, INTER_LINEAR) by rule 3."""
    Hin, Win = src.shape
    ax, ay, taps = _taps(mapx, mapy, Hin, Win)
    f = np.float32
    tx, ty = ax.astype(f) * f(1.0 / 32), ay.astype(f) * f(1.0 / 32)
    w = [(f(1) - ty) * (f(1) - tx), (f(1) - ty) * tx, ty * (f(1) - tx), ty * tx]
    p = [np.where(inside, src[ys, xs], f(0)) * wk for wk, (ys, xs, inside) in zip(w, taps)]
    return ((p[0] + p[1]) + p[2]) + p[3]


def erode3(v):
    """cv2.erode(v float32 [H, W], ones((3, 3))) by rule 4."""
    H, W = v.shape
    pad = np.full((H + 2, W + 2), np.inf, dtype=np.float32)
    pad[1:-1, 1:-1] = v
    out = pad[1:-1, 1:-1].copy()
    for dy in range(3):
        for dx in range(3):
            out = np.minimum(out, pad[dy:dy + H, dx:dx + W])
    return out


def flow_valid(depth_r, Tf_x, cx_self, cx_other, sign, mask_r):
    """The flow and valid of one view from its remapped depth and rectified mask (human_loader.py:74-85, :298-315).
    sign = +1 for view 0 (disparity -depth * Tf_x), -1 for view 1 (-depth * -Tf_x).  Returns (flow fp64, valid uint8)."""
    offset = float(cx_other) - float(cx_self)
    tf = float(Tf_x) if sign > 0 else -float(Tf_x)
    flow = offset - (-depth_r).astype(np.float64) * tf
    flow[depth_r < np.float32(0.05)] = 0
    valid = (mask_r[:, :, 0] / 255.0).astype(np.float32)
    valid = erode3(valid)
    valid = np.where(valid >= np.float32(0.66), np.float32(1), np.float32(0))
    flow = flow * valid.astype(np.float64)
    return flow, (valid * np.float32(255)).astype(np.uint8)


def tensor_contract(img_u8, mask_u8):
    """(img, mask) float32 CHW as stereo_to_dict_tensor makes them: img = (2 * (v / 255) - 1) * m_soft with m_soft =
    mask / 255, mask = (m_soft >= 0.5).  The divisions are fp32 divisions (CPU torch's uint8 / 255.0)."""
    f = np.float32
    v = np.moveaxis(img_u8, -1, 0).astype(f)
    m = np.moveaxis(mask_u8, -1, 0).astype(f) / f(255)
    img = (f(2) * (v / f(255)) - f(1)) * m
    return img, np.where(m >= f(0.5), f(1), f(0))


def rectify_pair(views, cams, src_res, depths=None):
    """The arrays of get_rectified_stereo_data for one pair.  views: ((img0, mask0), (img1, mask1)) uint8; cams:
    ((K0, R0, P0[:3,:3]), (K1, R1, P1[:3,:3])); depths: None or the two pts2depth outputs (float32 [Hin, Win]), with
    `cams` then also needing Tf_x in cams[2].  Returns the dict without 'camera'."""
    out = {}
    rd = []
    for k, ((img, mask), (K, R, P3)) in enumerate(zip(views, cams[:2])):
        mx, my = rectify_maps(K, R, P3, src_res, src_res)
        out[f"img{k}"] = remap_u8(img, mx, my)
        out[f"mask{k}"] = remap_u8(mask, mx, my)
        if depths is not None:
            rd.append(remap_f32(depths[k], mx, my))
    if depths is not None:
        Tf_x = cams[2]
        cx = (float(cams[0][2][0][2]), float(cams[1][2][0][2]))
        for k in range(2):
            out[f"flow{k}"], out[f"valid{k}"] = flow_valid(rd[k], Tf_x, cx[k], cx[1 - k], 1 - 2 * k, out[f"mask{k}"])
    return out
