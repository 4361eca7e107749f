"""Seeded stereo pairs for the rectification tests: ring cameras like prepare_data/render_data.py (a rotation about the
vertical axis, the camera 2.5 m from the centre), with their own K per view, soft-edged masks whose values cross 0.5*255
and 0.66*255, and an inverse-depth blob on a zero background (the `depth < 0.05` branch of the flow)."""
import numpy as np


def ring_extr(angle_deg, rng, tilt_deg=0.0, dist=2.5):
    a = np.deg2rad(angle_deg)
    Ry = np.array([[np.cos(a), 0, -np.sin(a)], [0, 1, 0], [np.sin(a), 0, np.cos(a)]])
    t = np.deg2rad(tilt_deg) * rng.uniform(-1, 1)
    Rx = np.array([[1, 0, 0], [0, np.cos(t), -np.sin(t)], [0, np.sin(t), np.cos(t)]])
    R = Rx @ Ry
    c = np.array([dist * np.sin(a), rng.uniform(-0.1, 0.1), -dist * np.cos(a)])
    E = np.zeros((3, 4))
    E[:, :3], E[:, 3] = R, -R @ c
    return E


def intr(H, W, rng):
    f = max(H, W) * rng.uniform(1.8, 2.6)
    return np.array([[f * rng.uniform(0.97, 1.03), 0, W / 2 + rng.uniform(-8, 8)],
                     [0, f, H / 2 + rng.uniform(-8, 8)], [0, 0, 1]])


def image(H, W, rng, C=3):
    yy, xx = np.mgrid[0:H, 0:W]
    base = 127 + 100 * np.sin(xx[..., None] / 7.0 + np.arange(C)) * np.cos(yy[..., None] / 11.0)
    return np.clip(base + rng.normal(0, 20, (H, W, C)), 0, 255).astype(np.uint8)


def soft_mask(H, W, rng, C=3, empty=False):
    if empty:
        return np.zeros((H, W, C), np.uint8)
    yy, xx = np.mgrid[0:H, 0:W]
    r = np.hypot((yy - H / 2) / (0.35 * H), (xx - W / 2) / (0.22 * W))
    m = np.clip((1.0 - r) * 6.0 + 0.5, 0, 1) * 255           # a ramp of ~1/6 of the radius: every byte value occurs
    return np.repeat(np.rint(m).astype(np.uint8)[..., None], C, -1)


def inv_depth(S, rng):
    """Inverse depth [S, S] float32 (what read_depth returns): ~1/2.5 m on an ellipse, 0 (background) elsewhere."""
    yy, xx = np.mgrid[0:S, 0:S]
    r = np.hypot((yy - S / 2) / (0.4 * S), (xx - S / 2) / (0.25 * S))
    d = np.where(r < 1, 0.4 + 0.02 * np.cos(xx / 5.0) + rng.uniform(-0.005, 0.005, (S, S)), 0.0)
    return d.astype(np.float32)


def pair(seed, Hin, Win, angle=22.5, tilt=0.0, C=3, Cm=3, empty=False):
    """(img0, mask0, K0, E0), (img1, mask1, K1, E1) of one seeded pair."""
    rng = np.random.default_rng(seed)
    views = []
    for k, a in enumerate((0.0, angle)):
        views.append((image(Hin, Win, rng, C), soft_mask(Hin, Win, rng, Cm, empty), intr(Hin, Win, rng),
                      ring_extr(a, rng, tilt)))
    return views


def stereo_rectify(K0, E0, K1, E1, src_res):
    """cv2.stereoRectify as the loader calls it; returns R0, R1, P0, P1."""
    import cv2
    r0, t0 = E0[:3, :3], E0[:3, 3:]
    r1, t1 = E1[:3, :3], E1[:3, 3:]
    A = np.eye(4)
    A[:3, :3], A[:3, 3:] = r0.T, -r0.T @ t0
    B = np.eye(4)
    B[:3, :3], B[:3, 3:] = r1, t1
    E = B @ A
    return cv2.stereoRectify(K0, np.zeros(4), K1, np.zeros(4), (src_res, src_res), E[:3, :3], E[:3, 3], flags=0)[:4]
