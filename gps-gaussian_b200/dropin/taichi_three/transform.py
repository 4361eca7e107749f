"""Rotations and the pinhole camera of the stand-in (reference prepare_data/taichi_three/transform.py).

The script star-imports this module and uses `rotationX`, `rotationY`, `math.radians` and `ti.init` from it, so `math`
and `ti` (the `taichi` stand-in) are public names here on purpose.
"""
import math

import taichi as ti
import numpy as np

from .common import AutoInit, repo_on_path, unsupported


def rotationX(angle):
    c, s = math.cos(angle), math.sin(angle)
    return [[1, 0, 0], [0, c, -s], [0, s, c]]


def rotationY(angle):
    c, s = math.cos(angle), math.sin(angle)
    return [[c, 0, s], [0, 1, 0], [-s, 0, c]]


def rotationZ(angle):
    c, s = math.cos(angle), math.sin(angle)
    return [[c, -s, 0], [s, c, 0], [0, 0, 1]]


def _normalized(v):
    n = math.sqrt(sum(x ** 2 for x in v))
    return [x / n for x in v]


def _cross(a, b):
    return [a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0]]


class Buffer:
    """A camera output (the reference's `img`, `zbuf` or `mask` field): `to_numpy()` gives the field's (res0, res1[, 3])
    float32 layout.  The data stays on the GPU until it is read."""

    def __init__(self, res, channels):
        self.shape = tuple(res)
        self._channels = channels
        self._data = None

    def _set(self, t):
        self._data = t

    def to_numpy(self):
        if self._data is None:
            shape = self.shape + ((self._channels,) if self._channels else ())
            return np.zeros(shape, np.float32)
        return self._data.cpu().numpy().swapaxes(0, 1)

    def to_torch(self, device=None):
        """The data in image layout [res1, res0(, 3)] (a CUDA tensor)."""
        return self._data if device is None else self._data.to(device)


def _given(value, default):
    """The reference's `value or default`: None and 0 both mean 'not given'."""
    return value if value else default


def _f32(values):
    return tuple(float(np.float32(v)) for v in values)


class Camera(AutoInit):
    """Rectilinear pinhole camera with the reference's conventions.

    `set()` places it at `pos` looking at `target`; its axes are x = normalize(up x fwd), y = fwd x x, z = fwd, with the
    default `up` = (0, -1, 0), so image y points down.  A new pose takes effect at once, new intrinsics at `_init()`.
    Until a pose or intrinsics are first uploaded the camera renders nothing (a NaN rotation), like the reference's
    zero-initialised fields."""

    def __init__(self, res=None, fx=None, fy=None, cx=None, cy=None, pos=(0, 0, -2), target=(0, 0, 0), up=(0, -1, 0),
                 fov=30):
        width, height = res if res else (512, 512)
        self.res = (width, height)
        self.img, self.zbuf, self.mask = Buffer(self.res, 3), Buffer(self.res, 0), Buffer(self.res, 3)
        tan_fov = math.tan(math.radians(fov))
        self.cx, self.cy = _given(cx, width // 2), _given(cy, height // 2)
        self.fx, self.fy = _given(fx, self.cx / tan_fov), _given(fy, self.cy / tan_fov)
        self._eye, self._look, self._up = pos, target, up
        self._axes = None                   # camera x, y, z axes in world coordinates (float64 lists)
        self._dev_pos, self._dev_inv_rot, self._dev_K = (0.0,) * 3, (math.nan,) * 9, (0.0,) * 4
        self.set(init=True)

    def set_intrinsic(self, fx=None, fy=None, cx=None, cy=None):
        self.fx, self.fy = _given(fx, self.fx), _given(fy, self.fy)
        if cx is not None:
            self.cx = cx
        if cy is not None:
            self.cy = cy

    def set(self, pos=None, target=None, up=None, init=False):
        """Move the camera (an `up` given here is used for this pose only, as in the reference)."""
        if pos is not None:
            self._eye = pos
        if target is not None:
            self._look = target
        eye, look = self._eye, self._look
        fwd = _normalized([look[k] - eye[k] for k in range(3)])
        x_axis = _normalized(_cross(self._up if up is None else up, fwd))
        self._axes = (x_axis, _cross(fwd, x_axis), fwd)
        if not init:
            self._upload_pose()

    def _upload_pose(self):
        cam_to_world = np.array(self._axes, np.float64).T
        self._dev_pos = _f32(self._eye)
        self._dev_inv_rot = _f32(np.linalg.inv(cam_to_world).reshape(9))

    def _init(self):
        self._upload_pose()
        self._dev_K = _f32((self.fx, self.fy, self.cx, self.cy))

    def render_camera(self):
        """The gps_gaussian_b200.mesh_render.Camera the next render draws with."""
        repo_on_path()
        from gps_gaussian_b200 import mesh_render
        return mesh_render.Camera(tuple(int(r) for r in self.res), *self._dev_K, self._dev_pos, self._dev_inv_rot)

    @property
    def eye(self):
        """The camera position last given to `set()` (or the constructor)."""
        return self._eye

    @property
    def target(self):
        return self._look

    def export_intrinsic(self):
        """K, float64 [3,3]."""
        return np.array([[self.fx, 0.0, self.cx], [0.0, self.fy, self.cy], [0.0, 0.0, 1.0]], dtype=np.float64)

    def export_extrinsic(self):
        """[R | t], float64 [3,4]: R's rows are the camera axes, t = -R pos (world to camera)."""
        world_to_cam = np.array(self._axes, np.float64)
        return np.concatenate([world_to_cam, (-world_to_cam @ np.asarray(self._eye, np.float64))[:, None]], axis=1)

    def __getattr__(self, name):
        if name.startswith("__"):
            raise AttributeError(name)
        raise unsupported(f"Camera.{name}")
