"""Flat-shaded, textured triangle mesh rendering on sm_90a (gpsg_mesh_render, csrc/mesh_render.cu): the renderer of the
reference's dataset script (prepare_data/taichi_three, `render_triangle`), deterministic and race-free.

    cam = mesh_render.camera((1024, 1024), fx, fy, cx, cy, pos, trans)      # trans: columns right, up, fwd
    (img, zbuf, mask), = mesh_render.render(verts, faces, [cam], light_dirs, light_colors, uvs, face_uvs, tex)

img [H,W,3], zbuf [H,W] (inverse depth: 1 / camera-space z, interpolated affinely on screen) and mask [H,W,3] are fp32
CUDA tensors with H = res[1], W = res[0]: the reference's `(res0, res1)` fields transposed to image layout, i.e. what
`field.to_numpy().swapaxes(0, 1)` gives.  Per pixel the face with the largest zindex wins, the highest face index among
equal zindex: the serial reading of the reference's loop, whatever the execution order.
"""
import ctypes as C
from typing import NamedTuple

import numpy as np
import torch

from . import _lib

MAX_CAMERAS = _lib.MESH_MAX_CAMERAS
MAX_LIGHTS = _lib.MESH_MAX_LIGHTS


class Camera(NamedTuple):
    """One pinhole camera of a render: res = (res0, res1) = (width, height), fp32 intrinsics, position and trans^-1."""
    res: tuple
    fx: float
    fy: float
    cx: float
    cy: float
    pos: tuple
    inv_rot: tuple        # 9 floats, row-major


def camera(res, fx, fy, cx, cy, pos, trans):
    """A Camera from the reference's quantities: `trans` [3,3] has the columns right, up, fwd and maps camera to world;
    its inverse is taken in fp64 and rounded to fp32 (the formulation csrc/mesh_render.cu documents)."""
    res = (int(res[0]), int(res[1]))
    if res[0] < 1 or res[1] < 1:
        raise ValueError(f"mesh_render.camera: res must be >= 1, got {res}")
    inv = np.linalg.inv(np.asarray(trans, np.float64).reshape(3, 3))
    f = lambda v: float(np.float32(v))
    return Camera(res, f(fx), f(fy), f(cx), f(cy), tuple(f(v) for v in np.asarray(pos, np.float64).reshape(3)),
                  tuple(f(v) for v in inv.reshape(9)))


def _check(name, t, dtype, cols, device):
    if not torch.is_tensor(t) or not t.is_cuda or t.dtype != dtype:
        raise TypeError(f"mesh_render: {name} must be a CUDA {dtype} tensor")
    if not t.is_contiguous():
        raise TypeError(f"mesh_render: {name} must be contiguous")
    if device is not None and t.device != device:
        raise TypeError(f"mesh_render: {name} is on {t.device}, verts on {device}")
    if cols is not None and (t.dim() != 2 or t.shape[1] != cols):
        raise ValueError(f"mesh_render: {name} must be [n, {cols}], got {tuple(t.shape)}")


def render(verts, faces, cameras, light_dirs=None, light_colors=None, uvs=None, face_uvs=None, tex=None):
    """Render the mesh into every camera (one launch chain on the current stream, no synchronisation).

    verts [V,3] fp32, faces [F,3] int32 vertex indices; uvs [T,2] fp32 with face_uvs [F,3] int32, or neither (every
    corner samples uv = (0, 0)); tex [Wt,Ht,3] fp32, indexed tex[i, j] at uv * (Wt, Ht) = (i, j) like the reference's
    texture field, or None (the sample is 1).  light_dirs / light_colors [L,3] (L <= 16): each light's unit vector
    towards the light (= -normalize(dir)) and colour; the face colour is 0.58 Lambert + 0.04 half-Lambert + 0.3 Blinn-Phong^10 summed over
    them, then mapped through sqrt(mix(blue, orange, c)).  All tensors on one CUDA device, contiguous.  A face whose index
    is out of range draws nothing.  Returns [(img, zbuf, mask)] per camera."""
    _check("verts", verts, torch.float32, 3, None)
    dev = verts.device
    _check("faces", faces, torch.int32, 3, dev)
    if (uvs is None) != (face_uvs is None):
        raise ValueError("mesh_render: uvs and face_uvs go together")
    if uvs is not None:
        _check("uvs", uvs, torch.float32, 2, dev)
        _check("face_uvs", face_uvs, torch.int32, 3, dev)
        if face_uvs.shape[0] != faces.shape[0]:
            raise ValueError(f"mesh_render: face_uvs has {face_uvs.shape[0]} rows, faces {faces.shape[0]}")
    if tex is not None:
        _check("tex", tex, torch.float32, None, dev)
        if tex.dim() != 3 or tex.shape[2] != 3 or tex.shape[0] < 1 or tex.shape[1] < 1:
            raise ValueError(f"mesh_render: tex must be [Wt, Ht, 3], got {tuple(tex.shape)}")
    cameras = list(cameras)
    if not 1 <= len(cameras) <= _lib.MESH_MAX_CAMERAS:
        raise ValueError(f"mesh_render: 1 to {_lib.MESH_MAX_CAMERAS} cameras, got {len(cameras)}")
    ld = np.zeros((0, 3), np.float32) if light_dirs is None else np.asarray(light_dirs, np.float32).reshape(-1, 3)
    lc = np.ones_like(ld) if light_colors is None else np.asarray(light_colors, np.float32).reshape(-1, 3)
    if ld.shape != lc.shape or len(ld) > _lib.MESH_MAX_LIGHTS:
        raise ValueError(f"mesh_render: up to {_lib.MESH_MAX_LIGHTS} lights with one colour each, got {ld.shape} / {lc.shape}")

    p = lambda t: None if t is None or t.numel() == 0 else t.data_ptr()
    mesh = _lib.Mesh(p(verts), p(faces), p(uvs), p(face_uvs), p(tex), int(verts.shape[0]), int(faces.shape[0]),
                     0 if uvs is None else int(uvs.shape[0]), 0 if tex is None else int(tex.shape[0]),
                     0 if tex is None else int(tex.shape[1]))
    scene = _lib.MeshScene()
    scene.num_cameras, scene.num_lights = len(cameras), len(ld)
    for i in range(len(ld)):
        scene.light_dir[i][:] = [float(v) for v in ld[i]]
        scene.light_color[i][:] = [float(v) for v in lc[i]]
    outs = []
    for k, cam in enumerate(cameras):
        W, H = cam.res
        img = torch.empty((H, W, 3), dtype=torch.float32, device=dev)
        zbuf = torch.empty((H, W), dtype=torch.float32, device=dev)
        mask = torch.empty((H, W, 3), dtype=torch.float32, device=dev)
        c = scene.cameras[k]
        c.width, c.height, c.fx, c.fy, c.cx, c.cy = W, H, cam.fx, cam.fy, cam.cx, cam.cy
        c.pos[:] = list(cam.pos)
        c.inv_rot[:] = list(cam.inv_rot)
        c.img, c.zbuf, c.mask = img.data_ptr(), zbuf.data_ptr(), mask.data_ptr()
        outs.append((img, zbuf, mask))
    max_pixels = max(c.res[0] * c.res[1] for c in cameras)
    nbytes = int(_lib.lib.gpsg_mesh_render_workspace_bytes(int(faces.shape[0]), max_pixels))
    if nbytes == 0:
        raise ValueError(f"mesh_render: a camera has too many pixels ({max_pixels})")
    ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    with torch.cuda.device(dev):
        rc = _lib.lib.gpsg_mesh_render(*_lib.device_stream(dev), mesh, scene, C.c_void_p(ws.data_ptr()), nbytes)
    _lib.check(rc, "gpsg_mesh_render")
    return outs
