"""Dataset renderer without a GPU: the C ABI's exports, workspace size and refusals; the `taichi_three` stand-in's
`readobj` against the reference's own loader and its cameras against render_data.py's conventions; and the serial
oracle (oracle/mesh_oracle.c) on analytic scenes."""
import ctypes as C
import importlib.util
import math
import os

import numpy as np
import pytest

import mesh_reference as mr

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_LOADER = os.path.join(ROOT, "oracle", "_ref", "prepare_data", "taichi_three", "loader.py")


# ---- C ABI --------------------------------------------------------------------------------------------------------

def _L(built_lib):
    from gps_gaussian_b200 import _lib
    return _lib


def _scene(L, n_cams=1, w=8, h=8, ptr=None):
    s = L.MeshScene()
    s.num_cameras, s.num_lights = n_cams, 0
    for k in range(n_cams):
        c = s.cameras[k]
        c.width, c.height = w, h
        c.img = c.zbuf = c.mask = ptr
    return s


def test_abi_exports_and_workspace(built_lib):
    L = _L(built_lib)
    for name in ("gpsg_mesh_render_workspace_bytes", "gpsg_mesh_render"):
        assert name in L.EXPORTED and hasattr(C.CDLL(built_lib), name)
    ws = L.lib.gpsg_mesh_render_workspace_bytes
    small, big = ws(1000, 1024 * 1024), ws(1000, 2048 * 2048)
    assert small >= 1024 * 1024 * 8 + 1000 * 64 and big - small >= 3 * 1024 * 1024 * 8
    assert ws(2000, 1024 * 1024) > small and ws(0, 16) > 0
    assert ws(-1, 16) == 0 and ws(10, 0) == 0 and ws(10, 1 << 31) == 0
    assert C.sizeof(L.MeshScene) > 0 and L.lib.gpsg_version() == 90


def test_abi_refusals(built_lib):
    L = _L(built_lib)
    f = L.lib.gpsg_mesh_render
    buf = (C.c_float * 4096)()
    p = C.cast(buf, C.c_void_p).value
    ws_aligned = (C.c_uint8 * (1 << 16))()
    wsp = (C.cast(ws_aligned, C.c_void_p).value + 255) // 256 * 256
    mesh = L.Mesh(p, p, None, None, None, 3, 1, 0, 0, 0)

    def err(m, s, w=wsp, nbytes=1 << 15):
        assert f(0, None, m, s, w, nbytes) == -1
        return L.lib.gpsg_last_error().decode()

    assert "negative count" in err(L.Mesh(p, p, None, None, None, -1, 1, 0, 0, 0), _scene(L, ptr=p))
    assert "num_cameras" in err(mesh, _scene(L, 0, ptr=p))
    assert "num_cameras" in err(mesh, _bad_cams(L, p))
    s = _scene(L, ptr=p)
    s.num_lights = L.MESH_MAX_LIGHTS + 1
    assert "num_lights" in err(mesh, s)
    assert "uvs and face_uvs" in err(L.Mesh(p, p, p, None, None, 3, 1, 3, 0, 0), _scene(L, ptr=p))
    assert "texture sizes" in err(L.Mesh(p, p, None, None, p, 3, 1, 0, 0, 4), _scene(L, ptr=p))
    assert "NULL pointer" in err(L.Mesh(p, None, None, None, None, 3, 1, 0, 0, 0), _scene(L, ptr=p))
    assert "camera size" in err(mesh, _scene(L, 1, 0, 8, ptr=p))
    assert "2^31 pixels" in err(mesh, _scene(L, 1, 65536, 32768, ptr=p))
    assert "NULL pointer" in err(mesh, _scene(L, ptr=None))
    assert "NULL pointer" in err(mesh, _scene(L, ptr=p), w=None)
    assert "256-byte aligned" in err(mesh, _scene(L, ptr=p), w=wsp + 8)
    assert "smaller than" in err(mesh, _scene(L, ptr=p), nbytes=16)


def _bad_cams(L, p):
    s = _scene(L, 1, ptr=p)
    s.num_cameras = L.MESH_MAX_CAMERAS + 1
    return s


# ---- readobj against the reference's loader ------------------------------------------------------------------------

OBJS = {
    "tri_v_vt_vn": "# c\nmtllib a.mtl\no body\nv 0 0 0\nv 1 0 0\nv 0 1 0\nv 1 1 0.5\nvt 0 0\nvt 1 0\nvt 0 1\nvt 1 1\n"
                   "vn 0 0 1\nusemtl m\nf 1/1/1 2/2/1 3/3/1\nf 2/2/1 4/4/1 3/3/1\n",
    "quad_v_vt": "v 0 0 0\nv 1 0 0\nv 1 1 0\nv 0 1 0\nvt 0 0\nvt 1 0\nvt 1 1\nvt 0 1\nf 1/1 2/2 3/3 4/4\n",
    "v_vn": "v 0 0 0\nv 1 0 0\nv 0 1 0\nv 1 1 1\nvn 0 0 1\nf 1//1 2//1 3//1 4//1\n",
    "bare_v": "v 0.5 0 0\n\nv 1 0 0\nv 0 1 0\ns off\ng grp\nf 1 2 3\n   \nv 2 2 2 0.1 0.2 0.3\n",
    "mixed_bad_numbers": "v 0 0 0\nv 1 x 0\nv 1 0 0\nv 0 1 0\nvt 0.1 0.2\nvt nope\nf 1/1 3/1 4/1\n",
}


@pytest.mark.skipif(not os.path.exists(REF_LOADER), reason="oracle/_ref is not staged")
@pytest.mark.parametrize("name", sorted(OBJS))
@pytest.mark.parametrize("scale", [1, 0.37])
def test_readobj_matches_reference_loader(tmp_path, name, scale):
    from taichi_three import readobj
    spec = importlib.util.spec_from_file_location("_ref_t3_loader", REF_LOADER)
    ref = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(ref)
    path = tmp_path / f"{name}.obj"
    path.write_text(OBJS[name])
    try:
        want = ref.readobj(str(path), scale=scale)
    except ValueError:                                 # ragged rows: the reference cannot build its arrays either
        with pytest.raises(ValueError):
            readobj(str(path), scale=scale)
        return
    got = readobj(str(path), scale=scale)
    assert set(got) == set(want)
    for k in want:
        if want[k] is None:
            assert got[k] is None, k
        else:
            assert got[k].dtype == want[k].dtype and got[k].shape == want[k].shape, k
            assert got[k].tobytes() == want[k].tobytes(), k


@pytest.mark.skipif(not os.path.exists(REF_LOADER), reason="oracle/_ref is not staged")
def test_readobj_procedural_scan_matches_reference(tmp_path):
    from gps_gaussian_b200 import synth_mesh
    from taichi_three import readobj
    spec = importlib.util.spec_from_file_location("_ref_t3_loader", REF_LOADER)
    ref = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(ref)
    obj, _ = synth_mesh.procedural_scan(4000, 64, seed=3)
    synth_mesh.write_obj(str(tmp_path / "s.obj"), obj)
    got, want = readobj(str(tmp_path / "s.obj")), ref.readobj(str(tmp_path / "s.obj"))
    for k in ("vi", "vt", "f"):
        assert got[k].tobytes() == want[k].tobytes()
    assert got["vn"] is None and want["vn"] is None
    assert np.array_equal(got["f"], obj["f"]) and np.abs(got["vi"] - obj["vi"]).max() < 1e-6


# ---- cameras --------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("angle", [0, 23, 97.5, 180, 301])
@pytest.mark.parametrize("hr", [False, True])
def test_ring_camera_export(angle, hr):
    from gps_gaussian_b200 import synth
    cam = mr.ring_camera(angle, hr=hr)
    K, E = cam.export_intrinsic(), cam.export_extrinsic()
    assert K.dtype == np.float64 and E.dtype == np.float64 and K.shape == (3, 3) and E.shape == (3, 4)
    R, t = E[:, :3], E[:, 3]
    assert np.abs(R @ R.T - np.eye(3)).max() < 1e-12 and abs(np.linalg.det(R) - 1) < 1e-12
    x = K @ (R @ np.array([0.0, 0.85, 0.0]) + t)
    assert np.abs(x[:2] / x[2] - K[:2, 2]).max() < 1e-9 and x[2] > 0
    if not hr:
        Ks, Es = synth.ring_camera(angle, 1024)
        assert np.abs(K - Ks).max() < 1e-9 and np.abs(E - Es).max() < 1e-9


# ---- the oracle on analytic scenes ---------------------------------------------------------------------------------

def _front_camera(res=(64, 64), f=10.0):
    """Camera at the origin looking down world +z with fx = fy = f, cx = cy = 0: camera (x, y, z) = world (-x, -y, z),
    so a camera-space point (x, y, f) lands on screen (x, y)."""
    from taichi_three import Camera
    cam = Camera(res=res)
    cam.set_intrinsic(f, f, 0.0, 0.0)
    cam.set(pos=[0.0, 0.0, 0.0], target=[0.0, 0.0, 1.0])
    cam._init()
    return cam


def _world(screen_xy, d=10.0, f=10.0):
    """World points whose camera-space depth is d and which land on the given screen points."""
    s = np.asarray(screen_xy, np.float64)
    return np.stack([-s[:, 0] * d / f, -s[:, 1] * d / f, np.full(len(s), d)], -1).astype(np.float32)


QUAD = [(-5.5, -3.5), (20.5, -3.5), (20.5, 30.5), (-5.5, 30.5)]
FRONT = [[0, 3, 2], [0, 2, 1]]          # (a - b) x (a - c) points at the camera: drawn


def _no_lights():
    return np.zeros((0, 3), np.float32), np.zeros((0, 3), np.float32)


def test_oracle_fronto_parallel_quad_coverage_depth_and_texels():
    d = 10.0
    cam = _front_camera()
    verts = _world(QUAD, d)
    tw = th = 64
    tex = np.random.default_rng(1).uniform(0, 1, (tw, th, 3)).astype(np.float32)
    uvs = (np.array(QUAD, np.float32) + 0.0) / np.float32(tw)      # uv * 64 = the screen position
    img, zbuf, mask = mr.oracle_render(cam, *_no_lights(), verts, np.array(FRONT, np.int32), uvs, np.array(FRONT, np.int32),
                                       tex)
    want = np.zeros((64, 64), bool)
    want[1:31, 1:21] = True                          # y in [1, 30], x in [1, 20]: row and column 0 are never drawn
    assert np.array_equal(mask[..., 0] == 1, want) and np.array_equal(mask[..., 1], mask[..., 2])
    assert np.abs(zbuf[want] * d - 1).max() < 1e-6 and (zbuf[~want] == 0).all() and (img[~want] == 0).all()
    colour = np.sqrt(np.array([0.0, 0.01, 0.05], np.float32))      # no light: sqrt(mix(blue, orange, 0))
    ys, xs = np.nonzero(want)
    texel = tex[xs, ys]                              # tex[i, j] at uv * (Wt, Ht) = (i, j): pixel (x, y) reads tex[x, y]
    ok = colour > 0
    assert np.abs(img[ys, xs][:, ok] / colour[ok] - texel[:, ok]).max() < 2e-5


def test_oracle_reversed_winding_draws_nothing():
    cam = _front_camera()
    back = np.array([f[::-1] for f in FRONT], np.int32)
    img, zbuf, mask = mr.oracle_render(cam, *_no_lights(), _world(QUAD), back)
    assert not img.any() and not zbuf.any() and not mask.any()


def test_oracle_coplanar_overlap_higher_index_wins():
    cam = _front_camera()
    tex = np.zeros((8, 8, 3), np.float32)
    tex[:4, :, 0] = 1.0                              # i < 4: red; i >= 4: blue
    tex[4:, :, 2] = 1.0
    verts = _world(QUAD)
    faces = np.array(FRONT + FRONT, np.int32)
    uvs = np.array([[0.25, 0.5], [0.75, 0.5]], np.float32)
    for first, second in ((0, 1), (1, 0)):
        fu = np.array([[first] * 3] * 2 + [[second] * 3] * 2, np.int32)
        img, _, mask = mr.oracle_render(cam, [[0, 0, -1]], [[1, 1, 1]], verts, faces, uvs, fu, tex)
        on = mask[..., 0] == 1
        chan = 0 if second == 0 else 2
        assert on.sum() == 600 and (img[on][:, chan] > 0).all() and (img[on][:, 2 - chan] == 0).all()


@pytest.mark.parametrize("light", [(0.3, -0.2, -1.0), (0.0, 0.0, -1.0), (0.9, 0.4, 0.2), (-0.5, 0.5, -0.4)])
def test_oracle_single_light_face_colour_closed_form(light):
    from taichi_three import Light
    cam = _front_camera()
    li = Light(list(light), color=[0.7, 1.0, 0.4])
    ld, lc = np.array([li.towards], np.float32), np.array([li.colour], np.float32)
    img, _, mask = mr.oracle_render(cam, ld, lc, _world(QUAD), np.array(FRONT, np.int32))
    on = mask[..., 0] == 1
    assert on.any() and (img[on] == img[on][0]).all()          # flat shading
    n = np.array([0.0, 0.0, -1.0])                            # camera-space normal of a face that faces the camera
    l = np.linalg.inv(np.array(cam._axes).T) @ np.array(li.towards)
    t = n @ l
    s = 0.58 * max(0.0, t) + 0.04 * (t * 0.5 + 0.5) + 0.3 * max(n @ (l * 0.5), 0.0) ** 10
    col = np.sqrt(np.array([0.0, 0.01, 0.05]) * (1 - s * lc[0]) + np.array([1.19, 1.04, 0.98]) * s * lc[0])
    assert np.abs(img[on][0] - col).max() < 2e-6


def test_standin_surface_and_refusals():
    import taichi_three as t3
    from taichi_three import transform
    for name in ("rotationX", "rotationY", "rotationZ", "math", "ti", "Camera"):
        assert hasattr(transform, name)
    assert transform.math is math and hasattr(transform.ti, "init")
    with pytest.raises(NotImplementedError):
        t3.SimpleModel
    with pytest.raises(NotImplementedError):
        t3.Camera(res=(8, 8)).from_mouse(None)
    with pytest.raises(NotImplementedError):
        t3.Light([0, 0, 1]).set([1, 0, 0])
    m = t3.StaticModel(4, obj={"vi": np.zeros((5, 3), np.float32), "vt": None, "vn": None,
                               "f": np.zeros((1, 3, 1), np.int32)})
    assert m.corner_fields == 1 and not hasattr(m, "init_tex")


def test_standin_does_not_draw_from_numpy_random():
    import taichi_three as t3
    np.random.seed(1314)
    before = np.random.get_state()
    cam = t3.Camera(res=(16, 16))
    cam.set_intrinsic(12.8, 12.8, 8, 8)
    cam.set(pos=[0, 1, 2], target=[0, 0.85, 0])
    cam._init()
    t3.Lights([t3.Light([0, 0, 1])]).init_data()
    cam.export_extrinsic(), cam.export_intrinsic()
    after = np.random.get_state()
    assert np.array_equal(after[1], before[1]) and after[2:] == before[2:]


# ---- the import finder: `python prepare_data/render_data.py` puts a shadowing taichi_three first on sys.path --------

PROBE = """
import taichi_three as t3
from taichi_three.transform import *
print(t3.__file__)
print(rotationX.__module__, ti.__name__, math.__name__)
"""


@pytest.mark.parametrize("patch", [True, False])
def test_patch_finder_beats_a_shadowing_taichi_three(tmp_path, patch):
    """A script run as `python dir/script.py` has dir first on sys.path; dir holds a `taichi_three` package that cannot
    import (the reference's needs Taichi).  With GPSG_PATCH=1 the stand-in is imported anyway; without it the shadowing
    package is, and fails."""
    import subprocess
    import sys
    from gps_gaussian_b200 import harness
    shadow = tmp_path / "prepare_data"
    (shadow / "taichi_three").mkdir(parents=True)
    (shadow / "taichi_three" / "__init__.py").write_text("raise ImportError('shadowing taichi_three imported')\n")
    (shadow / "probe.py").write_text(PROBE)
    p = subprocess.run([sys.executable, str(shadow / "probe.py")], cwd=str(tmp_path), env=harness.script_env(patch=patch),
                       capture_output=True, text=True, timeout=300)
    if patch:
        assert p.returncode == 0, p.stderr[-3000:]
        first, second = p.stdout.splitlines()[-2:]
        assert os.path.realpath(first) == os.path.realpath(
            os.path.join(ROOT, "gps-gaussian_b200", "dropin", "taichi_three", "__init__.py"))
        assert second == "taichi_three.transform taichi math"
    else:
        assert p.returncode != 0 and "shadowing taichi_three imported" in p.stderr


def test_oracle_nonfinite_uv_gives_canonical_nan():
    cam = _front_camera()
    tex = np.random.default_rng(4).uniform(0, 1, (8, 8, 3)).astype(np.float32)
    uvs = np.array([[np.nan, 0.5], [np.inf, 0.5], [-np.inf, np.nan], [0.25, 0.25]], np.float32)
    img, _, mask = mr.oracle_render(cam, [[0, 0, -1]], [[1, 1, 1]], _world(QUAD), np.array(FRONT, np.int32), uvs,
                                    np.array(FRONT, np.int32), tex)
    on = mask[..., 0] == 1
    bits = np.ascontiguousarray(img[on]).view(np.uint32)
    assert on.sum() == 600 and (bits == 0x7FFFFFFF).all()
