"""Serial reference of the dataset renderer (reference prepare_data/taichi_three `render_triangle`), for tests.

It runs the C oracle's restatement (`oracle_mesh_render` in oracle/mesh_oracle.c: faces in index order, the written fp32
op order) for one camera of the `taichi_three` stand-in, with the camera state the stand-in's renderer reads, and builds
the test meshes: the ring cameras of render_data.py and an adversarial mesh.
"""
import math

import numpy as np

from oracle import mesh_oracle


def ring_camera(angle, res=(1024, 1024), hr=False, dis=2.0, pitch=-8.0, look_at=(0.0, 0.85, 0.0)):
    """A stand-in Camera set up like render_data.py's `render()` (:147-172) for one view angle, `_init()` done."""
    from taichi_three import Camera
    from taichi_three.transform import rotationX, rotationY
    look_at = np.array(look_at)
    rotate = np.matmul(rotationY(math.radians(angle)), rotationX(math.radians(pitch)))
    cam_pos = look_at + np.matmul(rotate, np.array([0, 0, dis]))
    k = 2 if hr else 1
    cam = Camera(res=(res[0] * k, res[1] * k))
    cam.set_intrinsic(res[0] * 0.8 * k, res[1] * 0.8 * k, (res[0] * 0.5 - 0) * k, (res[1] * 0.5 + 25) * k)
    cam.set(pos=cam_pos, target=look_at)
    cam._init()
    return cam


def lights(seed=0, n=6):
    """(towards [n,3], colour [n,3]) of render_data.py's light ring (:86-95) with seeded tilts."""
    from taichi_three import Light
    from taichi_three.transform import rotationX, rotationY
    rng = np.random.default_rng(seed)
    out = []
    for l in range(n):
        rotate = np.matmul(rotationX(math.radians(rng.uniform(-30, 30))), rotationY(math.radians(360 // n * l)))
        out.append(Light([*np.matmul(rotate, np.array([0, 0, 1]))], color=[1.0, 1.0, 1.0]))
    return (np.array([li.towards for li in out], np.float32), np.array([li.colour for li in out], np.float32))


def oracle_render(cam, light_dir, light_color, verts, faces, uvs=None, face_uvs=None, tex=None):
    """The oracle's (img [H,W,3], zbuf [H,W], mask [H,W,3]) for a stand-in camera, in image layout ([y, x])."""
    rinv = np.array(cam._dev_inv_rot, np.float32).reshape(3, 3)
    img, zbuf, mask = mesh_oracle.render(cam.res, cam._dev_K, cam._dev_pos, rinv, light_dir, light_color, verts, faces,
                                         uvs, face_uvs, tex)
    return img.swapaxes(0, 1), zbuf.swapaxes(0, 1), mask.swapaxes(0, 1)


def adversarial_mesh(seed=0):
    """(verts, faces, uvs, face_uvs) seen from ring_camera(0): coplanar duplicates, shared edges, faces across every
    border, behind the camera and straddling z = 0, zero-area faces, large and small faces, uvs outside [0, 1]."""
    rng = np.random.default_rng(seed)
    V, F, T, FT = [], [], [], []

    def tri(p, uv=None):
        base = len(V)
        V.extend(p)
        F.append([base, base + 1, base + 2])
        tb = len(T)
        T.extend(uv if uv is not None else rng.uniform(-1.5, 2.5, (3, 2)))
        FT.append([tb, tb + 1, tb + 2])

    c = np.array([0.0, 0.85, 0.0])     # camera at (0, ~1.13, 1.98) looking at c: x right is world +x... approximately
    # a large quad (two triangles sharing an edge) in front of the body, then its coplanar duplicate on top (higher index)
    q = [c + [-0.5, -0.5, 0.3], c + [0.5, -0.5, 0.3], c + [0.5, 0.5, 0.3], c + [-0.5, 0.5, 0.3]]
    for _ in range(2):
        tri([q[0], q[2], q[1]]); tri([q[0], q[3], q[2]])
        tri([q[0], q[1], q[2]]); tri([q[0], q[2], q[3]])
    # faces across every border of the image and one covering all of it
    for sx, sy in ((-1, 0), (1, 0), (0, -1), (0, 1)):
        o = c + [sx * 1.3, sy * 1.3, 0.0]
        tri([o + [-0.6, -0.6, 0.1], o + [0.6, -0.5, 0.1], o + [0.0, 0.6, 0.1]])
        tri([o + [-0.6, -0.6, 0.1], o + [0.0, 0.6, 0.1], o + [0.6, -0.5, 0.1]])
    tri([c + [-20, -20, -0.5], c + [20, -20, -0.5], c + [0, 30, -0.5]])
    tri([c + [-20, -20, -0.5], c + [0, 30, -0.5], c + [20, -20, -0.5]])
    # behind the camera, and straddling its z = 0 plane (the camera sits near z = 1.98)
    for z0, z1 in ((3.0, 3.5), (1.5, 2.5), (2.4, 1.7)):
        tri([[-0.3, 1.0, z0], [0.3, 1.0, z1], [0.0, 1.3, z0]])
        tri([[-0.3, 1.0, z0], [0.0, 1.3, z0], [0.3, 1.0, z1]])
    # zero-area faces: a repeated vertex and a collinear triple
    tri([c, c, c + [0.1, 0.0, 0.0]])
    tri([c, c + [0.1, 0.1, 0.0], c + [0.2, 0.2, 0.0]])
    # many small random faces, some coplanar duplicates of each other, both windings
    for _ in range(3000):
        p = c + rng.uniform(-0.7, 0.7, 3) * [1, 1, 0.3]
        t = [p, p + rng.normal(0, 0.01, 3), p + rng.normal(0, 0.01, 3)]
        tri(t)
        if rng.uniform() < 0.1:
            tri(t)
    verts = np.array(V, np.float32)
    faces = np.array(F, np.int32)
    return verts, faces, np.array(T, np.float32), np.array(FT, np.int32)
