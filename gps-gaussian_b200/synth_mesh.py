"""Seeded procedural textured meshes for the dataset renderer's tests and timing (no scan data ships with the project).

`procedural_scan` is a human-sized body made of bumpy closed lat-long surfaces (torso, head, arms, legs) with a uv
layout and a random texture; `uv_sphere` is an exact-radius sphere for geometric checks.  Faces are wound so that
(b - a) x (c - a) points outwards, the orientation the reference's renderer draws.
"""
import math
import os

import numpy as np


def lat_long(center, radii, nlat, nlon, rng=None, bump=0.0):
    """Closed lat-long surface of about 2 * nlat * nlon triangles (the poles' degenerate ones dropped): verts [V,3],
    faces [F,3] (outward), uvs [V,2]."""
    th = np.linspace(0.0, math.pi, nlat + 1)
    ph = np.linspace(0.0, 2 * math.pi, nlon + 1)
    T, P = np.meshgrid(th, ph, indexing="ij")
    r = np.ones_like(T)
    if rng is not None and bump > 0:
        for _ in range(4):
            k, m, a, s = rng.integers(1, 6), rng.integers(1, 6), rng.uniform(0, bump), rng.uniform(0, 2 * math.pi)
            r = r + a * np.sin(k * T) * np.cos(m * P + s)
    d = np.stack([np.sin(T) * np.cos(P), np.cos(T), np.sin(T) * np.sin(P)], -1) * r[..., None]
    verts = (np.asarray(center, np.float64) + d * np.asarray(radii, np.float64)).reshape(-1, 3)
    uvs = np.stack([P / (2 * math.pi), 1.0 - T / math.pi], -1).reshape(-1, 2)
    idx = np.arange((nlat + 1) * (nlon + 1)).reshape(nlat + 1, nlon + 1)
    a, b, c, e = idx[:-1, :-1], idx[1:, :-1], idx[1:, 1:], idx[:-1, 1:]
    faces = np.concatenate([np.stack([a, b, c], -1).reshape(-1, 3), np.stack([a, c, e], -1).reshape(-1, 3)])
    v = verts[faces]
    n = np.cross(v[:, 1] - v[:, 0], v[:, 2] - v[:, 0])
    area = np.linalg.norm(n, axis=1)
    faces = faces[area > 1e-12]                          # the poles' degenerate triangles
    v, n = verts[faces], n[area > 1e-12]
    out = np.einsum("ij,ij->i", n, v.mean(1) - np.asarray(center)) >= 0
    faces[~out] = faces[~out][:, ::-1]
    return verts.astype(np.float32), faces.astype(np.int32), uvs.astype(np.float32)


def uv_sphere(center=(0.0, 0.85, 0.0), radius=0.4, nlat=96, nlon=192):
    """(verts, faces, uvs) of a sphere whose vertices lie exactly (up to fp32) on the given sphere."""
    return lat_long(center, (radius, radius, radius), nlat, nlon)


_PARTS = (  # centre, radii, share of the faces
    ((0.0, 1.15, 0.0), (0.20, 0.32, 0.12), 0.34),   # torso
    ((0.0, 1.62, 0.0), (0.10, 0.12, 0.11), 0.10),   # head
    ((-0.30, 1.15, 0.0), (0.06, 0.30, 0.06), 0.09),  # arms
    ((0.30, 1.15, 0.0), (0.06, 0.30, 0.06), 0.09),
    ((-0.10, 0.45, 0.0), (0.08, 0.44, 0.08), 0.19),  # legs
    ((0.10, 0.45, 0.0), (0.08, 0.44, 0.08), 0.19),
)


def procedural_scan(n_faces=100_000, tex_size=1024, seed=0):
    """(obj, texture): obj is `readobj`'s dict ('vi' [V,3], 'vt' [V,2], 'vn' None, 'f' [F,3,2] = v/vt) of a ~1.8 m body
    with about n_faces triangles; texture is a [tex_size, tex_size, 3] uint8 image (what cv2.imread returns)."""
    rng = np.random.default_rng(seed)
    vs, fs, ts, off = [], [], [], 0
    for center, radii, share in _PARTS:
        nlon = max(8, int(math.sqrt(n_faces * share)))
        nlat = max(4, int(n_faces * share / (2 * nlon)) + 1)
        v, f, t = lat_long(center, radii, nlat, nlon, rng, bump=0.06)
        vs.append(v); fs.append(f + off); ts.append(t); off += len(v)
    vi, f, vt = np.concatenate(vs), np.concatenate(fs), np.concatenate(ts)
    obj = {"vi": vi, "vt": vt, "vn": None, "f": np.stack([f, f], -1).astype(np.int32)}
    base = rng.integers(0, 256, (tex_size // 16 + 1, tex_size // 16 + 1, 3)).astype(np.float32)
    tex = np.kron(base, np.ones((16, 16, 1), np.float32))[:tex_size, :tex_size]
    tex = np.clip(tex + rng.normal(0, 12, tex.shape), 0, 255).astype(np.uint8)
    return obj, tex


def write_obj(path, obj):
    """Wavefront OBJ of a readobj-style dict, one-based, faces as v, v/vt or v/vt/vn by the dict's last axis."""
    os.makedirs(os.path.dirname(os.path.abspath(path)), exist_ok=True)
    lines = ["# procedural mesh"]
    lines += ["v %.7f %.7f %.7f" % tuple(p) for p in obj["vi"]]
    if obj.get("vt") is not None:
        lines += ["vt %.7f %.7f" % tuple(p) for p in obj["vt"]]
    if obj.get("vn") is not None:
        lines += ["vn %.7f %.7f %.7f" % tuple(p) for p in obj["vn"]]
    f = obj["f"] + 1
    if f.shape[2] == 1:
        lines += ["f %d %d %d" % tuple(r[:, 0]) for r in f]
    else:
        fmt = " ".join(["/".join(["%d"] * f.shape[2])] * 3)
        lines += [("f " + fmt) % tuple(r.reshape(-1)) for r in f]
    with open(path, "w") as fh:
        fh.write("\n".join(lines) + "\n")
