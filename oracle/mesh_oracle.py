"""ctypes wrapper of oracle/mesh_oracle.c, the serial restatement of the dataset renderer's triangle rasterizer (test
infrastructure, not product).

The shared library is compiled on first use with the oracle's flags (gcc -O2 -ffp-contract=off -fno-fast-math) into
oracle/_build/, or into the system temporary directory when the tree is read-only; `build()` (called by
`__graft_entry__.build()`) does the same ahead of time.

Why a recipe of its own rather than an entry in oracle/build.py's SRCS: the existing oracle files, that recipe included,
are the project's yardsticks and are kept byte for byte, so a new checker is added beside them, not into them.  The flags
are oracle/build.py's minus -fopenmp (this restatement is serial) and without the f64 variant (it is fp32 only).  The
library name carries a hash of the source, so a stale build is never loaded.
"""
import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "mesh_oracle.c")
_LIB = None


def _target():
    with open(SRC, "rb") as f:
        tag = hashlib.sha256(f.read()).hexdigest()[:16]
    name = f"libmesh_oracle_{tag}.so"
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
                               SRC, "-lm", "-o", tmp])
        os.replace(tmp, dst)
    return dst


def _lib():
    global _LIB
    if _LIB is None:
        _LIB = C.CDLL(build())
        _LIB.oracle_mesh_render.restype = C.c_int
    return _LIB


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def render(res, K, pos, rinv, light_dir, light_color, verts, face_verts, uvs=None, face_uvs=None, tex=None):
    """One camera.  res = (res0, res1); K = (fx, fy, cx, cy); pos [3]; rinv [3,3] = trans^-1 (rounded to fp32 here);
    light_dir / light_color [L,3]; verts [V,3]; face_verts [F,3]; uvs [T,2] and face_uvs [F,3] or None; tex [Wt,Ht,3] or
    None.  Returns (img [res0,res1,3], zbuf [res0,res1], mask [res0,res1,3]) float32: the reference's field layout."""
    W, H = int(res[0]), int(res[1])
    f32 = lambda a: np.ascontiguousarray(np.asarray(a, np.float32))
    i32 = lambda a: np.ascontiguousarray(np.asarray(a, np.int32))
    verts, fv = f32(verts).reshape(-1, 3), i32(face_verts).reshape(-1, 3)
    ld, lc = f32(light_dir).reshape(-1, 3), f32(light_color).reshape(-1, 3)
    uvs = None if uvs is None else f32(uvs).reshape(-1, 2)
    ft = None if face_uvs is None else i32(face_uvs).reshape(-1, 3)
    tex = None if tex is None else f32(tex)
    img = np.empty((W, H, 3), np.float32)
    zbuf = np.empty((W, H), np.float32)
    mask = np.empty((W, H, 3), np.float32)
    fx, fy, cx, cy = (C.c_float(float(np.float32(v))) for v in K)
    _lib().oracle_mesh_render(
        C.c_int(W), C.c_int(H), fx, fy, cx, cy, _p(f32(pos)), _p(f32(rinv).reshape(9)), C.c_int(len(ld)), _p(ld), _p(lc),
        _p(verts), C.c_int(len(verts)), _p(fv), C.c_int(len(fv)), _p(uvs), _p(ft), C.c_int(0 if uvs is None else len(uvs)),
        _p(tex), C.c_int(0 if tex is None else tex.shape[0]), C.c_int(0 if tex is None else tex.shape[1]), _p(img),
        _p(zbuf), _p(mask))
    return img, zbuf, mask
