"""Fixed-capacity textured mesh of the stand-in (reference prepare_data/taichi_three/model.py `StaticModel`)."""
import numpy as np
import torch

from .common import AutoInit, unsupported


class StaticModel(AutoInit):
    """A mesh of capacity N (vertices, uvs and faces each), drawn flat-shaded with a bilinear texture lookup.

    obj is `readobj`'s dict; tex is a [Wt, Ht, 3] uint8-valued array (the script passes the JPEG transposed and flipped)
    or None.  The face layout (corner fields: 1 = v, 2 = v/vt, 3 = v/vt/vn) is fixed at construction from which of
    `vt` / `vn` the obj has, and the texture's shape from `tex`, as the reference's fields are.  `_init()` uploads
    `init_obj` / `init_tex` to the GPU: faces beyond the obj's count draw nothing (the reference's zero padding gives them
    a NaN normal), and an obj with more than N vertices, uvs or faces raises."""

    def __init__(self, N, obj=None, tex=None):
        self.N = int(N)
        if obj is None:
            self.corner_fields = 1
        else:
            self.corner_fields = 3 if obj['vn'] is not None else 2 if obj['vt'] is not None else 1
        self.tex_shape = None if tex is None else tuple(tex.shape[:2])
        self._gpu = None
        for name, value in (("init_obj", obj), ("init_tex", tex)):     # read back by the script's change_all()
            if value is not None:
                setattr(self, name, value)

    def _padded(self, a, cols, what):
        a = np.asarray(a)
        if a.shape[0] > self.N:
            raise ValueError(f"StaticModel: the obj has {a.shape[0]} {what}, more than the capacity N = {self.N}")
        out = np.zeros((self.N, cols), np.float32)
        out[:a.shape[0]] = a
        return out

    def _init(self):
        dev = torch.device("cuda", torch.cuda.current_device())
        gpu = dict(verts=torch.zeros((self.N, 3), dtype=torch.float32, device=dev),
                   faces=torch.zeros((0, 3), dtype=torch.int32, device=dev), uvs=None, face_uvs=None, tex=None)
        obj = getattr(self, "init_obj", None)
        if obj is not None:
            if obj['vi'] is not None:
                gpu['verts'] = torch.from_numpy(self._padded(obj['vi'][:, :3], 3, "vertices")).to(dev)
            if obj['vt'] is not None:
                gpu['uvs'] = torch.from_numpy(self._padded(obj['vt'], 2, "uvs")).to(dev)
            if obj['vn'] is not None:
                self._padded(obj['vn'], 3, "normals")
            f = obj['f']
            if f is not None:
                f = np.asarray(f)
                if f.ndim != 3 or f.shape[1] != 3 or f.shape[2] != self.corner_fields:
                    raise ValueError(f"StaticModel: faces must be [F, 3, {self.corner_fields}] for this model, got {f.shape}")
                if f.shape[0] > self.N:
                    raise ValueError(f"StaticModel: the obj has {f.shape[0]} faces, more than the capacity N = {self.N}")
                gpu['faces'] = torch.from_numpy(np.ascontiguousarray(f[:, :, 0], np.int32)).to(dev)
                if gpu['uvs'] is not None:
                    # the reference reads uvs through corner field min(1, corner_fields - 1): the uv index, or the vertex index
                    # for bare `v` faces
                    col = min(1, self.corner_fields - 1)
                    gpu['face_uvs'] = torch.from_numpy(np.ascontiguousarray(f[:, :, col], np.int32)).to(dev)
        tex = getattr(self, "init_tex", None)
        if tex is not None:
            if tuple(tex.shape[:2]) != self.tex_shape or tex.shape[2:] != (3,):
                raise ValueError(f"StaticModel: texture {tex.shape} does not match the model's {self.tex_shape}")
            gpu['tex'] = torch.from_numpy(np.ascontiguousarray(tex.astype(np.float32) / 255)).to(dev)
        if gpu['uvs'] is None or gpu['faces'].shape[0] == 0:
            gpu['uvs'] = gpu['face_uvs'] = None
        self._gpu = gpu

    def render_inputs(self):
        """The device tensors of the last `_init()` (verts, faces, uvs, face_uvs, tex)."""
        if self._gpu is None:
            raise RuntimeError("StaticModel: render before _init()")
        return self._gpu

    def __getattr__(self, name):
        if name.startswith("__") or name in ("init_obj", "init_tex"):
            raise AttributeError(name)
        raise unsupported(f"StaticModel.{name}")
