"""Minimal stand-in for the `taichi` package, so that the UNMODIFIED reference `lib/TaichiRender.py` (imported by
train_stage1.py:16) imports and runs in an environment without taichi.  It provides only the surface that module touches
at import and construction time (`init`, `cuda`, `i32`, `data_oriented`, `Vector.field`, `types.ndarray`, `kernel`), and it
runs exactly one kernel: `TaichiRenderBatch.render_respective_color`, the stage-1 preview's z-buffer point splat, on
gps_gaussian_b200.point_splat (csrc/point_splat.cu).  That kernel is recognised by its qualified name and by a digest of
its source; any other kernel, or an edited one, raises NotImplementedError instead of running something else.

Results are the serial reading of the reference kernel (points in index order), which the reference's own Taichi kernel
only approximates: its colour write races with its atomic_max (DESIGN.md section 2).
"""
import hashlib
import inspect
import os
import sys

import torch

_REPO = os.path.dirname(os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))

cuda = "cuda"
cpu = "cpu"
i32 = "i32"
f32 = "f32"


def init(arch=None, **kwargs):
    """No runtime to start: the one supported kernel runs on the CUDA library."""
    return None


def data_oriented(cls):
    return cls


class _Field:
    def __init__(self, n, dtype, shape):
        self.n, self.dtype = n, dtype
        self.shape = tuple(shape) if isinstance(shape, (tuple, list)) else (shape,)


class Vector:
    @staticmethod
    def field(n, dtype, shape, **kwargs):
        """Records the shape only: the stand-in's kernel uses a field as its loop domain, never its storage."""
        return _Field(n, dtype, shape)


class types:
    @staticmethod
    def ndarray(*args, **kwargs):
        return "ndarray"


def kernel_digest(fn):
    """SHA-256 of a kernel's source with every run of whitespace collapsed to one space (None without a source file)."""
    try:
        src = inspect.getsource(fn)
    except (OSError, TypeError):
        return None
    return hashlib.sha256(" ".join(src.split()).encode()).hexdigest()


# `TaichiRenderBatch.render_respective_color` of the reference (lib/TaichiRender.py:13-24 at commit 0024776), decorator included
_SPLAT_QUALNAME = "TaichiRenderBatch.render_respective_color"
_SPLAT_DIGEST = "dc28aad16f0f451cf8e5d54f0a0eacb0fa8ddcc0958a509a162e1ca1f61c1028"


def _render_respective_color(self, pts, pts_mask, render_depth, render_color):
    for name, t in (("pts", pts), ("pts_mask", pts_mask), ("render_depth", render_depth), ("render_color", render_color)):
        if not torch.is_tensor(t) or not t.is_cuda or t.dtype != torch.float32:
            raise TypeError(f"taichi stand-in: {name} must be a CUDA float32 torch tensor (got {type(t).__name__} "
                            f"{getattr(t, 'dtype', '')} on {getattr(t, 'device', None)}); the stand-in runs this kernel on "
                            "the CUDA library only")
    if _REPO not in sys.path:
        sys.path.insert(0, _REPO)
    from gps_gaussian_b200.point_splat import point_splat
    B, N = self.coord.shape
    point_splat(pts, pts_mask, render_depth, render_color, B=B, N=N, res=self.res)


def kernel(fn):
    """Binds as a method like a Taichi kernel.  When called, runs the stage-1 splat if `fn` is the reference's kernel."""
    known = []

    def wrapper(*args, **kwargs):
        if not known:
            known.append(fn.__qualname__ == _SPLAT_QUALNAME and kernel_digest(fn) == _SPLAT_DIGEST)
        if not known[0]:
            raise NotImplementedError(
                f"taichi stand-in (gps-gaussian_b200/dropin/taichi): kernel {fn.__qualname__} is not supported; the stand-in "
                f"runs only the reference's unmodified {_SPLAT_QUALNAME} (its source digest differs or the name does not match)")
        bound = inspect.signature(fn).bind(*args, **kwargs)
        return _render_respective_color(*bound.args)

    wrapper.__name__, wrapper.__qualname__, wrapper.__doc__ = fn.__name__, fn.__qualname__, fn.__doc__
    wrapper.__wrapped__ = fn
    return wrapper
