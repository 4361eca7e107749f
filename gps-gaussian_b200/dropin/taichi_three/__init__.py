"""Stand-in for the reference's `prepare_data/taichi_three` (a Taichi software triangle rasterizer), so that the UNMODIFIED
`prepare_data/render_data.py` renders its training set here: faces are drawn by gps_gaussian_b200.mesh_render
(csrc/mesh_render.cu) instead of Taichi kernels.

It provides exactly the surface that script touches: `Scene`, `StaticModel`, `Camera`, `Light`, `Lights`, `readobj` and the
`taichi_three.transform` module (rotationX/Y/Z, with `math` and `ti` re-exported because the script takes `math.radians`
and `ti.init` from its star import).  Anything else of the reference's API raises NotImplementedError.  The results are the
serial reading of the reference's `render_triangle` (faces in index order), which its own kernel only approximates: its
colour write races with its atomic_max (DESIGN.md section 2).  Nothing here draws from `np.random`, so the script's
random sequence is the reference's.
"""
from .common import AutoInit, unsupported
from .light import Light, Lights
from .loader import readobj
from .model import StaticModel
from .scene import Scene
from .transform import Camera, rotationX, rotationY, rotationZ

__all__ = ["AutoInit", "Camera", "Light", "Lights", "Scene", "StaticModel", "readobj", "rotationX", "rotationY",
           "rotationZ"]


def __getattr__(name):
    if name.startswith("__"):
        raise AttributeError(name)
    raise unsupported(f"taichi_three.{name}")
