"""Directional lights of the stand-in (reference prepare_data/taichi_three/light.py)."""
import math

import numpy as np

from .common import AutoInit, unsupported


class Light(AutoInit):
    """A directional light shining along `dir` (default +z) with an rgb `color` (default white).  The renderer uses the
    unit vector towards the light, `towards` = -dir / |dir|."""

    def __init__(self, dir=None, color=None):
        shine = list(dir) if dir else [0, 0, 1]
        length = math.sqrt(sum(c * c for c in shine))
        self.towards = [-(c / length) for c in shine]
        self.colour = list(color) if color else [1, 1, 1]

    def _init(self):
        pass

    def set(self, *args, **kwargs):
        raise unsupported("Light.set")


class Lights(AutoInit):
    """The lights of a scene.  `init_data()` takes an fp32 snapshot of their directions and colours, which every later
    render uses (the scene calls it on its first render)."""

    def __init__(self, light_list):
        self.members = list(light_list)
        self.light_dirs = np.zeros((len(self.members), 3), np.float32)
        self.light_colors = np.ones((len(self.members), 3), np.float32)

    def init_data(self):
        if self.members:
            self.light_dirs[:] = [light.towards for light in self.members]
            self.light_colors[:] = [light.colour for light in self.members]

    def _init(self):
        self.init_data()
