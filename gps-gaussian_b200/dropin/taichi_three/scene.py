"""The scene of the stand-in (reference prepare_data/taichi_three/scene.py): models, cameras and lights, and `render()`."""
from .common import AutoInit, repo_on_path, unsupported


class Scene(AutoInit):
    """`render()` first initialises the scene, once: `init()` of every camera, then of every model, then the lights'
    snapshot.  Each render then clears and draws every camera; all cameras go through one gps_gaussian_b200.mesh_render
    call, i.e. one launch chain on the current stream.  One model per scene (the script's case); more raise
    NotImplementedError."""

    def __init__(self):
        self.models, self.cameras, self.lights = [], [], None

    def _attach(self, item, where):
        item.scene = self
        where.append(item)

    def add_model(self, model):
        self._attach(model, self.models)

    def add_camera(self, camera):
        self._attach(camera, self.cameras)

    def add_lights(self, lights):
        """Replaces the scene's lights (a `Lights`)."""
        self.lights = lights
        lights.scene = self

    def _init(self):
        for item in [*self.cameras, *self.models]:
            item.init()
        if self.lights is not None:
            self.lights.init_data()

    def render(self):
        """Clear every camera's img / zbuf / mask and draw the model into them (outputs stay on the GPU until read)."""
        self.init()
        if not self.cameras:
            return
        if len(self.models) > 1:
            raise unsupported("a scene with more than one model")
        import numpy as np
        import torch
        repo_on_path()
        from gps_gaussian_b200 import mesh_render
        views = [c.render_camera() for c in self.cameras]
        if self.models:
            m = self.models[0].render_inputs()
            mesh = (m['verts'], m['faces'], m['uvs'], m['face_uvs'], m['tex'])
        else:
            mesh = (torch.zeros((0, 3), dtype=torch.float32, device="cuda"),
                    torch.zeros((0, 3), dtype=torch.int32, device="cuda"), None, None, None)
        verts, faces, uvs, face_uvs, tex = mesh
        no_light = np.zeros((0, 3), np.float32)
        dirs = no_light if self.lights is None else self.lights.light_dirs
        cols = no_light if self.lights is None else self.lights.light_colors
        step = mesh_render.MAX_CAMERAS
        for first in range(0, len(views), step):
            outs = mesh_render.render(verts, faces, views[first:first + step], dirs, cols, uvs, face_uvs, tex)
            for camera, (img, zbuf, mask) in zip(self.cameras[first:], outs):
                camera.img._set(img)
                camera.zbuf._set(zbuf)
                camera.mask._set(mask)

    def __getattr__(self, name):
        if name.startswith("__"):
            raise AttributeError(name)
        raise unsupported(f"Scene.{name}")
