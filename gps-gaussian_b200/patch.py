"""Opt-in route for the H100 fast paths on the UNMODIFIED reference scripts (VERDICT r1 "missing" item 3).

With only `dropin/` on PYTHONPATH the reference's own Python still runs around the two drop-in extensions:
core/corr.py:53-61 builds the volume with einsum -> cuBLAS + `/sqrt(D)` + three `avg_pool2d` and looks it up with four
sampler launches + `cat` (:44-51); lib/GaussianRender.py:14-33 does ten boolean-mask gathers per sample before `render`.
`GPSG_PATCH=1` (read by `dropin/sitecustomize.py`, which Python imports at start-up when `dropin/` is on PYTHONPATH)
installs a post-import hook that, right after the reference executes those two modules, rebinds

    core.corr.CorrBlockFast1D, core.corr.CorrSampler   -> gps_gaussian_b200.corr   (fused wgmma build, fused lookup)
    lib.GaussianRender.pts2render                      -> gps_gaussian_b200.GaussianRender.pts2render (fused map ingest)

so `from core.corr import CorrBlockFast1D` (core/raft_stereo_human.py:6) and `from lib.GaussianRender import pts2render`
(train_stage2.py:15, test_view_interp.py:15) pick ours up.  Same names, signatures and results (tests/test_c3_gpu.py runs
the stage-2 step both ways).  `install()` / `uninstall()` do the same for modules that are already imported.

`GPSG_ANTIALIAS=1`, read once by `install()`, makes the rebound `pts2render` render with the opacity-compensated
screen-space filter (`pts2render_ex(..., antialiasing=True)`, forward and backward), so the unmodified training and
novel-view scripts train and render anti-aliased; unset or any other value keeps the reference's image.
"""
import importlib.abc
import importlib.machinery
import os
import sys

_ORIG = {}            # (module name, attribute) -> original object
_ANTIALIAS = False    # GPSG_ANTIALIAS=1 at install()


def _set(mod, attr, new):
    key = (mod.__name__, attr)
    if key not in _ORIG:
        _ORIG[key] = getattr(mod, attr, None)
    setattr(mod, attr, new)


def _patch_corr(mod):
    from gps_gaussian_b200 import corr as ours
    _set(mod, "CorrBlockFast1D", ours.CorrBlockFast1D)
    _set(mod, "CorrSampler", ours.CorrSampler)
    user = sys.modules.get("core.raft_stereo_human")          # `from core.corr import ...` copies the binding
    if user is not None and hasattr(user, "CorrBlockFast1D"):
        _set(user, "CorrBlockFast1D", ours.CorrBlockFast1D)


def _pts2render_antialiased(data, bg_color):
    """`pts2render` with the opacity-compensated screen-space filter (GPSG_ANTIALIAS=1)."""
    from gps_gaussian_b200 import GaussianRender as ours
    return ours.pts2render_ex(data, bg_color, antialiasing=True)


def _patch_render(mod):
    from gps_gaussian_b200 import GaussianRender as ours
    _set(mod, "pts2render", _pts2render_antialiased if _ANTIALIAS else ours.pts2render)


_TARGETS = {"core.corr": _patch_corr, "lib.GaussianRender": _patch_render}


class _PatchingLoader(importlib.abc.Loader):
    def __init__(self, inner, hook):
        self._inner, self._hook = inner, hook

    def create_module(self, spec):
        return self._inner.create_module(spec)

    def exec_module(self, module):
        self._inner.exec_module(module)
        self._hook(module)


class _Finder(importlib.abc.MetaPathFinder):
    def find_spec(self, name, path=None, target=None):
        hook = _TARGETS.get(name)
        if hook is None:
            return None
        for finder in sys.meta_path:
            if finder is self or not hasattr(finder, "find_spec"):
                continue
            spec = finder.find_spec(name, path, target)
            if spec is not None and spec.loader is not None:
                spec.loader = _PatchingLoader(spec.loader, hook)
                return spec
        return None


_FINDER = _Finder()


def install():
    """Hook future imports and patch what is already imported. Idempotent.  Reads GPSG_ANTIALIAS here, once."""
    global _ANTIALIAS
    _ANTIALIAS = os.environ.get("GPSG_ANTIALIAS", "") == "1"
    if _FINDER not in sys.meta_path:
        sys.meta_path.insert(0, _FINDER)
    for name, hook in _TARGETS.items():
        if name in sys.modules:
            hook(sys.modules[name])


def uninstall():
    if _FINDER in sys.meta_path:
        sys.meta_path.remove(_FINDER)
    for (modname, attr), orig in list(_ORIG.items()):
        mod = sys.modules.get(modname)
        if mod is not None and orig is not None:
            setattr(mod, attr, orig)
    _ORIG.clear()


def active():
    return _FINDER in sys.meta_path


def antialiasing():
    """Whether the installed patch renders with the screen-space filter (GPSG_ANTIALIAS=1 at install())."""
    return _ANTIALIAS
