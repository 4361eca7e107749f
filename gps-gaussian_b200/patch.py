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

`GPSG_RECTIFY=1`, read once by `install()`, also hooks `lib.human_loader` and rebinds two methods of its
`StereoHumanDataset` to the rectification kernels (gps_gaussian_b200.rectify, csrc/rectify.cu), with identical results:

    get_rectified_stereo_data -> rectify.rectify_stereo    (every main-process caller, the rectified_local/ cache included)
    get_test_item             -> rectify.stereo_item_cuda  (test_real_data.py: lmain/rmain img and mask arrive on the GPU)

Inside a DataLoader worker (forked, no CUDA) or without CUDA both call the reference's own method.  Unset or any other
value leaves `lib.human_loader` alone: it is then not even hooked.

`GPSG_FLOW_HEAD=1`, read once by `install()`, also hooks the disparity head of both training stages
(gps_gaussian_b200.flow_head, csrc/flow_head.cu):

    core.raft_stereo_human.FlowUpdateModule.upsample_flow -> fused convex upsampling (a class method, kept in _ORIG_METHODS)
    lib.loss.sequence_loss (and lib.network's copy)        -> flow_head.sequence_loss (one host synchronisation)

Inputs the kernels do not cover (CPU tensors, other dtypes or factors) reach the reference's own function.  The results
differ from the op chain's by fp32 re-association and by where fp16 rounding falls in the backward, which is why the
switch is opt-in.  Unset or any other value hooks neither.

`taichi_three` and its submodules always resolve to the stand-in in dropin/taichi_three (the dataset renderer on
csrc/mesh_render.cu).  `python prepare_data/render_data.py` puts prepare_data/ first on sys.path, where the reference's
own package, which cannot import without Taichi, would shadow anything on PYTHONPATH.
"""
import importlib.abc
import importlib.machinery
import logging
import os
import sys

_ORIG = {}            # (module name, attribute) -> original object
_ORIG_METHODS = {}    # (class, attribute) -> original function
_ANTIALIAS = False    # GPSG_ANTIALIAS=1 at install()
_RECTIFY = False      # GPSG_RECTIFY=1 at install()
_FLOW_HEAD = False    # GPSG_FLOW_HEAD=1 at install()


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


def _on_device():
    """The GPU route runs in the main process with CUDA; a DataLoader worker is forked and must not touch CUDA."""
    import torch
    return torch.utils.data.get_worker_info() is None and torch.cuda.is_available()


def _rectified_stereo_data(orig, mod):
    def get_rectified_stereo_data(self, main_view_data, ref_view_data):
        if not _on_device():
            return orig(self, main_view_data, ref_view_data)
        from gps_gaussian_b200 import rectify
        return rectify.rectify_stereo(main_view_data, ref_view_data, self.opt.src_res, pts2depth=mod.pts2depth)
    return get_rectified_stereo_data


def _test_item(orig, mod):
    """get_test_item with the rectified pair made on the GPU: load both views, then stereo_item_cuda, then the original
    intrinsics / extrinsics and the novel-view size, as the reference's method (lib/human_loader.py:390-419)."""
    def get_test_item(self, index, source_id):
        if not _on_device():
            return orig(self, index, source_id)
        import torch
        from gps_gaussian_b200 import rectify
        sample_name = self.sample_list[index % len(self.sample_list)]
        if self.use_processed_data:
            logging.error('test data loader not support processed data')
        views = [self.load_single_view(sample_name, sid, hr_img=False, require_mask=True, require_pts=False)
                 for sid in source_id[:2]]
        item = rectify.stereo_item_cuda(views[0], views[1], self.opt.src_res, sample_name, pts2depth=mod.pts2depth)
        for key, which in (('intr_ori', 2), ('extr_ori', 3)):
            item['lmain'][key] = torch.FloatTensor(views[0][which])
            item['rmain'][key] = torch.FloatTensor(views[1][which])
        size = self.opt.src_res * 2 if self.opt.use_hr_img else self.opt.src_res
        item['novel_view'] = {'height': torch.IntTensor([size]), 'width': torch.IntTensor([size])}
        return item
    return get_test_item


def _patch_loader(mod):
    cls = mod.StereoHumanDataset
    for attr, wrap in (("get_rectified_stereo_data", _rectified_stereo_data), ("get_test_item", _test_item)):
        key = (cls, attr)
        if key not in _ORIG_METHODS:
            _ORIG_METHODS[key] = cls.__dict__[attr]
        setattr(cls, attr, wrap(_ORIG_METHODS[key], mod))


def _patch_upsample(mod):
    from gps_gaussian_b200 import flow_head
    cls = mod.FlowUpdateModule
    key = (cls, "upsample_flow")
    if key not in _ORIG_METHODS:
        _ORIG_METHODS[key] = cls.__dict__["upsample_flow"]
    cls.upsample_flow = flow_head.make_upsample_flow(_ORIG_METHODS[key])


def _patch_loss(mod):
    from gps_gaussian_b200 import flow_head
    _set(mod, "sequence_loss", flow_head.sequence_loss)
    user = sys.modules.get("lib.network")                     # `from lib.loss import sequence_loss` copies the binding
    if user is not None and hasattr(user, "sequence_loss"):
        _set(user, "sequence_loss", flow_head.sequence_loss)


# Modules whose `from <module> import <attr>` made after install() copies the rebound object without _set seeing it;
# uninstall() puts the original back there too.
_COPIES = {("lib.loss", "sequence_loss"): ("lib.network",)}


def original(mod, attr):
    """The object `mod.attr` had before the patch rebound it (itself when it was never rebound)."""
    return _ORIG.get((mod.__name__, attr)) or getattr(mod, attr)


_TARGETS = {"core.corr": _patch_corr, "lib.GaussianRender": _patch_render}
_RECTIFY_TARGETS = {"lib.human_loader": _patch_loader}
_FLOW_HEAD_TARGETS = {"core.raft_stereo_human": _patch_upsample, "lib.loss": _patch_loss}


def _targets():
    return {**_TARGETS, **(_RECTIFY_TARGETS if _RECTIFY else {}), **(_FLOW_HEAD_TARGETS if _FLOW_HEAD else {})}


class _PatchingLoader(importlib.abc.Loader):
    def __init__(self, inner, hook):
        self._inner, self._hook = inner, hook

    def create_module(self, spec):
        return self._inner.create_module(spec)

    def exec_module(self, module):
        self._inner.exec_module(module)
        self._hook(module)


_STANDINS = ("taichi_three",)    # packages always taken from dropin/, whatever shadows them on sys.path
_DROPIN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "dropin")


def _standin_spec(name):
    top = name.split(".", 1)[0]
    if top not in _STANDINS:
        return None
    where = [_DROPIN] if name == top else [os.path.join(_DROPIN, *name.split(".")[:-1])]
    return importlib.machinery.PathFinder.find_spec(name, where)


class _Finder(importlib.abc.MetaPathFinder):
    def find_spec(self, name, path=None, target=None):
        spec = _standin_spec(name)
        if spec is not None:
            return spec
        hook = _targets().get(name)
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
    """Hook future imports and patch what is already imported. Idempotent.  Reads GPSG_ANTIALIAS, GPSG_RECTIFY and
    GPSG_FLOW_HEAD here, once."""
    global _ANTIALIAS, _RECTIFY, _FLOW_HEAD
    _ANTIALIAS = os.environ.get("GPSG_ANTIALIAS", "") == "1"
    _RECTIFY = os.environ.get("GPSG_RECTIFY", "") == "1"
    _FLOW_HEAD = os.environ.get("GPSG_FLOW_HEAD", "") == "1"
    if _FINDER not in sys.meta_path:
        sys.meta_path.insert(0, _FINDER)
    for name, hook in _targets().items():
        if name in sys.modules:
            hook(sys.modules[name])


def uninstall():
    if _FINDER in sys.meta_path:
        sys.meta_path.remove(_FINDER)
    for (modname, attr), orig in list(_ORIG.items()):
        mod = sys.modules.get(modname)
        if mod is not None and orig is not None:
            for user in filter(None, map(sys.modules.get, _COPIES.get((modname, attr), ()))):
                if getattr(user, attr, None) is getattr(mod, attr):
                    setattr(user, attr, orig)
            setattr(mod, attr, orig)
    _ORIG.clear()
    for (cls, attr), orig in list(_ORIG_METHODS.items()):
        setattr(cls, attr, orig)
    _ORIG_METHODS.clear()


def active():
    return _FINDER in sys.meta_path


def antialiasing():
    """Whether the installed patch renders with the screen-space filter (GPSG_ANTIALIAS=1 at install())."""
    return _ANTIALIAS


def rectify():
    """Whether the installed patch rectifies on the GPU (GPSG_RECTIFY=1 at install())."""
    return _RECTIFY


def flow_head():
    """Whether the installed patch runs the disparity head on the fused kernels (GPSG_FLOW_HEAD=1 at install())."""
    return _FLOW_HEAD
