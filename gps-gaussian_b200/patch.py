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

`GPSG_DECODE=1`, read once by `install()` and effective together with `GPSG_RECTIFY=1`, makes the rebound
`get_test_item` decode the two source JPEGs on the GPU (gps_gaussian_b200.jpeg, csrc/jpeg_decode.cu: Pillow's bytes) and
hand the device images to the rectification kernels without a host round trip.  The masks stay PNG on Pillow.  Unset or
any other value decodes with the reference's `read_img`, as before.

`GPSG_ENCODE=1`, read once by `install()`, also hooks `cv2` and rebinds `cv2.imwrite` to the GPU JPEG encoder
(gps_gaussian_b200.jpeg, csrc/jpeg_encode.cu: cv2's bytes), which covers every JPEG the entry scripts write.  A call goes
to the GPU when the extension is .jpg / .jpeg / .jpe (any case), the params are empty or only IMWRITE_JPEG_QUALITY (0..100)
and IMWRITE_JPEG_SAMPLING_FACTOR (4:4:4, 4:2:2, 4:2:0), the array is uint8 [H,W], [H,W,1] or [H,W,3] of at least
_MIN_NATIVE_PIXELS pixels (any strides), its directory exists, and it runs in the main process with CUDA.  Every other
call reaches cv2's own function with the same arguments.  Unset or any other value leaves `cv2` alone: it is then not
even hooked.

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
_DECODE = False       # GPSG_DECODE=1 at install()
_ENCODE = False       # GPSG_ENCODE=1 at install()


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


def _views_cuda(self, mod, sample_name, source_ids):
    """load_single_view(sample_name, sid, hr_img=False, require_mask=True, require_pts=False) of both views, with the
    two images decoded on the GPU in one call (lib/human_loader.py:190-211)."""
    import numpy as np
    from gps_gaussian_b200 import jpeg
    imgs = jpeg.read_img_cuda([self.img_path % (sample_name, sid) for sid in source_ids])
    return [(img, mod.read_img(self.mask_path % (sample_name, sid)), np.load(self.intr_path % (sample_name, sid)),
             np.load(self.extr_path % (sample_name, sid)), None) for img, sid in zip(imgs, source_ids)]


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
        if _DECODE:
            views = _views_cuda(self, mod, sample_name, source_id[:2])
        else:
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


_JPEG_EXTS = (".jpg", ".jpeg", ".jpe")
_JPEG_SAMPLING = {0x111111: "444", 0x211111: "422", 0x221111: "420"}   # cv2.IMWRITE_JPEG_SAMPLING_FACTOR_444/422/420
_IMWRITE_JPEG_QUALITY, _IMWRITE_JPEG_SAMPLING_FACTOR = 1, 7
# Below this many pixels cv2 on the host is faster than the upload, the launch chain and the download: on an H100 at 700 W,
# q95 4:2:0, the GPU route took 1.85 ms against cv2's 1.38 ms at 256^2 and 4.34 ms against 4.98 ms at 512^2 (DESIGN.md §5).
_MIN_NATIVE_PIXELS = 512 * 512


def _jpeg_route(args, kwargs):
    """(filename, array, quality, subsampling) when cv2.imwrite(*args, **kwargs) is encoded on the GPU, else None."""
    import numpy as np
    names = ("filename", "img", "params")
    if len(args) > 3 or any(k not in names[len(args):] for k in kwargs):
        return None
    bound = dict(zip(names, args), **kwargs)
    filename, img, params = bound.get("filename"), bound.get("img"), bound.get("params")
    if not isinstance(filename, str) or os.path.splitext(filename)[1].lower() not in _JPEG_EXTS:
        return None
    if type(img) is not np.ndarray or img.dtype != np.uint8:
        return None
    if not (img.ndim == 2 or (img.ndim == 3 and img.shape[2] in (1, 3))):
        return None
    H, W = img.shape[:2]
    if not (1 <= H <= 65500 and 1 <= W <= 65500) or H * W < _MIN_NATIVE_PIXELS:
        return None
    quality, subsampling = 95, "420"                   # cv2's defaults
    if params is not None:
        if not isinstance(params, (list, tuple)) or len(params) % 2:
            return None
        for key, val in zip(params[0::2], params[1::2]):
            if not all(isinstance(v, (int, np.integer)) and not isinstance(v, bool) for v in (key, val)):
                return None
            if key == _IMWRITE_JPEG_QUALITY and 0 <= val <= 100:
                quality = max(int(val), 1)             # quality 0 is libjpeg's 1
            elif key == _IMWRITE_JPEG_SAMPLING_FACTOR and int(val) in _JPEG_SAMPLING:
                subsampling = _JPEG_SAMPLING[int(val)]
            else:
                return None
    if not os.path.isdir(os.path.dirname(os.path.abspath(filename))) or not _in_main_process() or not _on_device():
        return None
    from gps_gaussian_b200 import jpeg
    if not jpeg.fits_one_call(H, W, 1 if img.ndim == 2 or img.shape[2] == 1 else 3, subsampling):
        return None                                    # too large for one launch chain: cv2 writes it
    return filename, img, quality, subsampling


def _in_main_process():
    """cv2.imwrite in a child process (a DataLoader worker, a multiprocessing.Pool of writers) stays on cv2: a forked
    child of a process that has used CUDA cannot use it again."""
    import multiprocessing
    return multiprocessing.parent_process() is None


def _make_imwrite(orig):
    def imwrite(*args, **kwargs):
        from gps_gaussian_b200 import jpeg
        route = _jpeg_route(args, kwargs)
        if route is not None:
            filename, img, quality, subsampling = route
            import torch
            try:
                data = jpeg.encode_host(img, quality, subsampling, order="bgr")
                with open(filename, "wb") as f:
                    f.write(data)
                return True
            except (OSError, torch.cuda.OutOfMemoryError):
                pass                                   # an unwritable path, or no device memory left: cv2 decides
        jpeg._ENC_COUNTS["fallback"] += 1
        return orig(*args, **kwargs)
    imwrite.__doc__ = orig.__doc__
    imwrite._gpsg_original = orig
    return imwrite


_CV2_MODULES = []     # module objects whose imwrite the patch rebound (see _patch_cv2)


def _patch_cv2(mod):
    """cv2.imwrite -> the GPU JPEG route.

    Imported after install(), cv2's package (cv2/__init__.py) imports its native extension under the same name "cv2",
    so this hook fires twice: first on the extension module, whose imwrite it wraps, then on the package, which by then
    has copied the wrapper from the extension.  Both module objects are kept in _CV2_MODULES and uninstall() restores
    imwrite on each of them, not only on whichever one sys.modules["cv2"] holds."""
    cur = getattr(mod, "imwrite", None)
    if cur is None:
        return
    if not hasattr(cur, "_gpsg_original"):
        _set(mod, "imwrite", _make_imwrite(cur))
    if not any(m is mod for m in _CV2_MODULES):
        _CV2_MODULES.append(mod)


# Modules whose `from <module> import <attr>` made after install() copies the rebound object without _set seeing it;
# uninstall() puts the original back there too.
_COPIES = {("lib.loss", "sequence_loss"): ("lib.network",)}


def original(mod, attr):
    """The object `mod.attr` had before the patch rebound it (itself when it was never rebound)."""
    return _ORIG.get((mod.__name__, attr)) or getattr(mod, attr)


_TARGETS = {"core.corr": _patch_corr, "lib.GaussianRender": _patch_render}
_RECTIFY_TARGETS = {"lib.human_loader": _patch_loader}
_FLOW_HEAD_TARGETS = {"core.raft_stereo_human": _patch_upsample, "lib.loss": _patch_loss}
_ENCODE_TARGETS = {"cv2": _patch_cv2}


def _targets():
    return {**_TARGETS, **(_RECTIFY_TARGETS if _RECTIFY else {}), **(_FLOW_HEAD_TARGETS if _FLOW_HEAD else {}),
            **(_ENCODE_TARGETS if _ENCODE else {})}


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
    """Hook future imports and patch what is already imported. Idempotent.  Reads GPSG_ANTIALIAS, GPSG_RECTIFY,
    GPSG_FLOW_HEAD, GPSG_DECODE and GPSG_ENCODE here, once."""
    global _ANTIALIAS, _RECTIFY, _FLOW_HEAD, _DECODE, _ENCODE
    _ANTIALIAS = os.environ.get("GPSG_ANTIALIAS", "") == "1"
    _RECTIFY = os.environ.get("GPSG_RECTIFY", "") == "1"
    _FLOW_HEAD = os.environ.get("GPSG_FLOW_HEAD", "") == "1"
    _DECODE = os.environ.get("GPSG_DECODE", "") == "1"
    _ENCODE = os.environ.get("GPSG_ENCODE", "") == "1"
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
    for mod in _CV2_MODULES:
        wrapper = getattr(mod, "imwrite", None)
        if hasattr(wrapper, "_gpsg_original"):
            mod.imwrite = wrapper._gpsg_original
    _CV2_MODULES.clear()


def active():
    return _FINDER in sys.meta_path


def antialiasing():
    """Whether the installed patch renders with the screen-space filter (GPSG_ANTIALIAS=1 at install())."""
    return _ANTIALIAS


def rectify():
    """Whether the installed patch rectifies on the GPU (GPSG_RECTIFY=1 at install())."""
    return _RECTIFY


def decode():
    """Whether the rebound get_test_item decodes the source JPEGs on the GPU (GPSG_DECODE=1 at install())."""
    return _DECODE


def encode():
    """Whether cv2.imwrite writes JPEGs through the GPU encoder (GPSG_ENCODE=1 at install())."""
    return _ENCODE


def flow_head():
    """Whether the installed patch runs the disparity head on the fused kernels (GPSG_FLOW_HEAD=1 at install())."""
    return _FLOW_HEAD
