"""Gaussian cache across novel views: the serving loop of reference test_view_interp.py:34-47, restructured.

The reference re-runs the whole network and `pts2render` for every novel view of a pair, although the pixel-aligned
Gaussians (data[view]['xyz', 'img', 'rot_maps', 'scale_maps', 'opacity_maps', 'pts_valid']) do not depend on the
novel camera.  `NovelViewRenderer` keeps them resident, computes every novel camera of the sweep in one host pass
(`novel_calib.calib_from_data`) and enqueues one sync-free forward per (sample, ratio) round-robin over a few CUDA
streams: no per-view gather, no host sync, no H2D camera copies inside the loop.  Two cache layouts:

  * mode="compact" (default): the valid pixels of both views are gathered ONCE per pair into the [P,k] tensors `render`
    takes (the reference's own gather, lib/GaussianRender.py:14-33 -- one sync per pair instead of ten per view); every
    view is then a `gpsg_rasterize_forward_planned` over ~P Gaussians (28 MB read at C2);
  * mode="maps": zero-copy -- every view is a `gpsg_rasterize_forward_maps_planned` over the 2*S^2 candidates in place
    (120 MB read at C2, but no construction cost at all: right when only one or two views are rendered per pair).

Images equal `get_novel_calib(ratio)` + `pts2render` per ratio bit for bit in both modes.  With aux=True the sweep also
carries the expected depth and the alpha matte of every view (aux mode of the planned forwards), equal to
`pts2render_aux` per ratio bit for bit.  With antialiasing=True every view is rendered with the opacity-compensated
screen-space filter (GPSG_FWD_ANTIALIAS), equal to `pts2render_ex(..., antialiasing=True)` per ratio bit for bit.
"""
import numpy as np
import torch

from . import _lib
from .GaussianRender import _RasterizeMaps, _RasterizeMapsAux, novel_settings
from .novel_calib import calib_from_data
from .planned import PlannedRasterizer

_VIEWS = ('lmain', 'rmain')
_MAX_TILE_SORT = 4096          # kMaxTileSort (csrc/gpsg_internal.cuh): longest tile list the in-CTA sort takes


class NovelViewRenderer:
    """cache = NovelViewRenderer(data, opt, bg_color); imgs = cache.render(ratios)   # [B, len(ratios), 3, H, W]

    `data` is the dict the network returns (reference lib/network.py:41-88) -- the same one `pts2render` takes."""

    def __init__(self, data, opt, bg_color, intr_key='intr', extr_key='extr', streams=4, capacity_pairs=None,
                 mode='compact', antialiasing=False):
        if mode not in ('compact', 'maps'):
            raise ValueError("mode must be 'compact' or 'maps'")
        self.mode = mode
        self.antialiasing = bool(antialiasing)
        self.data, self.opt, self.bg = data, opt, [float(v) for v in bg_color]
        self.keys = (intr_key, extr_key)
        x = data['lmain']['xyz']
        self.dev, self.bs = x.device, int(x.shape[0])
        f = lambda t: t.detach().to(torch.float32).contiguous()
        self.maps = []
        for i in range(self.bs):
            per = dict(valid=[], xyz=[], img=[], rot=[], scale=[], opacity=[])
            for v in _VIEWS:
                d = data[v]
                per['valid'].append(d['pts_valid'][i].reshape(-1).contiguous().view(torch.uint8))
                per['xyz'].append(f(d['xyz'][i]))
                per['img'].append(f(d['img'][i]))
                per['rot'].append(f(d['rot_maps'][i]))
                per['scale'].append(f(d['scale_maps'][i]))
                per['opacity'].append(f(d['opacity_maps'][i]))
            self.maps.append(per)
        self.S2 = int(self.maps[0]['valid'][0].numel())
        self.flat = []
        if mode == 'compact':
            for per in self.maps:
                sel = [v.view(torch.bool) for v in per['valid']]
                chw = lambda key, c: torch.cat([t.view(c, -1).t()[m] for t, m in zip(per[key], sel)], 0).contiguous()
                self.flat.append(dict(xyz=torch.cat([t.view(-1, 3)[m] for t, m in zip(per['xyz'], sel)], 0).contiguous(),
                                      rgb=chw('img', 3) * 0.5 + 0.5, rot=chw('rot', 4), scale=chw('scale', 3),
                                      opacity=chw('opacity', 1)))
            pmax = max(1, max(int(f['xyz'].shape[0]) for f in self.flat))
        nv = data['novel_view']
        self.H, self.W = int(nv['height'][0]), int(nv['width'][0])
        self.n_streams = max(1, int(streams))
        # about 2.6 tiles per valid Gaussian on the C2 workload; a quarter of the candidates valid -> ~0.65*2*S2 pairs;
        # 2*S2 leaves headroom and the overflow path grows it.
        cap = int(capacity_pairs) if capacity_pairs else max(2 * self.S2, 1 << 16)
        self.rast = [PlannedRasterizer(pmax if mode == 'compact' else 2 * self.S2, self.H, self.W, cap, self.dev)
                     for _ in range(self.n_streams)]
        self.streams = [torch.cuda.Stream(self.dev) for _ in range(self.n_streams)]

    def _enqueue(self, rast, settings, b, out, status_host=None, depth=None, alpha=None):
        """depth / alpha ([H,W] each, or None): aux outputs of the view."""
        if self.mode == 'compact':
            f = self.flat[b]
            if f['xyz'].shape[0] == 0:                                  # empty mask: background only (reference P == 0)
                out.copy_(torch.tensor(self.bg, device=self.dev).view(3, 1, 1).expand_as(out))
                if depth is not None:
                    depth.zero_()
                    alpha.zero_()
                return
            rast.forward(settings, f['xyz'], f['rgb'], f['opacity'], f['scale'], f['rot'], out=out, status_host=status_host,
                         depth=depth, alpha=alpha, antialiasing=self.antialiasing)
        else:
            m = self.maps[b]
            rast.forward_maps(settings, m['valid'], m['xyz'], m['img'], m['rot'], m['scale'], m['opacity'], out=out,
                              status_host=status_host, depth=depth, alpha=alpha, antialiasing=self.antialiasing)

    def _settings(self, cal, b, r):
        cam = np.concatenate([cal[k][b, r].reshape(-1) for k in ('world_view_transform', 'full_proj_transform',
                                                                  'camera_center')]).tolist()
        return novel_settings(self.H, self.W, cal['FovX'][b, r], cal['FovY'][b, r], self.bg, cam)

    def _render_exact(self, settings, b, out, depth=None, alpha=None):
        """Exact entry point (one host sync, radix fallback for over-long tile lists) for one view of sample b; depth /
        alpha ([H,W] or None): aux outputs."""
        if self.mode == 'compact':
            f = self.flat[b]
            radii = torch.empty((f['xyz'].shape[0],), dtype=torch.int32, device=self.dev)
            _lib.rasterize_forward(settings, out, radii, f['xyz'], f['opacity'], colors_precomp=f['rgb'],
                                   scales=f['scale'], rotations=f['rot'], out_depth=depth, out_alpha=alpha,
                                   antialiasing=self.antialiasing)
        else:
            m = self.maps[b]
            args = []
            for v in range(2):
                args += [m['valid'][v], m['xyz'][v], m['img'][v], m['rot'][v], m['scale'][v], m['opacity'][v]]
            flags = _lib.forward_flags(self.antialiasing)
            with torch.no_grad():
                if depth is None:
                    out.copy_(_RasterizeMaps.apply([settings], flags, *args)[0])
                else:
                    i, d, a = _RasterizeMapsAux.apply([settings], flags, *args)
                    out.copy_(i[0]); depth.copy_(d[0, 0]); alpha.copy_(a[0, 0])

    def render(self, ratios, out=None, check=True, aux=False):
        """Images [B, len(ratios), 3, H, W].  aux=True: returns (images, depth, alpha), depth and alpha
        [B, len(ratios), 1, H, W] (expected view-space depth and alpha matte of every view); self.last_aux holds them
        too, for check=False."""
        ratios = [float(r) for r in ratios]
        cal = calib_from_data(self.data, self.opt, ratios, *self.keys)
        if out is None:
            out = torch.empty((self.bs, len(ratios), 3, self.H, self.W), dtype=torch.float32, device=self.dev)
        depth = alpha = None
        if aux:
            new = lambda: torch.empty((self.bs, len(ratios), 1, self.H, self.W), dtype=torch.float32, device=self.dev)
            depth, alpha = new(), new()
        self.last_aux = (depth, alpha)
        maps = lambda b, r: (depth[b, r, 0], alpha[b, r, 0]) if aux else (None, None)
        result = lambda: (out, depth, alpha) if aux else out
        cur = torch.cuda.current_stream(self.dev)
        for s in self.streams:
            s.wait_stream(cur)
        jobs = [(b, r) for b in range(self.bs) for r in range(len(ratios))]
        status = torch.zeros((len(jobs), 4), dtype=torch.int32).pin_memory()       # one deferred status slot per job
        for k, (b, r) in enumerate(jobs):
            j = k % self.n_streams
            with torch.cuda.stream(self.streams[j]):
                self._enqueue(self.rast[j], self._settings(cal, b, r), b, out[b, r], status[k], *maps(b, r))
        for s in self.streams:
            cur.wait_stream(s)
        self.last_status = status
        if not check:
            return result()                                             # fully asynchronous; caller checks last_status
        torch.cuda.current_stream(self.dev).synchronize()
        # status[k] = (num_rendered, longest tile list, overflow flag) of job k.  Two different overflows (ADVICE r1):
        #  * more pairs than the binning buffer holds -> size the buffer from the reported count and render again;
        #  * a tile list longer than the in-CTA sort (kMaxTileSort = 4096): no buffer size helps -- that view goes through
        #    the exact entry point, whose global radix fallback handles any list length.
        for k, (b, r) in enumerate(jobs):
            n_pairs, max_tile, overflow = (int(v) for v in status[k, :3].tolist())
            if not overflow:
                continue
            settings = self._settings(cal, b, r)
            if max_tile > _MAX_TILE_SORT:
                self._render_exact(settings, b, out[b, r], *maps(b, r))
                continue
            rast = self.rast[0]
            rast.grow(needed_pairs=n_pairs)
            rast.status_host.zero_()
            self._enqueue(rast, settings, b, out[b, r], None, *maps(b, r))
            torch.cuda.synchronize(self.dev)
            if not rast.ok():
                st = rast.status()
                if st["max_tile"] > _MAX_TILE_SORT:
                    self._render_exact(settings, b, out[b, r], *maps(b, r))
                else:
                    raise _lib.GpsgError(f"novel view render: {st['num_rendered']} pairs do not fit capacity {rast.capacity}")
        torch.cuda.synchronize(self.dev)
        return result()


def render_novel_views(data, opt, ratios, bg_color, intr_key='intr', extr_key='extr', streams=4, mode='compact', aux=False,
                       antialiasing=False):
    """data['novel_view']['img_pred_sweep'] = [B, len(ratios), 3, H, W]; returns data.  aux=True also sets
    ['depth_pred_sweep'] and ['alpha_pred_sweep'], [B, len(ratios), 1, H, W].  antialiasing: see NovelViewRenderer."""
    nv = data['novel_view']
    res = NovelViewRenderer(data, opt, bg_color, intr_key, extr_key, streams, mode=mode,
                            antialiasing=antialiasing).render(ratios, aux=aux)
    if aux:
        nv['img_pred_sweep'], nv['depth_pred_sweep'], nv['alpha_pred_sweep'] = res
    else:
        nv['img_pred_sweep'] = res
    return data
