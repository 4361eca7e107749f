"""Host-buffer front end: render novel views whose Gaussians live in (pinned) HOST memory.

The reference moves a sample to the GPU with blocking `.cuda()` copies and then renders (train_stage2.py:155-157,
test_view_interp.py:55-59).  On an H100 the render itself takes ~0.3 ms while the 28 MB of per-view inputs take
~0.5 ms over PCIe, so the copies must overlap the compute: three CUDA streams (H2D, compute, D2H) and
double-buffered device staging slots; the render is the unchanged reference-signature call
`gaussian_renderer.render(data, idx, pts_xyz, pts_rgb, rotations, scales, opacity, bg_color)`.
"""
import torch

from .gaussian_renderer import render

_KEYS = ("means3D", "colors", "rots", "scales", "opacity")
_COLS = {"means3D": 3, "colors": 3, "rots": 4, "scales": 3, "opacity": 1}
_ROW = sum(_COLS.values())      # 14 floats per Gaussian


def _views(flat, n):
    """The five [n,k] arrays inside one packed fp32 buffer laid out [means3D | colors | rots | scales | opacity]."""
    out, off = {}, 0
    for k in _KEYS:
        c = _COLS[k]
        out[k] = flat[off:off + n * c].view(n, c)
        off += n * c
    return out


def pack_host(arrays):
    """Pack a dict of five [n,k] fp32 arrays (numpy or torch) into ONE pinned host buffer (one large DMA per view
    instead of five small ones).  Returns (packed pinned tensor of 14*n floats, n)."""
    n = int(arrays["means3D"].shape[0])
    flat = torch.empty(n * _ROW, dtype=torch.float32).pin_memory()
    for k, v in _views(flat, n).items():
        v.copy_(torch.as_tensor(arrays[k], dtype=torch.float32).reshape(n, _COLS[k]))
    return flat, n


class HostRenderPipeline:
    def __init__(self, device, max_points, height, width, slots=2):
        if slots < 2:
            # run() uploads item k+1 while item k renders: with one slot that upload would overwrite the inputs of a
            # render that has not started yet
            raise ValueError("HostRenderPipeline needs at least 2 staging slots")
        self.dev = torch.device(device)
        self.s_h2d, self.s_cmp, self.s_d2h = (torch.cuda.Stream(self.dev) for _ in range(3))
        self.stage = [torch.empty(max_points * _ROW, dtype=torch.float32, device=self.dev) for _ in range(slots)]
        self.ev_ready = [torch.cuda.Event() for _ in range(slots)]     # H2D of slot finished
        self.ev_free = [torch.cuda.Event() for _ in range(slots)]      # compute finished reading slot
        self.ev_img = [torch.cuda.Event() for _ in range(slots)]       # image of slot rendered
        self.ev_out = [torch.cuda.Event() for _ in range(slots)]       # image of slot copied to host
        self.img = [None] * slots
        self.used = [False] * slots
        self.slots = slots

    def _upload(self, slot, host):
        """host: (packed pinned tensor, n) from pack_host, or a dict of five pinned [n,k] tensors."""
        with torch.cuda.stream(self.s_h2d):
            if self.used[slot]:
                self.s_h2d.wait_event(self.ev_free[slot])
            if isinstance(host, tuple):
                flat, n = host
                self.stage[slot][:n * _ROW].copy_(flat, non_blocking=True)        # one DMA
            else:
                n = int(host["means3D"].shape[0])
                for k, v in _views(self.stage[slot], n).items():
                    v.copy_(host[k], non_blocking=True)
            self.ev_ready[slot].record(self.s_h2d)
        return n

    def run(self, items, out_host, bg_color=(0.0, 0.0, 0.0)):
        """items: list of (host inputs -- `pack_host(...)` result or a dict of pinned fp32 tensors --, reference-style `data` dict, idx);
        out_host: list of pinned [3,H,W] tensors (one per item).  Returns when everything has landed."""
        if not items:
            return
        counts = {0: self._upload(0, items[0][0])}
        with torch.no_grad():
            for k, (host, data, idx) in enumerate(items):
                slot = k % self.slots
                if k + 1 < len(items):
                    counts[(k + 1) % self.slots] = self._upload((k + 1) % self.slots, items[k + 1][0])
                with torch.cuda.stream(self.s_cmp):
                    self.s_cmp.wait_event(self.ev_ready[slot])
                    if self.img[slot] is not None:
                        self.s_cmp.wait_event(self.ev_out[slot])          # previous image of this slot has left
                    n = counts[slot]
                    d = _views(self.stage[slot], n)
                    img = render(data, idx, d["means3D"], d["colors"], d["rots"], d["scales"], d["opacity"], list(bg_color))
                    self.img[slot] = img
                    self.ev_free[slot].record(self.s_cmp)
                    self.ev_img[slot].record(self.s_cmp)
                    self.used[slot] = True
                with torch.cuda.stream(self.s_d2h):
                    self.s_d2h.wait_event(self.ev_img[slot])
                    out_host[k].copy_(img, non_blocking=True)
                    self.ev_out[slot].record(self.s_d2h)
        self.s_d2h.synchronize()
        self.s_cmp.synchronize()
