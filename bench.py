#!/usr/bin/env python
"""bench.py -- novel-views/sec of the H100 splat rasterizer on BASELINE config C2
(1024x1024, ~500k pixel-aligned Gaussians, fixed novel camera), plus the roofline of the dominant
kernel, the CPU baseline and the end-to-end (host-buffer) number.

    python bench.py [--gpus N] [--steps K] [--warmup W] [--views V] [--impl reference] [--dump-outputs DIR]

A "step" = R passes of the hot path over one batch of V independent synthetic view-pairs per GPU (seeds 1314+k, the C4
sharding unit); R = ceil(2000 / steps) so that the timed region is >= ~2.5 s of GPU work whatever --steps is (a burst of a
few ms overstates an issue-bound kernel's sustained clock; VERDICT r1 weak #10) and the NVML clock sampler sees > 100
samples under load.  N>1 is launched by torchrun (one rank per GPU); view-pairs are sharded across ranks, no data-path
collective (inference), `scaling: weak`.  `--train-c5` instead times the reference's stage-2 training step data-parallel
(2 pairs per GPU, one flat NCCL all-reduce of the gradients per step).

--impl reference: the reference has no runnable implementation of this path here (its rasterizer is the
absent third-party CUDA extension; lib/TaichiRender.py needs taichi + CUDA), so that arm times the CPU
oracle PORT of the same algorithm on the host cores (the one other place bench.py may execute oracle/).

--dump-outputs DIR: after the timed steps, rank 0 writes what the timed path returned in its last step as float32 .npy
files (see dump_outputs), so that two builds can be compared output for output on the same seeded inputs.
"""
import argparse
import json
import os
import sys
import threading
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

_CPU_THREADS = None
METRIC = "novel_views_per_sec_1024sq_500kgauss"
UNIT = "views/s"
RES = 1024


def _peaks():
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(p):
        try:
            return float(json.load(open(p))["hbm_gbs"]), "measured (MEASURED_PEAKS.json)"
        except Exception:
            pass
    return 3350.0, "fallback (H100 SXM data sheet, HBM3)"


class ClockSampler:
    """SM clock + throttle reasons sampled DURING the timed region (NVML; the fields nvidia-smi reports as clocks.sm,
    clocks.max.sm, clocks_event_reasons.*)."""

    def __init__(self, gpu_index, period_s=0.01):
        self.idx, self.period = gpu_index, period_s
        self.sm, self.reasons, self.power = [], set(), []
        self.stop_flag = threading.Event()
        self.thread = None
        self.max_mhz = None
        self.err = None

    def start(self):
        try:
            import pynvml
            pynvml.nvmlInit()
            vis = os.environ.get("CUDA_VISIBLE_DEVICES")
            phys = int(vis.split(",")[self.idx]) if vis and vis.split(",")[self.idx].isdigit() else self.idx
            h = pynvml.nvmlDeviceGetHandleByIndex(phys)
            self.max_mhz = float(pynvml.nvmlDeviceGetMaxClockInfo(h, pynvml.NVML_CLOCK_SM))
            names = {"hw_slowdown": getattr(pynvml, "nvmlClocksEventReasonHwSlowdown", 0x8),
                     "hw_thermal_slowdown": getattr(pynvml, "nvmlClocksEventReasonHwThermalSlowdown", 0x40),
                     "sw_thermal_slowdown": getattr(pynvml, "nvmlClocksEventReasonSwThermalSlowdown", 0x20),
                     "sw_power_cap": getattr(pynvml, "nvmlClocksEventReasonSwPowerCap", 0x4)}
            get_reasons = getattr(pynvml, "nvmlDeviceGetCurrentClocksEventReasons", None) or \
                pynvml.nvmlDeviceGetCurrentClocksThrottleReasons

            def loop():
                while not self.stop_flag.is_set():
                    try:
                        self.sm.append(float(pynvml.nvmlDeviceGetClockInfo(h, pynvml.NVML_CLOCK_SM)))
                        r = int(get_reasons(h))
                        for n, bit in names.items():
                            if r & bit:
                                self.reasons.add(n)
                        self.power.append(pynvml.nvmlDeviceGetPowerUsage(h) / 1000.0)
                    except Exception as e:  # keep sampling
                        self.err = repr(e)
                    time.sleep(self.period)
            self.thread = threading.Thread(target=loop, daemon=True)
            self.thread.start()
        except Exception as e:
            self.err = repr(e)

    def stop(self):
        self.stop_flag.set()
        if self.thread:
            self.thread.join(timeout=2)
        out = {"sm_mhz": float(np.median(self.sm)) if self.sm else None, "sm_max_mhz": self.max_mhz,
               "reasons": sorted(self.reasons), "samples": len(self.sm),
               "power_w_max": max(self.power) if self.power else None}
        if self.err and not self.sm:
            out["error"] = self.err
        return out


WORKLOAD = ("C2: 1024x1024 forward render, ~500k pixel-aligned Gaussians from 2 source views, fixed novel camera "
            "(ratio 0.5)")


def passes_per_step(steps, override=0):
    return int(override) if override else max(1, -(-2000 // max(1, int(steps))))


def bench_config(V, R, **extra):
    """The `config` object: identical in the b200 and the reference arm."""
    cfg = {"workload": WORKLOAD, "views_per_pass_per_gpu": int(V), "passes_per_step": int(R),
           "views_per_step_per_gpu": int(V * R)}
    cfg.update(extra)
    return cfg


def _source_hash(kernel="render_forward_kernel"):
    """sha256 over the CODE of a compositing kernel's sources (// comments and whitespace stripped, so a reworded comment
    does not invalidate a capture): stamps profiles/render_forward_traffic.json so that a stale ncu traffic figure is refused
    instead of silently reported."""
    import hashlib
    import re
    h = hashlib.sha256()
    main = "raster_backward.cu" if "backward" in kernel else "raster_render.cu"
    for f in (main, "slab_ring.cuh", "tma_bulk.cuh", "gpsg_internal.cuh"):
        with open(os.path.join(ROOT, "gps-gaussian_b200", "csrc", f), "r") as fh:
            code = re.sub(r"//[^\n]*", "", fh.read())
        h.update(re.sub(r"\s+", " ", code).strip().encode())
    return h.hexdigest()


TRAFFIC_FILE = os.path.join(ROOT, "profiles", "render_forward_traffic.json")


def _traffic(kernel):
    try:
        j = json.load(open(TRAFFIC_FILE))
    except Exception:
        return None, "no profiles/render_forward_traffic.json (no ncu capture of these kernels)"
    ent = j.get(kernel) if isinstance(j.get(kernel), dict) else (j if kernel == "render_forward_kernel" else None)
    if not ent:
        return None, "kernel not in traffic file"
    if ent.get("source_sha256") != _source_hash(kernel):
        return None, "stale: kernel sources changed since the ncu capture (source_sha256 mismatch)"
    return float(ent["dram_bytes_per_launch"]), ent.get("from", "ncu --set full")


DUMP_SAMPLE = 1 << 22          # pixel values of all views in color_sample.npy (16 MB)
DUMP_RADII = 1 << 20           # radii of all views in radii_sample.npy (4 MB)


def dump_outputs(out_dir, colors, radii, num_rendered):
    """What the timed path returned in its last step, as float32 / float64 .npy files (about 33 MB at 1024^2, whatever the
    number of views): color_view0 = the whole [3,H,W] image of the first view; color_sample = a fixed, seeded sample
    (DUMP_SAMPLE values, same indices in every run) of the flattened [V,3,H,W] images of all views; radii_sample = the same
    kind of sample (DUMP_RADII values) of every view's int32 radii, concatenated; num_rendered = the pair count of each
    view.  Inputs are seeded, so the same arguments give the same inputs."""
    import torch

    def sample(flat, n, seed):
        idx = np.sort(np.random.default_rng(seed).choice(flat.numel(), size=min(n, flat.numel()), replace=False))
        return flat[torch.from_numpy(idx).to(flat.device)]

    os.makedirs(out_dir, exist_ok=True)
    arrays = {"color_view0": colors[0].float().cpu().numpy(),
              "color_sample": sample(torch.stack(colors).reshape(-1), DUMP_SAMPLE, 1314).float().cpu().numpy(),
              "radii_sample": sample(torch.cat([r.reshape(-1) for r in radii]), DUMP_RADII, 1315).float().cpu().numpy(),
              "num_rendered": np.asarray(num_rendered, np.float64)}
    assert sum(a.nbytes for a in arrays.values()) <= 64 << 20, "output dump exceeds 64 MB"
    for name, a in arrays.items():
        np.save(os.path.join(out_dir, name + ".npy"), a)


def _scenes(n, first_seed):
    from gps_gaussian_b200 import synth
    return [synth.stereo_pair_scene(RES, seed=first_seed + k) for k in range(n)]


def _scenes_from_seeds(seeds):
    from gps_gaussian_b200 import synth
    return [synth.stereo_pair_scene(RES, seed=sd) for sd in seeds]


def _cpu_oracle_views_per_sec(sc, n_views, warm=1):
    """Times the CPU oracle port (forward: preprocess + bin + sort + composite) on the host cores."""
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from oracle.raster_oracle import RasterOracle
    o = RasterOracle("f32")
    fwd = lambda nt: o.forward(sc["means3D"], sc["colors"], sc["opacity"], sc["scales"], sc["rots"], sc["view"], sc["proj"],
                               sc["tanfovx"], sc["tanfovy"], sc["W"], sc["H"], sc["bg"], nthreads=nt)
    # torchrun exports OMP_NUM_THREADS=1; the CPU arm may use every host core.  Logical CPUs vs physical cores: pick
    # whichever thread count is faster on this box (one probe render each), so the baseline is not handicapped.
    global _CPU_THREADS
    if _CPU_THREADS is None:
        best = None
        for nt in sorted({o.max_threads(), max(1, o.max_threads() // 2)}, reverse=True):
            o.set_threads(nt)
            fwd(nt)
            t0 = time.perf_counter(); fwd(nt); dt = time.perf_counter() - t0
            if best is None or dt < best[0]:
                best = (dt, nt)
        _CPU_THREADS = best[1]
    threads = _CPU_THREADS
    o.set_threads(threads)
    run = lambda: fwd(threads)
    for _ in range(warm):
        run()
    t0 = time.perf_counter()
    for _ in range(n_views):
        run()
    dt = time.perf_counter() - t0
    return n_views / dt, threads, dt


def _taichi_port_views_per_sec(sc, reps=5):
    """Restated lib/TaichiRender.py point z-buffer (different algorithm; reported for context only)."""
    from oracle.raster_oracle import taichi_splat
    P = sc["means3D"].shape[0]
    hom = np.concatenate([sc["means3D"], np.ones((P, 1), np.float32)], 1) @ sc["proj"]
    ndc = hom[:, :2] / hom[:, 3:4]
    pts = np.concatenate([(ndc + 1) * 0.5 * RES, 1.0 / hom[:, 3:4], sc["colors"]], 1).astype(np.float32)[None]
    mask = np.ones((1, P), np.float32)
    taichi_splat(pts, mask, RES)
    t0 = time.perf_counter()
    for _ in range(reps):
        taichi_splat(pts, mask, RES)
    return reps / (time.perf_counter() - t0)


def run_reference_arm(args, rank, world):
    """CPU arm: same metric / unit / config as the b200 arm; each of the K steps is a bounded SAMPLE (one view) of the
    step's V*R views -- the CPU port renders ~5-20 views/s, a full step would take minutes."""
    if rank != 0:
        return
    R = passes_per_step(args.steps, args.passes)
    sc = _scenes(1, 1314)[0]
    vps, threads, _ = _cpu_oracle_views_per_sec(sc, 1, warm=max(1, min(args.warmup, 2)))   # warm-up
    t0 = time.perf_counter()
    n = 0
    for _ in range(args.steps):
        _cpu_oracle_views_per_sec(sc, 1, warm=0)
        n += 1
    dt = time.perf_counter() - t0
    val = n / dt
    line = {"impl": "reference", "metric": METRIC, "value": val, "unit": UNIT, "n_gpus": args.gpus, "steps": args.steps,
            "warmup": args.warmup, "ms_per_step": 1e3 * dt / max(n, 1), "higher_is_better": True, "scaling": "weak",
            "vs_baseline": None, "dtype": "f32", "data": "synthetic",
            "config": bench_config(args.views, R),
            "note": "reference GPU path (diff_gaussian_rasterization) and taichi are absent here; this is the CPU oracle "
                    "port of the same algorithm on the host cores",
            "cpu_baseline": {"value": val, "unit": UNIT, "cores": threads, "kind": "port",
                             "sample": f"each step = 1 of the step's {args.views * R} views (forward render of one C2 view, "
                                       f"P={int(sc['means3D'].shape[0])}); {n} steps, OpenMP over pixel rows"},
            "e2e": {"value": val, "unit": UNIT, "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}}
    print(json.dumps(line), flush=True)


def _corr_section(dev, hbm_peak_gbs):
    """Volume + pyramid build (fp16 wgmma kernel / fp16 + fp32 FFMA kernels) and the fused 4-level lookup, CUDA-event timed."""
    import torch
    from gps_gaussian_b200 import _lib
    from gps_gaussian_b200.corr import CorrBlockFast1D
    B, D, H, W = 2, 192, 128, 128
    gen = torch.Generator(device=dev).manual_seed(1314)
    f32 = [torch.randn(B, D, H, W, device=dev, generator=gen) for _ in range(2)]
    f16 = [t.half() for t in f32]
    coords = torch.stack(torch.meshgrid(torch.arange(H, device=dev), torch.arange(W, device=dev), indexing="ij")[::-1])[None]
    coords = (coords.float() + 6.0 * torch.randn(B, 2, H, W, device=dev, generator=gen)).contiguous()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

    def timed(fn, n=50):
        for _ in range(5):
            fn()
        torch.cuda.synchronize()
        e0.record()
        for _ in range(n):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / n

    out = {"shape": [B, D, H, W]}
    alg = lambda s: 2 * B * D * H * W * s + 1.875 * B * H * W * W * s          # SURVEY 8d: features in, volume + pyramid out
    with torch.no_grad():
        out["build_fp16_wgmma_ms"] = timed(lambda: CorrBlockFast1D(f16[0], f16[1]))
        _lib.set_corr_build("ffma")
        out["build_fp16_ffma_ms"] = timed(lambda: CorrBlockFast1D(f16[0], f16[1]))
        _lib.set_corr_build("wgmma")
        out["build_fp32_ffma_ms"] = timed(lambda: CorrBlockFast1D(f32[0], f32[1]))
        blk = CorrBlockFast1D(f16[0], f16[1])
        out["lookup_4level_fp16_ms"] = timed(lambda: blk(coords))
        # library data flow of the reference (core/corr.py:53-61 + :36-42) for comparison
        def ref_build():
            c = torch.einsum('aijk,aijh->ajkh', f16[0], f16[1]).reshape(B, H, W, 1, W) / torch.sqrt(torch.tensor(D).float())
            c = c.reshape(B * H * W, 1, 1, W)
            pyr = [c]
            for _ in range(3):
                c = torch.nn.functional.avg_pool2d(c, [1, 2], stride=[1, 2])
                pyr.append(c)
            return pyr
        out["build_fp16_torch_ops_ms"] = timed(ref_build)
    # backward of the build w.r.t. the feature maps (autograd through _BuildPyramid with a level-0 gradient)
    fa, fb_ = f16[0].clone().requires_grad_(True), f16[1].clone().requires_grad_(True)
    gvol = torch.randn(B, H, W, W, device=dev, generator=gen).half()

    def bwd():
        v0 = CorrBlockFast1D.corr(fa, fb_).squeeze(3)
        torch.autograd.grad(v0, (fa, fb_), gvol)
    out["build_fwd_bwd_fp16_wgmma_ms"] = timed(bwd, 20)
    _lib.set_corr_build("ffma")
    out["build_fwd_bwd_fp16_ffma_ms"] = timed(bwd, 20)
    _lib.set_corr_build("wgmma")
    # CPU port beside it (oracle, scalar C, 1 thread) on a bounded sample: 8 of the 128 rows of the same problem
    try:
        from oracle.corr_oracle import CorrOracle
        co = CorrOracle("f32")
        hs = 8
        n1, n2 = f32[0][:, :, :hs].cpu().numpy().copy(), f32[1][:, :, :hs].cpu().numpy().copy()
        cs = coords[:, :, :hs].cpu().numpy().copy()
        t0 = time.perf_counter()
        pyr = co.pyramid(n1, n2, 4)
        t_build = time.perf_counter() - t0
        t0 = time.perf_counter()
        co.lookup(pyr, cs, 4)
        t_look = time.perf_counter() - t0
        out["cpu_port"] = {"sample": f"rows 0..{hs - 1} of {H} (1/{H // hs} of the work), oracle C port, 1 thread",
                           "build_ms_sample": t_build * 1e3, "lookup_ms_sample": t_look * 1e3,
                           "build_ms_full_extrapolated": t_build * 1e3 * H / hs,
                           "lookup_ms_full_extrapolated": t_look * 1e3 * H / hs}
    except Exception as exc:
        out["cpu_port"] = {"error": repr(exc)}
    # per-KERNEL rooflines of the sampler side (BASELINE.md section 4 bytes; CUDA events around each launch, library-side):
    # the Python-call wall times above include allocation + ctypes, these do not
    try:
        co = coords.clone()
        vols = [v.detach() for v in blk._vols]
        grad = torch.randn(B, 36, H, W, device=dev, generator=gen).half()
        blk_g = CorrBlockFast1D(f16[0].clone().requires_grad_(True), f16[1].clone().requires_grad_(True))
        _lib.profile_enable(True)
        _lib.profile_read()
        n_it = 50
        for _ in range(n_it):
            o = blk_g(co)
            torch.autograd.grad(o, blk_g._vols, grad, retain_graph=False)
            CorrBlockFast1D(f16[0], f16[1])
        pr = _lib.profile_read()
        _lib.profile_enable(False)
        s2 = 2
        b_look = 4 * B * H * W * (10 * s2 + 4 + 9 * s2)          # 4 levels x (10 taps + coord + 9 outputs) per pixel
        b_look_bwd = 4 * B * H * W * (9 * s2 + 4) + sum(v.numel() for v in vols) * s2      # grads in + coord, dense grad volumes out
        roof = {}
        for key, name, nbytes in (("corr_forward", "corr_lookup_fwd_kernel (fused 4 levels)", b_look),
                                  ("corr_backward", "corr_lookup_bwd_kernel (fused 4 levels)", b_look_bwd),
                                  ("corr_build", "corr_build_tc_kernel (wgmma)", alg(2))):
            if pr.get(key, {}).get("calls"):
                ms = pr[key]["ms"] / pr[key]["calls"]
                roof[key] = {"kernel": name, "kernel_ms": ms, "algorithmic_bytes_per_launch": nbytes, "achieved_gbps": nbytes / (ms * 1e-3) / 1e9,
                             "frac_of_measured_hbm": nbytes / (ms * 1e-3) / 1e9 / hbm_peak_gbs, "bound": "hbm (launch-latency at this size)"}
        out["kernel_rooflines"] = roof
    except Exception as exc:
        out["kernel_rooflines"] = {"error": repr(exc)[:200]}
    out["build_fp16_wgmma_gbps"] = alg(2) / (out["build_fp16_wgmma_ms"] * 1e-3) / 1e9
    out["build_fp16_wgmma_hbm_frac"] = out["build_fp16_wgmma_gbps"] / hbm_peak_gbs
    out["note"] = "wall of the Python call (allocation of the 4 level tensors + 1 launch), CUDA events, back-to-back"
    return out


def _p2r_section(dev, args, rank, V):
    """Reference-signature pts2render(data, bg_color): fused map ingest vs the reference's gather data flow, the fused
    unprojection in front of it and the novel-view sweep around it (SURVEY 8f rows 1-3).  N=1 only."""
    import torch
    from types import SimpleNamespace
    from gps_gaussian_b200 import shard, synth as _synth
    from gps_gaussian_b200.GaussianRender import pts2render, pts2render_gather
    from gps_gaussian_b200.novel_calib import get_novel_calib
    from gps_gaussian_b200.novel_views import NovelViewRenderer
    from gps_gaussian_b200.unproject import flow2xyz
    scm = _synth.stereo_pair_scene(RES, seed=shard.unit_seeds(1314, V, rank)[0], keep_maps=True)
    camm = scm["cam"]
    pdata = {"novel_view": {"FovX": torch.tensor([camm["FovX"]], dtype=torch.float64),
                            "FovY": torch.tensor([camm["FovY"]], dtype=torch.float64),
                            "width": torch.tensor([RES]), "height": torch.tensor([RES]),
                            "world_view_transform": torch.tensor(camm["world_view_transform"])[None],
                            "full_proj_transform": torch.tensor(camm["full_proj_transform"])[None],
                            "camera_center": torch.tensor(camm["camera_center"])[None]}}
    for name, vw in zip(("lmain", "rmain"), scm["views"]):
        Tm = lambda a: torch.tensor(a).to(dev)[None]
        pdata[name] = {"img": Tm(vw["img"]), "pts_valid": torch.tensor(vw["valid"]).to(dev)[None], "xyz": Tm(vw["xyz"]),
                       "rot_maps": Tm(vw["rot_maps"]), "scale_maps": Tm(vw["scale_maps"]), "opacity_maps": Tm(vw["opacity_maps"])}
    p2r = {}
    with torch.no_grad():
        for nm, fn in (("fused_map_ingest", pts2render), ("gather_then_render", pts2render_gather)):
            for _ in range(3):
                fn(pdata, [0.0, 0.0, 0.0])
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(20):
                fn(pdata, [0.0, 0.0, 0.0])
            torch.cuda.synchronize()
            p2r[nm + "_ms"] = (time.perf_counter() - t0) * 1e3 / 20
    udata = {}
    for name, vw in zip(("lmain", "rmain"), scm["views"]):
        inv = np.where(vw["depth"] > 0, 1.0 / np.maximum(vw["depth"], 1e-6), 0.0).astype(np.float32)
        Kt = torch.tensor(vw["K"].astype(np.float32))[None].to(dev)
        udata[name] = {"flow_pred": torch.tensor(inv)[None, None].to(dev), "mask": torch.ones(1, 3, RES, RES, device=dev),
                       "intr": Kt, "extr": torch.tensor(np.vstack([vw["E"], [0, 0, 0, 1]]).astype(np.float32))[None].to(dev),
                       "ref_intr": Kt, "Tf_x": torch.tensor([1.0], device=dev)}
    with torch.no_grad():
        for _ in range(3):
            flow2xyz(udata)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(50):
            flow2xyz(udata)
        torch.cuda.synchronize()
        p2r["fused_unproject_both_views_ms"] = (time.perf_counter() - t0) * 1e3 / 50
    for name, vw in zip(("lmain", "rmain"), scm["views"]):
        pdata[name]["intr"] = torch.tensor(vw["K"].astype(np.float32))[None].to(dev)
        pdata[name]["extr"] = torch.tensor(vw["E"].astype(np.float32))[None].to(dev)
    opt = SimpleNamespace(use_hr_img=False, znear=_synth.ZNEAR, zfar=_synth.ZFAR, trans=[0.0, 0.0, 0.0], scale=1.0)
    ratios = [(i + 0.5) / 32 for i in range(32)]
    sweep = {"views_per_sweep": len(ratios)}
    with torch.no_grad():
        for mode in ("compact", "maps"):
            t0 = time.perf_counter()
            nvr = NovelViewRenderer(pdata, opt, [0.0, 0.0, 0.0], streams=args.streams, mode=mode)
            torch.cuda.synchronize()
            sweep[mode + "_build_ms"] = (time.perf_counter() - t0) * 1e3
            buf = torch.empty((1, len(ratios), 3, RES, RES), device=dev)
            nvr.render(ratios, out=buf)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(5):
                nvr.render(ratios, out=buf)
            torch.cuda.synchronize()
            sweep[mode + "_views_per_s"] = 5 * len(ratios) / (time.perf_counter() - t0)
            del nvr
        t0 = time.perf_counter()
        for r in ratios:
            pts2render(get_novel_calib(pdata, opt, ratio=r), [0.0, 0.0, 0.0])
        torch.cuda.synchronize()
        sweep["per_view_calib_plus_pts2render_views_per_s"] = len(ratios) / (time.perf_counter() - t0)
        sweep["max_abs_diff_last_view"] = float((buf[0, -1] - pdata["novel_view"]["img_pred"][0]).abs().max())
    p2r["novel_view_sweep"] = sweep
    return p2r


def _train_section(dev, calls, ndup, P, steps, V, peak):
    """Rasterizer forward+backward replay at C2 (the kernels BASELINE's efficiency target names), CUDA events around the
    whole loop, per-kernel events inside; plus the fused L1+SSIM loss beside the torch op chain."""
    import torch
    from gps_gaussian_b200 import _lib
    Rt = max(1, -(-400 // steps))
    grads = [torch.randn(3, RES, RES, device=dev) for _ in range(2)]
    for c in calls[:2]:
        c.forward(); c.backward(grads[0])
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    _lib.profile_enable(True)
    e0.record()
    for _ in range(steps * Rt):
        for i, c in enumerate(calls):
            c.forward(); c.backward(grads[i % 2])
    e1.record()
    torch.cuda.synchronize()
    tms = e0.elapsed_time(e1)
    tprof = _lib.profile_read()
    _lib.profile_enable(False)
    nd, pv, hw = float(np.mean(ndup)), float(np.mean(P)), RES * RES
    b_cbwd = 48 * nd + 20 * hw + 36 * nd                      # DESIGN.md section 5: slabs + (dL/dpix, T, n_contrib) + reduced grads
    b_pbwd = 116 * pv + 56 * pv
    rb, pb = tprof["render_backward"], tprof["preprocess_backward"]
    t_rb = rb["ms"] / max(rb["calls"], 1) * 1e-3
    t_pb = pb["ms"] / max(pb["calls"], 1) * 1e-3
    train = {"value": V * steps * Rt / (tms * 1e-3), "unit": "fwd+bwd views/s (1 GPU, exact one-sync entry points)",
             "timed_region_s": tms * 1e-3, "passes": steps * Rt,
             "stages_ms": {k: v["ms"] / max(v["calls"], 1) for k, v in tprof.items() if v["calls"]}}
    tr, src = _traffic("render_backward_q_kernel")
    roof_b = {"bound": "hbm", "kernel": "render_backward_q_kernel", "achieved": b_cbwd / t_rb / 1e9, "peak": peak, "unit": "GB/s",
              "frac": b_cbwd / t_rb / 1e9 / peak, "traffic": tr, "traffic_source": src, "algorithmic_bytes_per_launch": b_cbwd,
              "kernel_ms": t_rb * 1e3, "preprocess_backward": {"achieved": b_pbwd / t_pb / 1e9, "frac": b_pbwd / t_pb / 1e9 / peak,
                                                                "kernel_ms": t_pb * 1e3, "algorithmic_bytes_per_launch": b_pbwd},
              "note": "FP32-issue + L2-RED bound by design (DESIGN.md section 5); HBM fraction reported because the metric asks for it"}
    import torch.nn.functional as F
    from gps_gaussian_b200.loss import fused_l1_ssim

    def torch_ops_loss(x, y):
        gw = torch.tensor([np.exp(-(i - 5) ** 2 / 4.5) for i in range(11)], dtype=torch.float32, device=dev)
        gw = gw / gw.sum()
        win = (gw[:, None] * gw[None, :]).expand(3, 1, 11, 11).contiguous()
        cv = lambda t: F.conv2d(t, win, padding=5, groups=3)
        m1, m2 = cv(x), cv(y)
        s1, s2, s12 = cv(x * x) - m1 * m1, cv(y * y) - m2 * m2, cv(x * y) - m1 * m2
        sm = ((2 * m1 * m2 + 1e-4) * (2 * s12 + 9e-4)) / ((m1 * m1 + m2 * m2 + 1e-4) * (s1 + s2 + 9e-4))
        return 0.8 * (x - y).abs().mean() + 0.2 * (1.0 - sm.mean())

    gt_img = calls[1].color.detach().clone()[None]
    lt = {}
    for nm, fn in (("fused_fwd_bwd_ms", fused_l1_ssim), ("torch_ops_fwd_bwd_ms", torch_ops_loss)):
        xi = calls[0].color.detach().clone()[None].requires_grad_(True)
        for _ in range(3):
            fn(xi, gt_img).backward()
        torch.cuda.synchronize()
        e0.record()
        for _ in range(20):
            fn(xi, gt_img).backward()
        e1.record()
        torch.cuda.synchronize()
        lt[nm] = e0.elapsed_time(e1) / 20
    train["l1_ssim_loss_1024sq"] = lt
    return train, roof_b


def _c3_section(dev, n_steps=6):
    """BASELINE config C3 on this GPU: the reference's OWN RtStereoHumanModel + loader + train_stage2.py:57-89 step (AMP,
    GradScaler) from oracle/_ref against the drop-ins, 512^2 sources / 1024^2 render, batch 2 -- plain drop-ins and with
    the GPSG_PATCH fused paths.  Stage split by CUDA events between the statements of the step; rasterizer kernel time from
    the library's own per-kernel events."""
    import tempfile
    import torch
    from gps_gaussian_b200 import _lib, harness, patch, synth_dataset
    if harness.staged_reference() is None:
        return {"unavailable": "oracle/_ref not staged (build() stages it where the original project is checked out)"}
    root = tempfile.mkdtemp(prefix="gpsg_c3_")
    synth_dataset.write_dataset(root, n_train=2, n_val=1, res=512, hr=True)
    out = {"config": "C3: reference RtStereoHumanModel (5 144 408 params), AMP + GradScaler, batch 2, 512^2 stereo pair -> "
                     "1024^2 novel view, loss flow + 0.8 L1 + 0.2 (1-SSIM), AdamW", "steps_timed": n_steps}
    for mode in ("dropin", "dropin+GPSG_PATCH"):
        if mode != "dropin":
            patch.install()
        try:
            cfg = harness.load_cfg(root, src_res=512, num_steps=1000, batch_size=2)
            st = harness.C3State(cfg, device=str(dev))
            import lib.GaussianRender as ref_gr
            batches = [st.batch(k) for k in (0, 2)]
            for k in range(3):
                harness.c3_step(st, dict_copy(batches[k % 2]), pts2render=ref_gr.pts2render)
            torch.cuda.synchronize()
            timers = {}
            _lib.profile_enable(True)
            t0 = time.perf_counter()
            last = None
            for k in range(n_steps):
                last = harness.c3_step(st, dict_copy(batches[k % 2]), pts2render=ref_gr.pts2render, timers=timers)
            torch.cuda.synchronize()
            wall = (time.perf_counter() - t0) * 1e3 / n_steps
            prof = _lib.profile_read()
            _lib.profile_enable(False)
            kern = {k: v["ms"] / n_steps for k, v in prof.items() if v["calls"]}
            fwd_k = sum(v for k, v in kern.items() if k in ("preprocess", "scan", "duplicate", "sort", "gather", "tile_scan", "scatter", "tile_sort", "render_forward"))
            bwd_k = sum(v for k, v in kern.items() if k in ("render_backward", "preprocess_backward"))
            corr_k = sum(v for k, v in kern.items() if k.startswith("corr"))
            out[mode] = {"step_ms_wall": wall, "pixels_per_s": 2 * 1024 * 1024 / (wall * 1e-3),
                         "stages_ms": {k: v / n_steps for k, v in timers.items()},
                         "rasterizer_fwd_kernels_ms": fwd_k, "rasterizer_bwd_kernels_ms": bwd_k, "corr_kernels_ms": corr_k,
                         "kernels_ms": kern, "loss": float(last["loss"]), "grad_scale": last["scale_after"],
                         "scaler_skipped": bool(last["scale_after"] < last["scale_before"])}
            del st
        except Exception as exc:
            out[mode] = {"error": repr(exc)[:400]}
        finally:
            patch.uninstall()
    import shutil
    shutil.rmtree(root, ignore_errors=True)
    return out


def dict_copy(data):
    """Shallow per-view copy of a reference batch dict (the model writes its outputs into it)."""
    return {k: (dict(v) if isinstance(v, dict) else v) for k, v in data.items()}


def run_c5(args, rank, world, local_rank):
    """BASELINE config C5: stage-2 TRAINING data-parallel -- the reference's own model + step from oracle/_ref, 2 stereo
    pairs of 1024^2 per GPU (2048^2 novel view, use_hr_img), ONE flat NCCL all-reduce (5 144 408 fp32 = 20.6 MB) between
    backward and unscale_ (train_stage2.py:83-85).  metric: pixels/s of source-pair pixels trained on (16 x 1024^2 per
    step at N=8), plus the exposed all-reduce time (step with all-reduce minus step without)."""
    import tempfile
    import torch
    import torch.distributed as dist
    from gps_gaussian_b200 import harness, patch, shard
    torch.cuda.set_device(local_rank)
    dev = torch.device("cuda", local_rank)
    shard.init(backend="nccl", device=dev)
    res = args.c5_res
    root = os.path.join(tempfile.gettempdir(), f"gpsg_c5_data_{res}")
    if rank == 0 and not os.path.exists(os.path.join(root, "done")):
        from gps_gaussian_b200 import synth_dataset
        synth_dataset.write_dataset(root, n_train=2, n_val=1, res=res, hr=True)
        cfg0 = harness.load_cfg(root, src_res=res, num_steps=1000, batch_size=2)
        harness.add_reference_to_path()
        from lib.human_loader import StereoHumanDataset
        StereoHumanDataset(cfg0.dataset, phase='train')          # one rank writes rectified_local/, the others read it
        open(os.path.join(root, "done"), "w").close()
    shard.barrier(dev)
    if args.patch:
        patch.install()
    cfg = harness.load_cfg(root, src_res=res, num_steps=1000, batch_size=2)
    st = harness.C3State(cfg, seed=1314, device=str(dev))            # same seed => identical replicas
    import lib.GaussianRender as ref_gr
    batches = [st.batch(k) for k in (0, 2)]
    bucket = [None]

    def ar(params):
        bucket[0] = shard.allreduce_grads(list(params), bucket[0])

    for k in range(max(3, args.warmup)):
        harness.c3_step(st, dict_copy(batches[k % 2]), pts2render=ref_gr.pts2render, allreduce=ar)
    sampler = ClockSampler(local_rank)
    res_ms = {}
    from gps_gaussian_b200 import _lib
    _lib.profile_enable(2)                     # count our own kernel launches (process-wide: the backward runs on autograd's thread)
    _lib.profile_read()
    for label, fn in (("with_allreduce", ar), ("without_allreduce", None)):
        shard.barrier(dev)
        if label == "with_allreduce":
            sampler.start()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        timers = {}
        e0.record()
        for k in range(args.steps):
            harness.c3_step(st, dict_copy(batches[k % 2]), pts2render=ref_gr.pts2render, allreduce=fn, timers=timers)
        e1.record()
        shard.barrier(dev)
        res_ms[label] = shard.max_over_ranks(e0.elapsed_time(e1), dev) / args.steps
        res_ms[label + "_stages"] = {k: v / args.steps for k, v in timers.items()}
        if label == "with_allreduce":
            clocks = sampler.stop()
            launches = sum(v["launches"] for v in _lib.profile_read().values())
    # replicas must still be identical after the averaged updates
    flat = torch.cat([p.detach().reshape(-1) for p in st.model.parameters()])
    chk = torch.stack([flat.double().sum(), flat.double().abs().sum()])
    lo, hi = chk.clone(), chk.clone()
    if world > 1:
        dist.all_reduce(lo, op=dist.ReduceOp.MIN); dist.all_reduce(hi, op=dist.ReduceOp.MAX)
    in_sync = bool(torch.equal(lo, hi))
    if rank == 0:
        px = 2 * res * res * world
        ms = res_ms["with_allreduce"]
        line = {"metric": "stage2_train_source_pixels_per_sec", "value": px / (ms * 1e-3), "unit": "pixels/s", "n_gpus": world,
                "steps": args.steps, "warmup": max(3, args.warmup), "ms_per_step": ms, "higher_is_better": True, "scaling": "weak",
                "vs_baseline": None, "dtype": "fp16 autocast nets + fp32 rasterizer (reference AMP)", "data": "synthetic",
                "config": {"workload": f"C5: stage-2 training, reference RtStereoHumanModel from oracle/_ref, 2 pairs/GPU of {res}^2 "
                                       f"(render {2 * res}^2), global batch {2 * world}, flat NCCL all-reduce of 5144408 fp32 grads",
                           "fast_paths": "GPSG_PATCH fused paths" if args.patch else "plain drop-ins", "parallelism": f"dp{world}"},
                "exposed_comm_ms": res_ms["with_allreduce_stages"].get("allreduce"),
                "exposed_comm_note": "CUDA-event time of the all-reduce stage between backward and unscale_ (flatten + NCCL SUM + "
                                     "divide + unflatten; nothing overlaps it); the step-time difference of two separate loops is also given "
                                     "but includes the drift of the training state",
                "step_ms_minus_step_ms_without_allreduce": ms - res_ms["without_allreduce"],
                "ms_per_step_without_allreduce": res_ms["without_allreduce"],
                "stages_ms": res_ms["with_allreduce_stages"], "allreduce_bytes": 5144408 * 4, "replicas_in_sync": in_sync,
                "clocks": clocks, "gpu_launches": int(launches)}
        print(json.dumps(line), flush=True)
    if world > 1:
        dist.destroy_process_group()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--views", type=int, default=8, help="view-pairs per GPU per pass")
    ap.add_argument("--passes", type=int, default=0, help="passes over the V views per step (default ceil(2000/steps))")
    ap.add_argument("--streams", type=int, default=8, help="CUDA streams the independent views of a pass are issued on")
    ap.add_argument("--impl", default="b200", choices=["b200", "reference"])
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--no-numa-bind", action="store_true", help="do not pin the process to the GPU-local NUMA node")
    ap.add_argument("--train", action="store_true", help="(default on; kept for compatibility)")
    ap.add_argument("--no-train", action="store_true", help="skip the rasterizer fwd+bwd block")
    ap.add_argument("--no-c3", action="store_true", help="skip the C3 block (reference stage-2 step against the drop-ins)")
    ap.add_argument("--no-extras", action="store_true", help="skip pts2render / sweep / correlation side measurements")
    ap.add_argument("--train-c5", action="store_true", help="time data-parallel stage-2 training (C5) instead of the render")
    ap.add_argument("--c5-res", type=int, default=1024)
    ap.add_argument("--patch", action="store_true", help="C5: use the GPSG_PATCH fused paths")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="write the images (and radii) the timed path computed in its last step to DIR/*.npy")
    args = ap.parse_args()
    args.warmup = max(args.warmup, 3) if args.impl == "b200" else args.warmup

    rank = int(os.environ.get("RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    if args.impl == "reference":
        run_reference_arm(args, rank, world)
        return

    import torch
    import torch.distributed as dist
    if not torch.cuda.is_available():
        raise SystemExit("bench.py: no CUDA device (the product path has no CPU fallback)")
    if args.train_c5:
        run_c5(args, rank, world, local_rank)
        return
    torch.cuda.set_device(local_rank)
    dev = torch.device("cuda", local_rank)
    from gps_gaussian_b200 import shard
    numa = shard.bind_host_to_gpu(local_rank) if not args.no_numa_bind else {"bound": False, "why": "--no-numa-bind"}
    shard.init(backend="nccl", device=dev)

    from gps_gaussian_b200 import _lib
    from gps_gaussian_b200.introspect import RasterCall, to_device

    V = args.views
    R = passes_per_step(args.steps, args.passes)
    scenes = [s_ for s_ in _scenes_from_seeds(shard.unit_seeds(1314, V, rank))]
    from gps_gaussian_b200.planned import PlannedRasterizer
    from gps_gaussian_b200.introspect import make_settings
    calls = [RasterCall(sc, to_device(sc, dev), dev) for sc in scenes]       # exact (one-sync) entry point
    P = [c.P for c in calls]
    for c in calls:
        c.forward()
    torch.cuda.synchronize()
    # device-resident loop: the sync-free planned entry point (caller-owned buffers, capacity = 1.25 x pairs)
    planned = [PlannedRasterizer(c.P, RES, RES, int(c.num_rendered * 1.25) + 1024, dev) for c in calls]
    pargs = [(make_settings(c.sc), c.inp["means3D"], c.inp["colors"], c.inp["opacity"], c.inp["scales"], c.inp["rots"])
             for c in calls]

    # independent views are issued round-robin on `--streams` CUDA streams: the latency-bound binning kernels of one
    # view overlap the issue-bound compositing of another (each planned rasterizer owns its buffers)
    side = [torch.cuda.Stream(dev) for _ in range(max(1, args.streams))]

    def one_pass():
        main = torch.cuda.current_stream(dev)
        for st in side:
            st.wait_stream(main)
        for k, (pr, a) in enumerate(zip(planned, pargs)):
            with torch.cuda.stream(side[k % len(side)]):
                pr.forward(*a)
        for st in side:
            main.wait_stream(st)

    def step():
        for _ in range(R):
            one_pass()

    def barrier():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    for _ in range(args.warmup):
        step()
    barrier()
    ndup = [c.num_rendered for c in calls]
    sampler = ClockSampler(local_rank)
    sampler.start()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    _lib.profile_enable(2)                    # count launches only: no per-kernel events inside the timed region
    barrier()
    e0.record()
    for _ in range(args.steps):
        step()
    e1.record()
    barrier()
    ms = e0.elapsed_time(e1)
    prof_overlapped = _lib.profile_read()
    if args.dump_outputs and rank == 0:
        dump_outputs(args.dump_outputs, [pr.color for pr in planned], [pr.radii[:c.P] for pr, c in zip(planned, calls)],
                     [pr.status()["num_rendered"] for pr in planned])
    clocks = sampler.stop()
    ms = shard.max_over_ranks(ms, dev)
    # Per-kernel durations for the roofline: with several streams the kernels of different views time-share the SMs, so
    # an event pair around one launch also counts the other views' work.  The same passes are therefore re-run on ONE
    # stream (serialised, like ncu's launch list) with per-kernel CUDA events on, and the kernel time is taken from that.
    def pass_serial():
        for pr, a in zip(planned, pargs):
            pr.forward(*a)
    _lib.profile_enable(True)
    pass_serial()
    barrier()
    _lib.profile_read()
    n_serial = max(16, (args.steps * R) // 8)
    e0.record()
    for _ in range(n_serial):
        pass_serial()
    e1.record()
    barrier()
    serial_ms_per_view = e0.elapsed_time(e1) / (n_serial * V)
    prof = _lib.profile_read()
    _lib.profile_enable(False)
    planned_ok = all(pr.ok() for pr in planned) and all(torch.equal(pr.color, c.color) for pr, c in zip(planned, calls))
    if not planned_ok:
        raise SystemExit("bench.py: planned forward overflowed or differs from the exact entry point")
    # same loop replayed from CUDA graphs (one graph per scene): reported as an extra, not as `value`
    for pr, a in zip(planned, pargs):
        pr.capture(*a)
    barrier()
    e0.record()
    main = torch.cuda.current_stream(dev)
    for _ in range(args.steps * R):
        for st in side:
            st.wait_stream(main)
        for k, pr in enumerate(planned):
            with torch.cuda.stream(side[k % len(side)]):
                pr.replay()
        for st in side:
            main.wait_stream(st)
    e1.record()
    barrier()
    graph_ms = shard.max_over_ranks(e0.elapsed_time(e1), dev)
    total_views = V * R * args.steps * world
    graph_value = total_views / (graph_ms * 1e-3)
    value = total_views / (ms * 1e-3)

    # ---- end-to-end through the reference-facing call, HOST buffers, copies inside the timed region ----
    from gps_gaussian_b200.pipeline import HostRenderPipeline, pack_host
    host = []
    for sc in scenes:
        h = pack_host(sc)            # one pinned buffer per view: [means3D | colors | rots | scales | opacity]
        cam = sc["cam"]
        data = {"novel_view": {"FovX": torch.tensor([cam["FovX"]], dtype=torch.float64),
                               "FovY": torch.tensor([cam["FovY"]], dtype=torch.float64),
                               "width": torch.tensor([RES]), "height": torch.tensor([RES]),
                               "world_view_transform": torch.tensor(cam["world_view_transform"])[None].pin_memory(),
                               "full_proj_transform": torch.tensor(cam["full_proj_transform"])[None].pin_memory(),
                               "camera_center": torch.tensor(cam["camera_center"])[None].pin_memory()}}
        host.append((h, data))
    out_host = [torch.empty((3, RES, RES), dtype=torch.float32).pin_memory() for _ in range(V)]
    h2d_pass = sum(h[0].numel() * 4 for h, _ in host)
    d2h_pass = V * out_host[0].numel() * 4
    pipe = HostRenderPipeline(dev, max(P), RES, RES)
    items = [(h, data, 0) for h, data in host]
    Re = max(1, -(-480 // args.steps))                  # e2e passes per step: >= ~2 s of wall clock at ~4.5 ms per pass

    # one step = Re passes over the V host-resident views, submitted to the pipeline as ONE stream of V*Re views (each view:
    # its own 28 MB pinned-host -> device upload, render through `render(data, idx, ...)`, 12.6 MB image back to pinned host
    # memory -- the V output buffers are reused pass after pass).  r1 drained the pipeline after every 8 views, which charges
    # one un-overlapped upload + download per 8 views to the link-bound loop.
    items_step = items * Re
    outs_step = out_host * Re

    def e2e_step():
        pipe.run(items_step, outs_step)    # returns once every image of the step is in host memory

    pipe.run(items, out_host); pipe.run(items, out_host); pipe.run(items, out_host)
    barrier()
    t0 = time.perf_counter()
    for _ in range(args.steps):
        e2e_step()
    barrier()
    e2e_ms = (time.perf_counter() - t0) * 1e3        # host wall clock: includes every copy, sync and Python overhead
    e2e_ms = shard.max_over_ranks(e2e_ms, dev)
    e2e_val = V * Re * args.steps * world / (e2e_ms * 1e-3)
    # cross-check the last image of the step against the device-resident render of the same scene
    e2e_err = float((out_host[V - 1].to(dev) - calls[V - 1].color).abs().max())
    # what bounds it: the host link.  Pinned H2D / D2H copy bandwidth with the same per-view transfer sizes (28 MB in,
    # 12.6 MB out), measured on ALL ranks at the same time (ranks on one socket share its PCIe root complex / memory
    # controllers) and gathered, so the per-rank figure at N GPUs is the ceiling the N-GPU e2e number runs against.
    link = {}
    hbuf, dbuf = host[0][0][0], torch.empty_like(host[0][0][0], device=dev)
    dimg = torch.empty((3, RES, RES), dtype=torch.float32, device=dev)
    s_in, s_out = torch.cuda.Stream(dev), torch.cuda.Stream(dev)

    def both(n):
        for _ in range(n):
            with torch.cuda.stream(s_in):
                dbuf.copy_(hbuf, non_blocking=True)
            with torch.cuda.stream(s_out):
                out_host[0].copy_(dimg, non_blocking=True)
    for name, fn, nbytes in (("h2d_alone_gbps", lambda n: [dbuf.copy_(hbuf, non_blocking=True) for _ in range(n)], hbuf.numel() * 4),
                             ("d2h_alone_gbps", lambda n: [out_host[0].copy_(dimg, non_blocking=True) for _ in range(n)], dimg.numel() * 4),
                             ("h2d_while_d2h_gbps", both, hbuf.numel() * 4)):
        fn(3)
        barrier()
        t0 = time.perf_counter()
        fn(40)
        torch.cuda.synchronize()
        link[name] = 40 * nbytes / (time.perf_counter() - t0) / 1e9
        barrier()
    mine = torch.tensor([link["h2d_alone_gbps"], link["d2h_alone_gbps"], link["h2d_while_d2h_gbps"]], dtype=torch.float64, device=dev)
    if world > 1:
        allr = [torch.zeros_like(mine) for _ in range(world)]
        dist.all_gather(allr, mine)
        per_rank = [[round(float(v), 2) for v in t.tolist()] for t in allr]
    else:
        per_rank = [[round(float(v), 2) for v in mine.tolist()]]
    link["concurrent_per_rank_[h2d,d2h,h2d_while_d2h]_gbps"] = per_rank
    link["h2d_while_d2h_gbps_min_over_ranks"] = min(r[2] for r in per_rank)
    link["e2e_h2d_gbps_per_gpu"] = e2e_val / world * (h2d_pass / V) / 1e9
    link["e2e_frac_of_link"] = link["e2e_h2d_gbps_per_gpu"] / link["h2d_while_d2h_gbps_min_over_ranks"]

    p2r = corr = train = roof_b = c3 = None
    peak, peak_src = _peaks()
    if world == 1:
        try:
            if not args.no_extras:
                p2r = _p2r_section(dev, args, rank, V)
        except Exception as exc:
            p2r = {"error": repr(exc)[:300]}
        if not args.no_train:
            try:
                train, roof_b = _train_section(dev, calls, ndup, P, args.steps, V, peak)
            except Exception as exc:                               # never lose the headline line to an auxiliary measurement
                train, roof_b = {"error": repr(exc)[:300]}, None

    if rank != 0:
        if world > 1:
            dist.destroy_process_group()
        return

    # ---- roofline of the dominant kernel (compositing), algorithmic bytes per launch (DESIGN.md) ----
    nd, hw = float(np.mean(ndup)), RES * RES
    b_comp = 48.0 * nd + 12.0 * hw + 8.0 * hw          # slab fetch + rgb out + final_T/n_contrib
    rf = prof["render_forward"]
    t_kernel = rf["ms"] / max(rf["calls"], 1) * 1e-3
    achieved = b_comp / t_kernel / 1e9
    stages = {k: v["ms"] / max(v["calls"], 1) for k, v in prof.items() if v["calls"]}
    own = sum(v["launches"] for k, v in prof_overlapped.items() if k not in ("scan", "sort"))   # launches in the timed region
    cubl = sum(v["launches"] for k, v in prof_overlapped.items() if k in ("scan", "sort"))
    traffic, traffic_src = _traffic("render_forward_kernel")

    if world == 1 and not args.no_extras:
        # the other half of the path: RAFT-Stereo 1-D correlation at the C2 input size (fmaps [2,192,128,128])
        try:
            corr = _corr_section(dev, peak)
        except Exception as exc:                                   # never lose the headline line to an auxiliary measurement
            corr = {"error": repr(exc)[:300]}
    if world == 1 and not args.no_c3:
        try:
            c3 = _c3_section(dev)
        except Exception as exc:
            c3 = {"error": repr(exc)[:400]}

    cpu = None
    if world == 1 and not args.no_cpu_baseline:
        shard.unbind_host()                                      # the CPU arm may use every host core
        vps, threads, dt = _cpu_oracle_views_per_sec(scenes[0], 8)
        cpu = {"value": vps, "unit": UNIT, "cores": threads, "kind": "port",
               "sample": f"8 forward renders of one C2 view ({dt:.1f} s), CPU oracle port, OpenMP compositing",
               "taichi_point_splat_port_views_per_s": _taichi_port_views_per_sec(scenes[0]),
               "host_cpu_count": os.cpu_count()}

    line = {"metric": METRIC, "value": value, "unit": UNIT, "n_gpus": world, "steps": args.steps, "warmup": args.warmup,
            "ms_per_step": ms / args.steps, "higher_is_better": True, "scaling": "weak", "vs_baseline": None,
            "dtype": "f32", "data": "synthetic",
            "config": bench_config(V, R, P_mean=float(np.mean(P)), N_dup_mean=nd,
                                   parallelism=f"view-pairs sharded over {world} GPU(s); {len(side)} CUDA stream(s) per GPU",
                                   l2=f"{V} distinct scenes per pass, ~{(56 * np.mean(P) + 96 * nd + 20 * hw) / 1e6:.0f} MB touched per "
                                      "view > 50 MB L2 between reuses",
                                   timed_region_s=ms * 1e-3),
            "roofline": {"bound": "hbm", "kernel": "render_forward_kernel", "achieved": achieved, "peak": peak,
                         "unit": "GB/s", "frac": achieved / peak, "traffic": traffic, "traffic_source": traffic_src,
                         "peak_source": peak_src,
                         "algorithmic_bytes_per_launch": b_comp, "kernel_ms": t_kernel * 1e3,
                         "kernel_ms_source": "CUDA events around the launch, serialised single-stream pass inside bench.py",
                         "serial_ms_per_view": serial_ms_per_view,
                         "note": "compositing is FP32/SFU-issue-bound by design (about 130 FLOP/B); see DESIGN.md"},
            "roofline_backward": roof_b,
            "stages_ms": stages, "value_cuda_graph_replay": graph_value, "pts2render_ms_per_call": p2r, "corr": corr,
            "entry_point": "gpsg_rasterize_forward_planned (sync-free; verified bit-identical to gpsg_rasterize_forward)",
            "cpu_baseline": cpu,
            "e2e": {"value": e2e_val, "unit": UNIT, "h2d_bytes_per_step": int(h2d_pass * Re), "d2h_bytes_per_step": int(d2h_pass * Re),
                    "passes_per_step": Re, "timed_region_s": e2e_ms * 1e-3,
                    "api": "gps_gaussian_b200.pipeline.HostRenderPipeline.run(all views of the step) -> gaussian_renderer.render(data, idx, "
                           "...) per view; pinned-host inputs, 3-stream H2D/compute/D2H overlap, host wall clock", "max_abs_diff_vs_device_path": e2e_err,
                    "host_link": link, "host_numa_binding": numa},
            "gpu_launches": int(own), "cub_launches": int(cubl), "clocks": clocks, "train": train, "train_c3": c3}
    print(json.dumps(line), flush=True)
    if world > 1:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
