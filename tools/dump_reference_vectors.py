#!/usr/bin/env python
"""Dump golden vectors from the REAL third-party extensions, for the day a machine that has them is available
(SURVEY.md section 8c; VERDICT r1 "missing" item 6).

The rasterizer arithmetic GPS-Gaussian calls lives in graphdeco-inria/diff-gaussian-rasterization (pre-`antialiasing`
API, 2-tuple return) and the sampler in princeton-vl/RAFT-Stereo `sampler/` (`corr_sampler`); neither is in this image,
so oracle/gpsg_oracle.c is "parity unpinned" (DESIGN.md section 2).  Run this script ONCE on any CUDA machine where

    pip install git+https://github.com/graphdeco-inria/diff-gaussian-rasterization   (the revision GPS-Gaussian was built on)
    cd RAFT-Stereo/sampler && python setup.py install

succeeded -- with THIS repository's `gps-gaussian_b200/dropin` NOT on PYTHONPATH -- and commit the files it writes to
tests/golden/.  tests/test_reference_vectors.py then pins (i) the CPU oracle and (ii) the sm_90a kernels to the real
extension's outputs: radii bit-exact, RGB <= 1e-4, gradients <= 1e-3 rel (BASELINE.json north_star), sampler <= 1e-6.

    python tools/dump_reference_vectors.py [--out tests/golden] [--device cuda:0]

Inputs are the seeded synthetic scenes of gps_gaussian_b200/synth.py (numpy only), so the vectors are reproducible from
this repository alone; outputs are stored as float32 npz (a few MB).
"""
import argparse
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

RASTER_CASES = {            # name -> synth.random_cube_scene kwargs (same cases as tests/test_raster_gpu.py)
    "c1": dict(P=10_000, res=256),
    "ragged_bg": dict(P=4000, res=250, spread=0.6, scale_mul=4.0, bg=(0.3, 0.6, 0.9), seed=11),
    "saturating": dict(P=300, res=64, spread=0.3, scale_mul=12.0, bg=(1.0, 1.0, 1.0), seed=11),
    "wide_cloud": dict(P=2000, res=130, spread=3.0, scale_mul=1.0, bg=(0.0, 0.0, 0.0), seed=11),
}
CORR_CASES = {"b2_h32_w16_d32": dict(B=2, D=32, H=16, W=32)}


def _require_real(mod, ours_marker="gps-gaussian_b200"):
    if ours_marker in (getattr(mod, "__file__", "") or ""):
        raise SystemExit(f"{mod.__name__} resolves to this repository's drop-in ({mod.__file__}); remove dropin/ from "
                         "PYTHONPATH -- the point of this script is to record the REAL extension")


def dump_raster(out_dir, device):
    import torch
    import diff_gaussian_rasterization as dgr
    _require_real(dgr)
    from gps_gaussian_b200 import synth
    for name, kw in RASTER_CASES.items():
        kw = dict(kw)
        sc = synth.random_cube_scene(kw.pop("P"), kw.pop("res"), **kw)
        T = lambda a: torch.tensor(np.asarray(a, np.float32), device=device, requires_grad=True)
        m, c, op, s, r = T(sc["means3D"]), T(sc["colors"]), T(sc["opacity"]), T(sc["scales"]), T(sc["rots"])
        m2d = torch.zeros_like(m, requires_grad=True)
        cam = lambda k, shape: torch.tensor(np.asarray(sc[k], np.float32).reshape(shape), device=device)
        rs = dgr.GaussianRasterizationSettings(
            image_height=int(sc["H"]), image_width=int(sc["W"]), tanfovx=float(sc["tanfovx"]), tanfovy=float(sc["tanfovy"]),
            bg=cam("bg", (3,)), scale_modifier=1.0, viewmatrix=cam("view", (4, 4)), projmatrix=cam("proj", (4, 4)),
            sh_degree=3, campos=cam("campos", (3,)), prefiltered=False, debug=False)
        img, radii = dgr.GaussianRasterizer(raster_settings=rs)(means3D=m, means2D=m2d, opacities=op, shs=None,
                                                                colors_precomp=c, scales=s, rotations=r, cov3D_precomp=None)
        g = np.random.default_rng(0).standard_normal(tuple(img.shape)).astype(np.float32)
        img.backward(torch.from_numpy(g).to(device))
        np.savez_compressed(os.path.join(out_dir, f"raster_reference_{name}.npz"), case=name,
                            color=img.detach().cpu().numpy(), radii=radii.cpu().numpy().astype(np.int32), grad_out=g,
                            dL_dmeans3D=m.grad.cpu().numpy(), dL_dmeans2D=m2d.grad.cpu().numpy(), dL_dcolors=c.grad.cpu().numpy(),
                            dL_dopacity=op.grad.cpu().numpy(), dL_dscales=s.grad.cpu().numpy(), dL_drots=r.grad.cpu().numpy(),
                            extension=str(getattr(dgr, "__file__", "?")))
        print("wrote raster", name, tuple(img.shape), int((radii > 0).sum()), "visible")


def dump_corr(out_dir, device):
    import torch
    import corr_sampler
    _require_real(corr_sampler)
    from gps_gaussian_b200 import synth
    for name, kw in CORR_CASES.items():
        f1, f2, coords = synth.corr_inputs(kw["B"], kw["D"], kw["H"], kw["W"])
        vol = np.einsum("bdhw,bdhv->bhwv", f1, f2).astype(np.float32) / np.float32(np.sqrt(np.float32(kw["D"])))
        v = torch.from_numpy(vol).to(device)
        cd = torch.from_numpy(coords).to(device)
        out, = corr_sampler.forward(v, cd, 4)
        g = np.random.default_rng(1).standard_normal(tuple(out.shape)).astype(np.float32)
        gv, = corr_sampler.backward(v, cd, torch.from_numpy(g).to(device), 4)
        np.savez_compressed(os.path.join(out_dir, f"corr_reference_{name}.npz"), volume=vol, coords=coords, radius=4,
                            out=out.cpu().numpy(), grad_out=g, grad_volume=gv.cpu().numpy())
        print("wrote corr", name, tuple(out.shape))


if __name__ == "__main__":
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--out", default=os.path.join(ROOT, "tests", "golden"))
    ap.add_argument("--device", default="cuda:0")
    ap.add_argument("--skip-corr", action="store_true")
    a = ap.parse_args()
    os.makedirs(a.out, exist_ok=True)
    dump_raster(a.out, a.device)
    if not a.skip_corr:
        dump_corr(a.out, a.device)
