"""Generate tests/golden/novel_calib_golden.npz from the REFERENCE's own get_novel_calib (lib/utils.py:8-54).

Run with GPSG_REFERENCE naming a checkout of the original project (+ scipy):  python tests/golden/make_novel_calib_golden.py
The reference ends with five `.cuda()` copies; there is no GPU here, so `torch.Tensor.cuda` is shimmed to the identity
for the duration of the call (the values are unaffected).  Cases: the benchmark's ring cameras (22.5 deg apart), random
rotation pairs up to ~170 deg apart, perturbed intrinsics, `use_hr_img` on/off, non-zero trans / scale."""
import os
import sys
from types import SimpleNamespace

import numpy as np
import torch

sys.path.insert(0, os.environ["GPSG_REFERENCE"])
from lib.utils import get_novel_calib  # noqa: E402
from scipy.spatial.transform import Rotation as Rot  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from gps_gaussian_b200 import synth  # noqa: E402

RATIOS = [0.0, 0.1, 0.5, 0.9, 1.0]


def main():
    rng = np.random.default_rng(1314)
    res = 1024
    K0, E0 = synth.ring_camera(-11.25, res)
    K1, E1 = synth.ring_camera(+11.25, res)
    intr0, intr1, extr0, extr1 = [K0], [K1], [E0], [E1]
    for ang in (5.0, 60.0, 120.0, 170.0):
        Ra = Rot.random(random_state=int(ang)).as_matrix()
        axis = rng.standard_normal(3); axis /= np.linalg.norm(axis)
        Rb = Rot.from_rotvec(axis * np.deg2rad(ang)).as_matrix() @ Ra
        extr0.append(np.concatenate([Ra, rng.uniform(-2, 2, (3, 1))], 1))
        extr1.append(np.concatenate([Rb, rng.uniform(-2, 2, (3, 1))], 1))
        Ka, Kb = K0.copy(), K1.copy()
        Ka[0, 0] *= rng.uniform(0.8, 1.2); Ka[1, 1] *= rng.uniform(0.8, 1.2); Ka[:2, 2] += rng.uniform(-30, 30, 2)
        Kb[0, 0] *= rng.uniform(0.8, 1.2); Kb[1, 1] *= rng.uniform(0.8, 1.2); Kb[:2, 2] += rng.uniform(-30, 30, 2)
        intr0.append(Ka); intr1.append(Kb)
    f32 = lambda xs: torch.tensor(np.stack(xs).astype(np.float32))
    bs = len(intr0)
    out = dict(intr0=f32(intr0).numpy(), intr1=f32(intr1).numpy(), extr0=f32(extr0).numpy(), extr1=f32(extr1).numpy(),
               ratios=np.array(RATIOS), width=np.full(bs, res, np.int32), height=np.full(bs, res, np.int32))
    cuda = torch.Tensor.cuda
    torch.Tensor.cuda = lambda self, *a, **k: self
    try:
        for tag, opt in (("plain", SimpleNamespace(use_hr_img=False, znear=0.01, zfar=100.0, trans=[0.0, 0.0, 0.0], scale=1.0)),
                         ("hr", SimpleNamespace(use_hr_img=True, znear=0.01, zfar=100.0, trans=[0.0, 0.0, 0.0], scale=1.0)),
                         ("shift", SimpleNamespace(use_hr_img=False, znear=0.05, zfar=20.0, trans=[0.1, -0.2, 0.3], scale=1.5))):
            side = 2 * res if opt.use_hr_img else res
            acc = {k: [] for k in ("FovX", "FovY", "world_view_transform", "full_proj_transform", "camera_center")}
            for r in RATIOS:
                data = {"lmain": {"intr": f32(intr0), "extr": f32(extr0)}, "rmain": {"intr": f32(intr1), "extr": f32(extr1)},
                        "novel_view": {"width": torch.full((bs,), side, dtype=torch.int32),
                                       "height": torch.full((bs,), side, dtype=torch.int32)}}
                data = get_novel_calib(data, opt, ratio=r)
                for k in acc:
                    acc[k].append(data["novel_view"][k].numpy())
            for k, v in acc.items():
                out[f"{tag}_{k}"] = np.stack(v, 1)                      # [bs, n_ratios, ...]
            out[f"{tag}_side"] = np.int32(side)
    finally:
        torch.Tensor.cuda = cuda
    np.savez_compressed(os.path.join(HERE, "novel_calib_golden.npz"), **out)
    print({k: v.shape for k, v in out.items()})


if __name__ == "__main__":
    main()
