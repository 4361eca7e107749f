"""Generate tests/golden/unproject_golden.npz from the REFERENCE's own flow2depth / depth2pc.

Run with GPSG_REFERENCE naming a checkout of the original project:  python tests/golden/make_unproject_golden.py
Imports lib/utils.py:87-119 and replays lib/network.py:64-69 (flow2gsparms) on seeded fp64 inputs on the CPU;
stores inputs, depth, xyz, pts_valid and the autograd gradient d(loss)/d(flow_pred) for a random d(loss)/d(xyz)."""
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.environ["GPSG_REFERENCE"])
from lib.utils import depth2pc, flow2depth  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from gps_gaussian_b200 import synth  # noqa: E402


def main():
    torch.set_default_dtype(torch.float64)      # depth2pc builds its pixel grid with the default dtype
    rng = np.random.default_rng(1314)
    B, S = 2, 24
    K0, E0 = synth.ring_camera(-11.25, S)
    K1, E1 = synth.ring_camera(+11.25, S)
    intr = torch.tensor(np.stack([K0, K1]))
    extr = torch.tensor(np.stack([np.vstack([E0, [0, 0, 0, 1]]), np.vstack([E1, [0, 0, 0, 1]])]))    # [B,4,4] like the loader
    ref_intr = intr.clone(); ref_intr[:, 0, 2] += torch.tensor([3.5, -2.25])
    tf_x = torch.tensor([-410.0, 395.5])
    mask = torch.tensor((rng.uniform(size=(B, 3, S, S)) > 0.4).astype(np.float64))
    flow = torch.tensor(rng.uniform(-60, -20, (B, 1, S, S)), requires_grad=True)
    data = {"ref_intr": ref_intr, "intr": intr, "flow_pred": flow, "Tf_x": tf_x, "mask": mask}
    depth = flow2depth(data)
    xyz = depth2pc(depth, extr, intr).view(B, -1, 3)
    valid = (depth != 0.0).view(B, -1)
    g = torch.tensor(rng.standard_normal((B, S * S, 3)))
    gd = torch.tensor(rng.standard_normal((B, 1, S, S)))
    ((xyz * g).sum() + (depth * gd).sum()).backward()
    np.savez_compressed(os.path.join(HERE, "unproject_golden.npz"), flow=flow.detach().numpy(), mask=mask.numpy(),
                        intr=intr.numpy(), extr=extr.numpy(), ref_intr=ref_intr.numpy(), tf_x=tf_x.numpy(),
                        depth=depth.detach().numpy(), xyz=xyz.detach().numpy(), valid=valid.numpy(), g_xyz=g.numpy(),
                        g_depth=gd.numpy(), d_flow=flow.grad.numpy())
    print("wrote unproject_golden.npz", xyz.shape, int(valid.sum()))


if __name__ == "__main__":
    main()
