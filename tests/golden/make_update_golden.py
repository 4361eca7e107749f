"""Generate tests/golden/update_golden.npz from the REFERENCE's own BasicMultiUpdateBlock and FlowUpdateModule
(core/update.py, core/raft_stereo_human.py).

Run with GPSG_REFERENCE naming a checkout of the original project:  python tests/golden/make_update_golden.py
The parameters and inputs are tests/update_cases.py's closed-form values (exact in fp16, fp32 and fp64), so the file
holds only outputs.  Everything runs in fp64 on the CPU with corr_implementation 'reg' (pure torch):
  step_<B>x<H>x<W>_{h,delta,mask}   one BasicMultiUpdateBlock iteration on update_cases.inputs(B, H, W)
  loop_{flow_up,pred0,pred1,pred2}  FlowUpdateModule.forward on update_cases.fmaps, three iterations, test mode and not
FlowUpdateModule.forward casts the fmaps to fp32 for 'reg' and builds coords0 / coords1 with coords_grid in fp32; the
generator runs it with a CorrBlock1D that casts the (fp32-exact) fmaps back to fp64 and with coords_grid in fp64, so the
only fp32 step left is the lookup's own `.float()` of its output, which oracle/update_torch64.loop64 restates.  Outputs
are stored in fp32 (the tests compare against the fp64 restatement at 1e-6 of each output's range).
"""
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.environ["GPSG_REFERENCE"])
import update_cases as uc  # noqa: E402
import core.raft_stereo_human as rsh  # noqa: E402
from core.update import BasicMultiUpdateBlock  # noqa: E402

F64 = torch.float64


def args():
    return types.SimpleNamespace(mixed_precision=False, n_gru_layers=1, slow_fast_gru=None, hidden_dims=[96, 96, 96],
                                 corr_levels=4, corr_radius=4, n_downsample=3, corr_implementation="reg")


def load(block):
    with torch.no_grad():
        e, g, f = block.encoder, block.gru08, block.flow_head
        mods = (e.convc1, e.convc2, e.convf1, e.convf2, e.conv, g.convz, g.convr, g.convq, f.conv1, f.conv2,
                block.mask[0], block.mask[2])
        ps = uc.params(0)
        for i, m in enumerate(mods):
            m.weight.copy_(ps[2 * i])
            m.bias.copy_(ps[2 * i + 1])


class CorrBlock1D64(rsh.CorrBlock1D):
    def __init__(self, fmap1, fmap2, **kw):
        super().__init__(fmap1.to(F64), fmap2.to(F64), **kw)

    def __call__(self, coords):
        return super().__call__(coords).to(F64)      # the reference's lookup returns .float(): rounded to fp32


def coords_grid64(batch, ht, wd):
    ys, xs = torch.meshgrid(torch.arange(ht, dtype=F64), torch.arange(wd, dtype=F64), indexing="ij")
    return torch.stack([xs, ys])[None].repeat(batch, 1, 1, 1)


def main():
    out = {}
    a = args()
    blk = BasicMultiUpdateBlock(a, hidden_dims=a.hidden_dims).to(F64)
    load(blk)
    with torch.no_grad():
        for B, H, W in uc.STEP_CASES:
            inp = uc.inputs(B, H, W)
            flow = inp["coords1"] - coords_grid64(B, H, W)
            net, mask, delta = blk([inp["net"]], [list(inp["czrq"].split(96, 1))], inp["corr"], flow,
                                   iter32=False, iter16=False)
            tag = f"step_{B}x{H}x{W}_"
            out[tag + "h"], out[tag + "delta"], out[tag + "mask"] = net[0], delta, mask
        rsh.CorrBlock1D, rsh.coords_grid = CorrBlock1D64, coords_grid64
        m = rsh.FlowUpdateModule(a).to(F64)
        load(m.update_block)
        B, H, W, iters = uc.LOOP_CASE
        f1, f2 = uc.fmaps(B, H, W)
        inp = uc.inputs(B, H, W)
        run = lambda test_mode: m(f1, f2, [inp["net"]], [list(inp["czrq"].split(96, 1))], iters, None, test_mode)
        out["loop_flow_up"] = run(True)
        for i, p in enumerate(run(False)):
            out[f"loop_pred{i}"] = p
    np.savez_compressed(os.path.join(HERE, "update_golden.npz"),
                        **{k: v.to(torch.float32).numpy() for k, v in out.items()})


if __name__ == "__main__":
    main()
