"""Generate tests/golden/flow_head_golden.npz from the REFERENCE's own FlowUpdateModule.upsample_flow and
lib.loss.sequence_loss.

Run with GPSG_REFERENCE naming a checkout of the original project:  python tests/golden/make_flow_head_golden.py
Runs both on the CPU on seeded inputs.  Upsampling cases `up_<name>_*`: inputs, output, and the autograd gradients of flow
and mask for a random upstream gradient on every output channel.  Sequence-loss cases `sl_<name>_*`: inputs (fp32), the
loss, metrics and prediction gradients of the fp32 run and of an fp64 run on the same values, or the exception raised.
"""
import os
import sys
import types

import numpy as np
import torch

sys.path.insert(0, os.environ["GPSG_REFERENCE"])
from core.raft_stereo_human import FlowUpdateModule  # noqa: E402
from lib.loss import sequence_loss  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))

# name: (f, N, D, H, W, flow dtype, mask dtype, logit scale, special)
UPSAMPLE = {
    "f8_f64": (8, 1, 2, 4, 5, torch.float64, torch.float64, 3.0, None),
    "f4_w1_f64": (4, 1, 2, 6, 1, torch.float64, torch.float64, 3.0, None),
    "f2_d1_f64": (2, 2, 1, 3, 4, torch.float64, torch.float64, 3.0, None),
    "f8_f32": (8, 1, 2, 3, 6, torch.float32, torch.float32, 3.0, None),
    "f8_f16": (8, 2, 2, 3, 4, torch.float32, torch.float16, 3.0, None),
    "f4_large_f32": (4, 1, 2, 3, 5, torch.float32, torch.float32, 60.0, "large"),
    "f2_nonfinite_f32": (2, 1, 2, 3, 4, torch.float32, torch.float32, 3.0, "nonfinite"),
    "f4_nonfinite_f16": (4, 1, 2, 3, 4, torch.float32, torch.float16, 3.0, "nonfinite"),
}


def upsample_case(rng, f, N, D, H, W, fdt, mdt, scale, special):
    flow = rng.uniform(-20, 5, (N, D, H, W))
    flow[:, 1:] = rng.uniform(-3, 3, flow[:, 1:].shape)           # a non-zero y channel
    mask = rng.standard_normal((N, 9 * f * f, H, W)) * scale
    if special == "large":
        mask += 50.0                                               # exp overflows in fp32 without the max subtraction
    if special == "nonfinite":
        mv = mask.reshape(N, 9, f * f, H, W)
        mv[0, :, 0, 0, 0] = -np.inf                                # all 9 taps -inf -> NaN
        mv[0, 4, 1, 0, 1] = np.inf                                 # one +inf -> NaN
        mv[0, 2, 2, 1, 0] = np.nan                                 # one NaN -> NaN
        mv[0, :5, 3 % (f * f), 1, 2] = -np.inf                     # some -inf among finite logits: weight 0
    flow_t = torch.tensor(flow, dtype=fdt, requires_grad=True)
    mask_t = torch.tensor(mask, dtype=mdt, requires_grad=True)
    me = types.SimpleNamespace(args=types.SimpleNamespace(n_downsample=int(np.log2(f))))
    out = FlowUpdateModule.upsample_flow(me, flow_t, mask_t)
    g = torch.tensor(rng.standard_normal(tuple(out.shape)), dtype=out.dtype)
    (out * g).sum().backward()
    return dict(factor=np.int64(f), flow=flow_t.detach().numpy(), mask=mask_t.detach().numpy(), out=out.detach().numpy(),
                g=g.numpy(), d_flow=flow_t.grad.numpy(), d_mask=mask_t.grad.numpy())


# name: (P, N, H, W, valid fraction, special)
SEQLOSS = {
    "p3": (3, 2, 8, 9, 0.6, None),
    "p2_ties": (2, 1, 7, 5, 0.7, "ties"),
    "p3_inf_outside": (3, 2, 4, 6, 0.5, "inf_outside"),
    "p3_empty": (3, 1, 4, 4, 0.0, None),
    "p2_inf_inside": (2, 1, 4, 4, 0.8, "inf_inside"),
    "p1": (1, 1, 4, 4, 0.8, None),
}


def seqloss_case(rng, P, N, H, W, frac, special):
    gt = rng.uniform(-40, 0, (N, 1, H, W)).astype(np.float32)
    valid = rng.uniform(size=(N, 1, H, W)).astype(np.float32)
    valid = np.where(valid < frac, valid * 0.5 / max(frac, 1e-9) + 0.5, valid * 0.49).astype(np.float32)
    if frac == 0.0:
        valid[:] = 0.25
    valid.reshape(-1)[:2] = [0.5, np.nextafter(np.float32(0.5), np.float32(0))]     # the threshold itself, both sides
    preds = [(gt + rng.normal(0, 3.0 / (i + 1), gt.shape)).astype(np.float32) for i in range(P)]
    if special == "ties":
        for p in preds:
            p.reshape(-1)[::3] = gt.reshape(-1)[::3]
        preds[-1].reshape(-1)[1::4] = gt.reshape(-1)[1::4] + np.float32(1.0)       # EPE exactly 1
        preds[-1].reshape(-1)[2::4] = gt.reshape(-1)[2::4] - np.float32(3.0)       # EPE exactly 3 (up to rounding)
    if special == "inf_outside":
        gt[valid < 0.5] = np.inf
    if special == "inf_inside":
        gt.reshape(-1)[np.flatnonzero(valid.reshape(-1) >= 0.5)[0]] = -np.inf
    rec = dict(gt=gt, valid=valid, preds=np.stack(preds), g=np.float32(rng.uniform(0.5, 2.0)))
    for tag, dt in (("f32", torch.float32), ("f64", torch.float64)):
        ps = [torch.tensor(p, dtype=dt, requires_grad=True) for p in preds]
        try:
            loss, metrics = sequence_loss(ps, torch.tensor(gt, dtype=dt), torch.tensor(valid, dtype=dt))
        except (AssertionError, ZeroDivisionError) as e:
            rec["raises"] = type(e).__name__
            return rec
        (loss * float(rec["g"])).backward()
        rec[f"loss_{tag}"] = loss.detach().numpy()
        rec[f"metrics_{tag}"] = np.array([metrics["train_epe"], metrics["train_1px"], metrics["train_3px"]])
        rec[f"grads_{tag}"] = np.stack([p.grad.numpy() for p in ps])
    rec["raises"] = ""
    return rec


def main():
    rng = np.random.default_rng(2024)
    out = {}
    for name, spec in UPSAMPLE.items():
        for k, v in upsample_case(rng, *spec).items():
            out[f"up_{name}_{k}"] = v
    for name, spec in SEQLOSS.items():
        for k, v in seqloss_case(rng, *spec).items():
            out[f"sl_{name}_{k}"] = v
    np.savez_compressed(os.path.join(HERE, "flow_head_golden.npz"), **out)
    print("wrote flow_head_golden.npz:", len(UPSAMPLE), "upsampling cases,", len(SEQLOSS), "sequence-loss cases")


if __name__ == "__main__":
    main()
