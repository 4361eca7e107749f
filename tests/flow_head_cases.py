"""Seeded inputs for the disparity-head tests against oracle/flow_head_torch64.py, shared by the CPU and GPU files.

`SWEEP` is what tests/test_flow_head_fp64_gpu.py runs through the kernels; tests/test_flow_head_torch64_cpu.py runs the
fp32 emulation over it (at N = 1) and shows that each mutant of the emulation breaks a bound on one of its cases.
For every factor f the widths sit on both sides of one, two and three times each segment width (the forward's
TW = 512/f and the backward's TW = 256/f) and at 1, 2, 3, so multi-segment widths with W % 4 in {1, 2, 3} and ragged last
segments are all there; H, N and D cycle through {7, 1, 2}, {3, 1} and {2, 1}.  Both mask dtypes run every width.
`ALIGN` passes the mask, or the incoming gradient, as a view at an element offset of 1 or 2 into a larger buffer with
W % 4 == 0, so each side takes its scalar path while the other stays vectorised (an fp32 mask at offset 2 loads scalar in
the forward and in float2 vectors in the backward).  `STAGES` are the training shapes, `LOSS` the sequence-loss cases.
"""
import dataclasses

import numpy as np
import torch

FACTORS = (2, 4, 8)
DTYPES = {"f32": torch.float32, "f16": torch.float16}
LOGITS = ("normal", "large", "neginf", "nan")


@dataclasses.dataclass(frozen=True)
class Case:
    f: int
    N: int
    D: int
    H: int
    W: int
    dtype: str = "f32"
    logits: str = "normal"
    g: str = "ch1"                 # "ch1_zero": dL/dout channel 1 is 0, as training passes it
    needs: str = "both"            # "mask": flow without grad (grad_flow NULL); "flow": mask without grad
    mask_off: int = 0
    g_off: int = 0
    seed: int = 0

    @property
    def id(self):
        s = f"f{self.f}-{self.N}x{self.D}x{self.H}x{self.W}-{self.dtype}-{self.logits}"
        if self.D == 2:
            s += "-" + self.g
        if self.needs != "both":
            s += "-only_" + self.needs
        if self.mask_off or self.g_off:
            s += f"-moff{self.mask_off}-goff{self.g_off}"
        return s


def widths(f):
    fwd, bwd = 512 // f, 256 // f
    return sorted({1, 2, 3} | {m * tw + e for tw in (fwd, bwd) for m in (1, 2, 3) for e in (-1, 0, 1)})


def _sweep():
    cases, i = [], 0
    for f in FACTORS:
        for W in widths(f):
            for di, dt in enumerate(DTYPES):
                cases.append(Case(f, (3, 1)[(i // 3) % 2], (2, 1)[i % 2], (7, 1, 2)[i % 3], W, dt,
                                  LOGITS[(i + 2 * di) % 4], ("ch1_zero", "ch1")[(i // 2) % 2], seed=1000 + 2 * i + di))
            i += 1
    for j, (f, H, W) in enumerate(((8, 96, 160), (8, 160, 96), (4, 33, 200), (2, 7, 300))):
        for di, dt in enumerate(DTYPES):
            cases.append(Case(f, 1, 2, H, W, dt, ("normal", "large")[(j + di) % 2], "ch1_zero", seed=2000 + 2 * j + di))
    for j, dt in enumerate(DTYPES):
        cases.append(Case(2, 2, 2, 2, 257, dt, "neginf", "ch1", needs="mask", seed=2100 + j))
        cases.append(Case(4, 2, 1, 3, 129, dt, "nan", needs="flow", seed=2110 + j))
    return cases


def _align():
    cases = []
    for j, dt in enumerate(DTYPES):
        for off in (1, 2):
            cases.append(Case(4, 2, 2, 3, 132, dt, "normal", "ch1", mask_off=off, seed=3000 + 4 * j + off))
            cases.append(Case(8, 2, 2, 2, 68, dt, "neginf", "ch1_zero", g_off=off, seed=3010 + 4 * j + off))
    return cases


SWEEP = _sweep()
ALIGN = _align()
STAGES = [Case(8, 12, 2, 128, 128, "f32", "normal", "ch1_zero", seed=4000),
          Case(8, 4, 2, 128, 128, "f16", "normal", "ch1_zero", seed=4001)]


def inputs(case, n=None):
    """(flow fp32 [N,D,H,W], mask [N,9f^2,H,W] in the case's dtype, g fp32 [N,D,fH,fW]) as CPU tensors; n keeps only
    the first n batch elements (the same values as the full case's)."""
    rng = np.random.default_rng(case.seed)
    f, N, D, H, W = case.f, case.N, case.D, case.H, case.W
    flow = rng.uniform(-20, 5, (N, D, H, W))
    if D == 2:
        flow[:, 1] = rng.uniform(-3, 3, (N, H, W))
    m = rng.standard_normal((N, 9, f * f, H, W)) * 4.0
    if case.logits == "large":                 # every fine pixel's logits around one offset up to 1e4 (6e4 in fp16)
        big = 1e4 if case.dtype == "f32" else 6e4
        m += rng.uniform(-big, big, (N, 1, f * f, H, W))
    elif case.logits == "neginf":              # about 15 % of the taps at -inf: weight exactly 0
        m[rng.uniform(size=m.shape) < 0.15] = -np.inf
    elif case.logits == "nan":                 # one NaN, one +inf and one all -inf fine pixel in batch element 0
        p = rng.choice(f * f * H * W, 3, replace=False)
        ij, hw = np.unravel_index(p, (f * f, H * W))
        h, w = np.unravel_index(hw, (H, W))
        m[0, 2, ij[0], h[0], w[0]] = np.nan
        m[0, 4, ij[1], h[1], w[1]] = np.inf
        m[0, :, ij[2], h[2], w[2]] = -np.inf
    g = rng.standard_normal((N, D, f * H, f * W))
    if D == 2 and case.g == "ch1_zero":
        g[:, 1] = 0.0
    mask = m.reshape(N, 9 * f * f, H, W).astype(np.float16 if case.dtype == "f16" else np.float32)
    out = (torch.from_numpy(flow.astype(np.float32)), torch.from_numpy(mask), torch.from_numpy(g.astype(np.float32)))
    return out if n is None else tuple(t[:n].contiguous() for t in out)


# ---- sequence loss ----------------------------------------------------------------------------------------------------

@dataclasses.dataclass(frozen=True)
class LossCase:
    P: int
    N: int
    H: int
    W: int
    gt: str = "f32"
    valid: str = "half"            # "half": about half the pixels; "most": > 2^24 at N = 17, 1024^2, with an odd count
    seed: int = 0

    @property
    def id(self):
        return f"P{self.P}-{self.N}x{self.H}x{self.W}-gt_{self.gt}-valid_{self.valid}"


LOSS = [LossCase(3, 12, 1024, 1024, "f16", seed=5000), LossCase(3, 12, 1024, 1024, "f32", seed=5001),
        LossCase(3, 17, 1024, 1024, "f16", "most", seed=5002),
        LossCase(3, 1, 1, 255, seed=5011), LossCase(12, 1, 1, 256, "f16", seed=5012),
        LossCase(3, 1, 528, 256, seed=5013), LossCase(32, 1, 1, 528 * 256 + 1, "f16", seed=5014),
        LossCase(2, 2, 37, 69, "f16", seed=5015)]


def loss_inputs(case, n=None, device="cpu"):
    """(preds [P x fp32 [N,1,H,W]], gt fp32/fp16, valid fp32), generated on `device`; n caps the batch size.
    gt is inf outside the valid set, a seventh of the last prediction ties gt (sign 0), and a few of its EPEs are
    exactly 1 and 3."""
    N = case.N if n is None else min(n, case.N)
    gen = torch.Generator(device=device).manual_seed(case.seed)
    shape = (N, 1, case.H, case.W)
    gt = (torch.rand(shape, generator=gen, device=device) * -40).to(DTYPES[case.gt])
    valid = torch.rand(shape, generator=gen, device=device)
    if case.valid == "most":
        valid = (valid >= 0.01).float()
    valid.view(-1)[:2] = torch.tensor([0.5, float(np.nextafter(np.float32(0.5), np.float32(0)))])
    if case.valid == "most" and int((valid >= 0.5).sum()) % 2 == 0:   # an odd count: float(count) rounds above 2^24
        valid.view(-1)[int(torch.nonzero(valid.view(-1) < 0.5)[1])] = 1.0
    gt[valid < 0.5] = float("inf")
    fin = gt.float().nan_to_num(posinf=0.0)
    preds = [fin + torch.randn(shape, generator=gen, device=device) * (3.0 / (i + 1)) for i in range(case.P)]
    last = preds[-1].view(-1)
    last[::7] = fin.view(-1)[::7]
    last[1::11] = fin.view(-1)[1::11] + 1.0
    last[2::13] = fin.view(-1)[2::13] - 3.0
    return preds, gt, valid
