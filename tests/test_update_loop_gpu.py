"""GPU: the disparity update block (csrc/update_block.cu through gps_gaussian_b200.update) on every iteration of the real
loop, per element, and the kernels' bit-for-bit properties.

`make_update_forward` runs on the reference's own FlowUpdateModule with `update.step` wrapped.  Before each step the
wrapper fills every workspace region but h, and the mask buffer, with NaN (h too on the first step): inside a step only
h and coords1 are read before they are written, so nothing else can carry over from the previous iteration.  After the
step every stage is checked per element from the kernels' own inputs to it (oracle/update_torch64.py's stage checks,
with h_in the NCHW net on the first step and the carried NHWC h after it), and the worst ratio per stage goes to
$GPSG_PARITY_LOG, one record per iteration.  Cases: the stage-2 eval shape 128 x 128 at B = 2 and 4 in test mode (mask on
the last iteration only) and train mode (mask on every one), 12 iterations, flow_init, the fp16 corr of
CorrBlockFast1D beside the fp32 one of CorrBlock1D, 256 x 256 (several units per CTA), widths on both sides of the
64-column tile (63, 64, 65, 128, 129) at heights 1, 2, 3 (the 2-row tile), and 96 x 160.

Each (tile, N-block) unit sums its K chunks in a fixed order whichever CTA runs it, so the following hold bit for bit
(fp16 regions and the mask compared as int16, coords1 as int32): a step carrying h from the previous one equals a fresh
poisoned workspace given that h as net; a B = 4 step equals each sample run alone, also with NaN and +-inf in one
sample's net, corr, coords1 and context at its first and last rows and on the 63 | 64 column seam (where the other
samples still equal their solo runs and the poisoned one's NaN positions are fp64's); cz / cr / cq split from a wider
context equal the packed run; an fp32 corr of fp16 values equals the fp16 corr; and a step with the mask head equals
one without it on everything else."""
import types

import pytest
import torch

from helpers import record
from gps_gaussian_b200 import harness, update
from oracle import update_torch64 as ut

pytestmark = pytest.mark.gpu
needs_ref = pytest.mark.skipif(harness.staged_reference() is None, reason="oracle/_ref not staged")
NAN = float("nan")


@pytest.fixture(autouse=True)
def poisoned_outputs(monkeypatch):
    """torch.empty inside update returns NaN-filled floating buffers and 0xFF-filled bytes (NaN in every fp16 view of
    the workspace), so an element the kernels skip shows."""
    def nan(fn):
        def make(*a, **k):
            t = fn(*a, **k)
            if t.is_floating_point():
                t.fill_(NAN)
            elif t.dtype == torch.uint8:
                t.fill_(0xFF)
            return t
        return make
    fake = types.SimpleNamespace(**{n: getattr(torch, n) for n in dir(torch) if not n.startswith("__")})
    fake.empty, fake.empty_like = nan(torch.empty), nan(torch.empty_like)
    monkeypatch.setattr(update, "torch", fake)


def params(seed):
    """Conv2d's default init: weights and biases uniform in +-1/sqrt(fan_in), fp32."""
    g = torch.Generator().manual_seed(seed)
    out = []
    for i, s in enumerate(update.PARAM_SHAPES):
        fan = update.PARAM_SHAPES[i - (i % 2)]
        k = 1.0 / (fan[1] * fan[2] * fan[3]) ** 0.5
        out.append(((torch.rand(s, generator=g) * 2 - 1) * k).float())
    return out


# ---- every iteration of the loop, per element ------------------------------------------------------------------------

class CheckedStep:
    """`update.step` with the workspace poisoned before and every stage checked after each call."""

    def __init__(self, tag, module):
        self.tag, self.real, self.worst = tag, update.step, []
        self.ps = [p.detach() for p in update.params_of(module.update_block)]

    def __call__(self, corr, coords1, net, czrq, czrq_bs, packed, ws, mask=None):
        B, _, H, W = coords1.shape
        reg = update.regions(ws, B, H, W)
        h_in = (net if net is not None else reg["h"].permute(0, 3, 1, 2)).float()
        for k, v in reg.items():
            if k != "h" or net is not None:
                v.fill_(NAN)
        if mask is not None:
            mask.fill_(NAN)
        corr_in, coords_in = corr.float(), coords1.clone()
        self.real(corr, coords1, net, czrq, czrq_bs, packed, ws, mask)
        r = {k: v.permute(0, 3, 1, 2).float() for k, v in reg.items()}
        got = dict(h_in=h_in, corr=corr_in, coords1_in=coords_in, x=r["x"], cf1=r["cf1"], cf2=r["cf2"], z=r["z"],
                   rh=r["rh"], h=r["h"], fh1=r["hid"][:, :256], delta=r["delta"], coords1=coords1.clone(),
                   czrq=torch.as_strided(czrq, (B, 3 * ut.HID, H, W), (czrq_bs, H * W, W, 1)))
        if mask is not None:
            got["m1"], got["mask"] = r["hid"][:, 256:], mask.float()
        chk = ut.stage_checks(self.ps, got)
        worst = {k: ut.ratio(got[k], *chk[k]) for k in chk}
        record(f"update_loop:{self.tag}:iter{len(self.worst)}", **worst)
        self.worst.append(worst)


def _args(**kw):
    a = types.SimpleNamespace(mixed_precision=True, n_gru_layers=1, slow_fast_gru=None, hidden_dims=[96, 96, 96],
                              corr_levels=4, corr_radius=4, n_downsample=3, corr_implementation="reg")
    for k, v in kw.items():
        setattr(a, k, v)
    return a


def _loop(monkeypatch, tag, B, H, W, iters=3, test_mode=True, flow_init=False, corr="reg", seed=0):
    harness.add_reference_to_path()
    import core.raft_stereo_human as rsh
    torch.manual_seed(seed)
    m = rsh.FlowUpdateModule(_args(corr_implementation=corr)).cuda().eval()
    g = torch.Generator().manual_seed(seed + 1)
    f1, f2 = (torch.randn(B, 64, H, W, generator=g).half().cuda() for _ in range(2))
    net = torch.tanh(torch.randn(B, 96, H, W, generator=g)).half().cuda()
    ctx = (torch.randn(B, 288, H, W, generator=g) * 0.7).half().cuda()
    fi = None
    if flow_init:
        fi = (torch.randn(B, 2, H, W, generator=g) * 2).cuda()
        fi[:, 1] = 0
    chk = CheckedStep(tag, m)
    monkeypatch.setattr(update, "step", chk)
    update.reset_update_counts()
    with torch.no_grad():
        out = update.make_update_forward(rsh.FlowUpdateModule.__dict__["forward"])(
            m, f1, f2, [net.clone()], [list(ctx.split(96, 1))], iters, fi, test_mode)
    assert update.update_counts() == {"steps": iters, "forwards": 1}
    assert len(chk.worst) == iters
    for i, w in enumerate(chk.worst):
        assert ("mask" in w) == (not test_mode or i == iters - 1), (i, sorted(w))
    print(f"{tag}: worst per stage over {iters} iterations",
          {k: max(w.get(k, 0.0) for w in chk.worst) for k in ut.KEYS})
    bad = [(i, w) for i, w in enumerate(chk.worst) if max(w.values()) > 1.0]
    assert not bad, bad
    return out


@needs_ref
@pytest.mark.parametrize("test_mode", [True, False], ids=["test", "train"])
@pytest.mark.parametrize("B", [2, 4])
def test_loop_stage2_shape(monkeypatch, B, test_mode):
    _loop(monkeypatch, f"b{B}_128_{'test' if test_mode else 'train'}", B, 128, 128, test_mode=test_mode, seed=B)


@needs_ref
def test_loop_twelve_iterations(monkeypatch):
    _loop(monkeypatch, "b2_128_iters12", 2, 128, 128, iters=12, seed=12)


@needs_ref
def test_loop_flow_init(monkeypatch):
    _loop(monkeypatch, "b2_128_flow_init", 2, 128, 128, test_mode=False, flow_init=True, seed=5)


@needs_ref
def test_loop_fp16_corr(monkeypatch):
    """"reg_cuda": CorrBlockFast1D's fp16 lookup (every other case runs "reg", CorrBlock1D's fp32 one)."""
    _loop(monkeypatch, "b2_128_reg_cuda", 2, 128, 128, test_mode=False, corr="reg_cuda", seed=7)


@needs_ref
def test_loop_256(monkeypatch):
    _loop(monkeypatch, "b2_256", 2, 256, 256, seed=9)


EDGE_SHAPES = [(H, W) for H in (1, 2, 3) for W in (63, 64, 65, 128, 129)] + [(96, 160)]


@needs_ref
@pytest.mark.parametrize("shape", EDGE_SHAPES, ids=lambda s: "x".join(map(str, s)))
def test_loop_tile_edges(monkeypatch, shape):
    H, W = shape
    _loop(monkeypatch, f"b2_{H}x{W}", 2, H, W, test_mode=False, seed=H * W)


# ---- bit for bit ----------------------------------------------------------------------------------------------------

def _inputs(B, H, W, seed, corr_dtype=torch.float16):
    g = torch.Generator().manual_seed(seed)
    corr = (torch.randn(B, 36, H, W, generator=g) * 2).half().to(corr_dtype)
    ys, xs = torch.meshgrid(torch.arange(H, dtype=torch.float32), torch.arange(W, dtype=torch.float32), indexing="ij")
    coords1 = torch.stack([xs, ys])[None] + torch.randn(B, 2, H, W, generator=g) * 3
    net = torch.tanh(torch.randn(B, 96, H, W, generator=g)).half()
    czrq = (torch.randn(B, 288, H, W, generator=g) * 0.7).half()
    return {k: v.cuda() for k, v in dict(corr=corr, coords1=coords1.float(), net=net, czrq=czrq).items()}


def _workspace(B, H, W):
    ws = update.workspace(B, H, W, torch.device("cuda"))
    ws.fill_(0xFF)
    return ws


def _step(packed, inp, net="net", ws=None, mask=True, czrq=None, bs=None):
    """One step; returns {region / coords1 / mask: integer view} and the workspace.  net=None carries h in ws."""
    B, _, H, W = inp["coords1"].shape
    ws = _workspace(B, H, W) if ws is None else ws
    c1 = inp["coords1"].clone()
    mk = torch.full((B, update.MASK_C, H, W), NAN, dtype=torch.float16, device="cuda") if mask else None
    czrq = inp["czrq"] if czrq is None else czrq
    update.step(inp["corr"], c1, inp[net] if net else None, czrq, czrq.stride(0) if bs is None else bs, packed, ws, mk)
    out = {k: v.permute(0, 3, 1, 2).contiguous().view(torch.int16) for k, v in update.regions(ws, B, H, W).items()}
    if not mask:
        out["hid"] = out["hid"][:, :256]
    out["coords1"] = c1.view(torch.int32)
    if mask:
        out["mask"] = mk.view(torch.int16)
    return out, ws


def _assert_bits(a, b, what, keys=None):
    for k in keys or a:
        assert torch.equal(a[k], b[k]), (what, k, int((a[k] != b[k]).sum()))


SHAPES = [(2, 128, 128), (3, 7, 130)]


@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "x".join(map(str, s)))
def test_carry_identity(shape):
    """Step 2 on the workspace step 1 left (net=None) equals a fresh poisoned workspace given step 1's h as net."""
    B, H, W = shape
    packed = update.pack([p.cuda() for p in params(1)])
    first = _inputs(B, H, W, 1)
    out1, ws = _step(packed, first)
    second = _inputs(B, H, W, 2)
    second["coords1"] = out1["coords1"].view(torch.float32).clone()
    second["h1"] = out1["h"].view(torch.float16).contiguous()
    carried, _ = _step(packed, second, net=None, ws=ws)
    fresh, _ = _step(packed, second, net="h1")
    _assert_bits(carried, fresh, "carry")
    # and a third step, without the mask head on the carried workspace
    third = dict(second, coords1=carried["coords1"].view(torch.float32).clone(),
                 h2=carried["h"].view(torch.float16).contiguous())
    carried, _ = _step(packed, third, net=None, ws=ws, mask=False)
    fresh, _ = _step(packed, third, net="h2", mask=False)
    _assert_bits(carried, fresh, "carry, no mask")


def _sample(inp, b):
    return {k: v[b:b + 1].contiguous() for k, v in inp.items()}


POISON = [("net", 5, "first", 63, NAN), ("net", 40, "last", 64, float("inf")), ("corr", 3, "first", 64, -float("inf")),
          ("corr", 20, "last", 63, NAN), ("coords1", 0, "first", 63, float("inf")), ("coords1", 1, "last", 64, NAN),
          ("czrq", 10, "first", 64, NAN), ("czrq", 130, "last", 63, -float("inf")), ("czrq", 250, 3, 0, float("inf"))]


def test_batch_independence():
    """A B = 4 step equals each sample alone at B = 1; with NaN / +-inf in sample 1 the others still do, and sample 1's
    NaN positions are fp64's under the stage checks."""
    B, H, W = 4, 7, 130
    ps = params(3)
    packed = update.pack([p.cuda() for p in ps])
    inp = _inputs(B, H, W, 3)
    whole, _ = _step(packed, inp)
    solo = [_step(packed, _sample(inp, b))[0] for b in range(B)]
    for b in range(B):
        _assert_bits({k: v[b:b + 1] for k, v in whole.items()}, solo[b], f"sample {b}")
    bad = {k: v.clone() for k, v in inp.items()}
    for name, c, row, col, v in POISON:
        y = 0 if row == "first" else H - 1 if row == "last" else row
        bad[name][1, c, y, col] = v
    got = update.step_with_workspace(bad["corr"], bad["coords1"], bad["net"], bad["czrq"], [p.cuda() for p in ps])
    poisoned, _ = _step(packed, bad)
    for b in (0, 2, 3):
        _assert_bits({k: v[b:b + 1] for k, v in poisoned.items()}, solo[b], f"sample {b} beside a non-finite sample 1")
    assert not torch.isfinite(got["h"][1]).all()
    got["czrq"] = bad["czrq"]
    chk = ut.stage_checks(ps, got)
    worst = {k: ut.ratio(got[k], *chk[k]) for k in chk}
    record("update_loop:non_finite_sample", **worst)
    assert max(worst.values()) <= 1.0, worst


@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "x".join(map(str, s)))
def test_context_stride(shape):
    """cz / cr / cq split from channels 32 .. 319 of a [B,384,H,W] tensor give the packed [B,288,H,W] run's bits."""
    B, H, W = shape
    packed = update.pack([p.cuda() for p in params(4)])
    inp = _inputs(B, H, W, 4)
    g = torch.Generator().manual_seed(40)
    wide = torch.randn(B, 384, H, W, generator=g).half().cuda()
    wide[:, 32:320] = inp["czrq"]
    view = wide[:, 32:320]
    assert update.czrq_stride(list(view.split(96, 1)), B, H, W) == 384 * H * W
    _assert_bits(_step(packed, inp, czrq=view)[0], _step(packed, inp)[0], "context stride")


def test_fp32_corr_of_fp16_values():
    B, H, W = 2, 9, 70
    packed = update.pack([p.cuda() for p in params(5)])
    inp = _inputs(B, H, W, 5)
    _assert_bits(_step(packed, dict(inp, corr=inp["corr"].float()))[0], _step(packed, inp)[0], "fp32 corr")


@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "x".join(map(str, s)))
def test_mask_head_is_additive(shape):
    B, H, W = shape
    packed = update.pack([p.cuda() for p in params(6)])
    inp = _inputs(B, H, W, 6)
    with_mask, _ = _step(packed, inp)
    without, _ = _step(packed, inp, mask=False)
    with_mask["hid"] = with_mask["hid"][:, :256]
    _assert_bits(with_mask, without, "mask head", keys=("h", "x", "cf1", "cf2", "z", "rh", "hid", "delta", "coords1"))
