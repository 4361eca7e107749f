"""Independent fp64 torch restatement of the disparity head (TEST INFRASTRUCTURE ONLY), with per-element error bounds.

`upsample_flow64(flow, mask, f)` is the convex upsampling of `FlowUpdateModule.upsample_flow` (reference
core/raft_stereo_human.py) in differentiable torch: the mask viewed as [N,1,9,f,f,H,W], softmax over the 9 taps, the
3x3 `F.unfold` of f*flow with zero padding 1, the product summed over the taps, then the permute to [N,D,f*H,f*W].  In
fp64 on the exact device inputs (fp16 masks widen exactly) it is the maths; `forward_and_grads` takes dL/dflow and
dL/dmask from autograd.  It runs on the CPU or on CUDA.  `sequence_loss64` is lib/loss.py's sequence loss in fp64 on
the fp32 differences p - gt the kernel forms.

Bounds.  u = 2^-24, gamma(n) = n u / (1 - n u).  Per fine pixel, tap k: w_k the fp64 weight, dm_k = |m_k - max m|,
U_{d,k} = f * flow at the tap, g_d = dL/dout.  csrc/flow_head.cu computes in fp32 with __fmul_rn / __fadd_rn (no FMA):

  weights     e_k = expf(m_k - mx): the subtraction rounds by dm_k u relative in the argument, expf adds 2 ulp (4u), so
              |de_k| <= (4 + dm_k) u e_k.  The 9-term sum adds 8 roundings and sum_j w_j (4 + dm_j) u <= (4 + 8/e) u
              (w_j dm_j <= dm_j e^-dm_j <= 1/e), the division one more:
                  err_w(k) = w_k gamma(C_W + dm_k) + 2^-126,      C_W = 4 + 8 + 2.95 + 1 -> 16
              (2^-126 covers subnormal weights).  fp16 masks round the fp32 weight to fp16, by at most half an fp16
              ulp of it: + max(2^-11 (w_k + err_w32(k)), 2^-25).
  out         sum_k fl(w_k U_k) in tap order: 9 roundings on each term (1 product, 8 additions):
                  |out - out64| <= sum_k |U_k| err_w(k) + gamma(C_S) sum_k w_k |U_k|,      C_S = 9
  dL/dmask    dW_k = round_T(g_0 U_0k + g_1 U_1k) (2 roundings on a_k = sum_d |g_d U_dk|), s = sum_k fl(dW_k w_k)
              (9 roundings on sum_j w_j a_j, plus 2 from dW), fl(dW_k - s) and the product (2 on w_k |dW_k - s|):
                  err_w(k) |dW_k - s| + (w_k + err_w(k)) E_k,
                  E_k = sum_j err_w(j) |dW_j| + gamma(C_D) (a_k + sum_j w_j a_j + |dW_k - s|),      C_D = 2 + 9 + 2 -> 13
              (the product multiplies the error of the difference by the computed weight, hence w_k + err_w(k)).
              fp16 masks round the fp32 dW to fp16, by r_k = 2^-11 (|dW_k| + gamma(2) a_k) + 2^-25 at most, which adds
              r_k + sum_j (w_j + err_w(j)) r_j to E_k, and round the fp32 result B to fp16: + 2^-11 (w_k |dW_k - s| + B)
              + 2^-25.  Rounding dW to the mask dtype is the op chain's own deviation from the maths (its softmax
              backward runs on the fp16 grad).
  dL/dflow    f * sum_k TS_k(y+1-ky, x+1-kx), TS_k = sum_i sum_j fl(w_k g): a term passes 1 product, f-1 additions
              over j, f-1 over i and 8 over the taps (x f is exact):
                  f (sum err_w |g| + gamma(C_T (2f + 7)) sum w |g|)  over the terms that feed the coarse pixel, C_T = 1.
  underflow   a product below the fp32 subnormal range rounds to 0 or 2^-149: every bound has an absolute floor TINY =
              2^-140, which covers up to 512 such roundings and nothing a formula error could hide in.
  NaN         out, dL/dmask and dL/dflow are NaN exactly where fp64 autograd is: a NaN logit, a +inf logit or 9 -inf
              logits make the fine pixel's weights NaN (the kernel header spells this out).
  loss        m_i = fl(float(S_i) * fl(1 / float(c))) with S_i the fp64 partial sums of |d| (error < 2^-40 u relative at
              the kernel's summation depth) and c the valid count: float(S_i), float(c) (exact up to 2^24), the
              reciprocal and the product are 4 roundings, the weight product 1, and the fp32 sum over P predictions
              adds up to P - 1 more on a sum of positive terms:  |loss - loss64| <= gamma(P + 4) |loss64|.  The weights
              are the fp32 roundings of lib/loss.py's Python floats, as the op chain multiplies by them.
  EPE         fl(sqrt(fl(d d))) is within 1.5 u of |d|, then the same 4 roundings: 5.5 u <= gamma(P + 4) for P >= 2.
  fractions   exactly float(c1) * (1 / float(c)) in fp32, c1 and c the exact counts (ep < 1, ep < 3 on the fp32 ep).

The constants were fixed from this derivation and checked on the CPU against oracle/flow_head_oracle.py with the
kernels' dtype boundaries over tests/flow_head_cases.py before any device run (tests/test_flow_head_torch64_cpu.py
prints the utilisation).
"""
import numpy as np
import torch
import torch.nn.functional as F

F64 = torch.float64
U = 2.0 ** -24
C_W = 16.0
C_S = 9.0
C_D = 13.0
C_T = 1.0
TINY = 2.0 ** -140


def gamma(n):
    return n * U / (1.0 - n * U)


def _fine(t, N, D, f, H, W):
    """[N,D,f*H,f*W] -> [N,D,f,f,H,W] (i, j, h, w)."""
    return t.reshape(N, D, H, f, W, f).permute(0, 1, 3, 5, 2, 4)


def _taps(flow, f):
    """[N,D,H,W] -> f*flow at the 9 taps, zero outside the image: [N,D,9,H,W] (tap k = 3*ky + kx)."""
    N, D, H, W = flow.shape
    return F.unfold(f * flow, [3, 3], padding=1).view(N, D, 9, H, W)


def upsample_flow64(flow, mask, f):
    """flow [N,D,H,W], mask [N,9f^2,H,W] -> [N,D,fH,fW], differentiable, in the inputs' dtype (pass fp64)."""
    N, D, H, W = flow.shape
    w = torch.softmax(mask.view(N, 1, 9, f, f, H, W), dim=2)
    up = _taps(flow, f).view(N, D, 9, 1, 1, H, W)
    out = torch.sum(w * up, dim=2)
    return out.permute(0, 1, 4, 2, 5, 3).reshape(N, D, f * H, f * W)


def forward_and_grads(flow, mask, f, g, need_flow=True, need_mask=True):
    """fp64 (out, dL/dflow, dL/dmask) by autograd of <upsample_flow64(flow, mask, f), g>, on the inputs' device; a
    gradient not asked for is None."""
    fl = flow.detach().to(F64).requires_grad_(need_flow)
    m = mask.detach().to(F64).requires_grad_(need_mask)
    out = upsample_flow64(fl, m, f)
    wrt = [t for t in (fl, m) if t.requires_grad]
    grads = torch.autograd.grad(out, wrt, g.detach().to(F64)) if wrt else ()
    it = iter(grads)
    dflow = next(it) if need_flow else None
    dmask = next(it) if need_mask else None
    return out.detach(), dflow, dmask


def upsample_terms(flow, mask, f, g):
    """The per-element magnitudes the bounds are made of, fp64, with [N,9,f,f,H,W] per fine pixel and tap:
    w, dm = |m - max m|, dW = sum_d g_d U_d and |dW|, a = sum_d |g_d U_d|; per fine pixel [N,1,f,f,H,W]:
    s = sum_k w dW, sw_dW = sum_k w |dW|, sw_a = sum_k w a; per channel [N,D,f,f,H,W]: wU = sum_k w |U|;
    per channel and coarse tap source [N,D,9,H,W]: ts_wg = sum_{i,j} w |g| (the magnitude of the tap sums)."""
    N, D, H, W = flow.shape
    with torch.no_grad():
        m = mask.to(F64).view(N, 9, f, f, H, W)
        w = torch.softmax(m, dim=1)
        dm = (m - m.amax(dim=1, keepdim=True)).abs()
        Ut = _taps(flow.to(F64), f)[:, :, :, None, None]                    # [N,D,9,1,1,H,W]
        G = _fine(g.to(F64), N, D, f, H, W)[:, :, None]                    # [N,D,1,f,f,H,W]
        dW = (G * Ut).sum(1)
        a = (G * Ut).abs().sum(1)
        t = dict(w=w, dm=dm, dW=dW, abs_dW=dW.abs(), a=a)
        t["s"] = (w * dW).sum(1, keepdim=True)
        t["sw_dW"] = (w * dW.abs()).sum(1, keepdim=True)
        t["sw_a"] = (w * a).sum(1, keepdim=True)
        t["wU"] = (w[:, None] * Ut.abs()).sum(2)
        t["ts_wg"] = (w[:, None] * G.abs()).sum((3, 4))
    return t


def weight_error(t, mask_dtype):
    """err_w per fine pixel and tap (see the module docstring); 0 where the weight is exactly 0 (a -inf tap)."""
    w = t["w"]
    e = torch.where(w > 0, w * gamma(C_W + t["dm"]), torch.zeros_like(w)) + 2.0 ** -126
    if mask_dtype == torch.float16:
        e = e + torch.clamp((w + e) * 2.0 ** -11, min=2.0 ** -25)     # half an fp16 ulp of the fp32 weight
    return e


def bounds(flow, mask, f, g, mask_dtype=None):
    """Per-element bounds {"out": [N,D,fH,fW], "dmask": [N,9f^2,H,W], "dflow": [N,D,H,W]} on the kernels' results for
    these inputs (mask_dtype defaults to the mask's)."""
    N, D, H, W = flow.shape
    mask_dtype = mask_dtype or mask.dtype
    t = upsample_terms(flow, mask, f, g)
    ew = weight_error(t, mask_dtype)
    with torch.no_grad():
        Ut = _taps(flow.to(F64), f)[:, :, :, None, None].abs()
        out = (Ut * ew[:, None]).sum(2) + gamma(C_S) * t["wU"]
        out = out.permute(0, 1, 4, 2, 5, 3).reshape(N, D, f * H, f * W)
        w, diff = t["w"], (t["dW"] - t["s"]).abs()
        err_diff = (ew * t["abs_dW"]).sum(1, keepdim=True) + gamma(C_D) * (t["a"] + t["sw_a"] + diff)
        if mask_dtype == torch.float16:
            # dW rounded to fp16: half an fp16 ulp of the fp32 dW, which is within gamma(2) a of dW
            dr = 2.0 ** -11 * (t["abs_dW"] + gamma(2) * t["a"]) + 2.0 ** -25
            err_diff = err_diff + dr + ((w + ew) * dr).sum(1, keepdim=True)
        dmask = ew * diff + (w + ew) * err_diff
        if mask_dtype == torch.float16:
            dmask = dmask + 2.0 ** -11 * (w * diff + dmask) + 2.0 ** -25   # half an fp16 ulp of the fp32 result
        dmask = dmask.reshape(N, 9 * f * f, H, W)
        G = _fine(g.to(F64), N, D, f, H, W).abs()[:, :, None]
        ts = (ew[:, None] * G).sum((3, 4)) + gamma(C_T * (2 * f + 7)) * t["ts_wg"]
        fold = F.fold(ts.reshape(N, D * 9, H * W), (H, W), 3, padding=1)
        dflow = f * fold
    return {"out": out + TINY, "dmask": dmask + TINY, "dflow": dflow + TINY}


def ratio(got, want, bound):
    """Worst |got - want| / bound over the elements where want is not NaN (0 where they agree exactly); inf when the
    NaN positions differ."""
    got = torch.as_tensor(got).to(device=want.device, dtype=F64).reshape(want.shape)
    nan = torch.isnan(want)
    if not torch.equal(torch.isnan(got), nan):
        return float("inf")
    err = (got - want).abs()
    r = torch.where(nan | (err == 0), torch.zeros_like(err), err / bound)
    return float(r.max()) if r.numel() else 0.0


def weights32(n_pred, gamma_=0.9):
    """lib/loss.py's prediction weights, rounded to fp32 as the op chain's `i_weight * tensor` rounds them."""
    g = gamma_ ** (15 / (n_pred - 1))
    return [float(np.float32(g ** (n_pred - i - 1))) for i in range(n_pred)]


def sequence_loss64(preds, gt, valid, gamma_=0.9, fp32_diff=True):
    """-> dict(loss, epe: fp64 0-dim tensors; c1, c3, count: ints) over v = valid >= 0.5, on the inputs' device.
    fp32_diff: the maths on the fp32 differences p - gt (the op chain's and the kernel's) with the fp32 weights; False:
    exact differences and the Python weights, which is lib/loss.py run in fp64."""
    v = valid >= 0.5
    if fp32_diff:
        d = [(p.float() - gt.float())[v].to(F64) for p in preds]
        w = weights32(len(preds), gamma_)
        ep32 = d[-1].float().mul(d[-1].float()).sqrt()
    else:
        d = [(p.to(F64) - gt.to(F64))[v] for p in preds]
        g = gamma_ ** (15 / (len(preds) - 1))
        w = [g ** (len(preds) - i - 1) for i in range(len(preds))]
        ep32 = d[-1].abs()
    n = int(v.sum())
    loss = sum(wi * di.abs().sum() / n for wi, di in zip(w, d))
    return {"loss": loss, "epe": d[-1].abs().sum() / n, "c1": int((ep32 < 1).sum()), "c3": int((ep32 < 3).sum()),
            "count": n}


def loss_bound(n_pred):
    """Relative bound on the loss and the EPE mean."""
    return gamma(n_pred + 4)


def fraction32(c, count):
    """float(c) * (1 / float(count)) in fp32, as a Python float."""
    return float(np.float32(c) * (np.float32(1) / np.float32(count)))
