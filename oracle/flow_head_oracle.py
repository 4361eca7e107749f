"""numpy restatement of the disparity head from its maths (csrc/flow_head.cu; reference FlowUpdateModule.upsample_flow and
lib/loss.py's sequence_loss), used by the tests.

Convex upsampling with factor f, tap k = 3*ky + kx, mask channel k*f^2 + i*f + j:
    w[n,k,i,j,h,w]      = exp(m_k - max m) / sum_k exp(m_k - max m)              (softmax over the 9 taps)
    U[n,d,k,h,w]        = f * flow[n,d,h+ky-1,w+kx-1]                             (0 outside the image)
    out[n,d,h*f+i,w*f+j] = sum_k w * U
Backward with G[n,d,i,j,h,w] = dL/dout[n,d,h*f+i,w*f+j]:
    dW[k]    = sum_d G_d U_d[k];   dmask[k] = w[k] (dW[k] - sum_k' w[k'] dW[k'])
    TS[d,k]  = sum_{i,j} w[k] G_d; dflow[n,d,y,x] = f * sum_k TS[d,k](y+1-ky, x+1-kx)
`dtype=None` computes everything in fp64.  `dtype=np.float32 / np.float16` applies the dtype boundaries of the fused
kernels: weights computed in fp32 and rounded to that dtype, fp32 products summed in tap order, dW rounded to that dtype
before the softmax backward, dmask rounded to it.  That is the fp32 emulation the fp64 bounds of
oracle/flow_head_torch64.py were fixed against; `mutant=` (one of MUTANTS) makes it the kernel with that bug, so that
tests/test_flow_head_torch64_cpu.py can show each bug breaks a bound.

Sequence loss over predictions p_i, ground truth g and the mask v = (valid >= 0.5):
    loss = sum_i gamma'^(P-1-i) mean_v |p_i - g|,  gamma' = gamma^(15/(P-1))
    EPE  = |p_last - g| over v;  metrics = mean EPE, mean(EPE < 1), mean(EPE < 3)
    dloss/dp_i = gamma'^(P-1-i) sign(p_i - g) / |v| on v, 0 elsewhere.
"""
import numpy as np

# The bugs a kernel could have, for the emulation below (upsampling) and `sequence_loss_kernel` (the loss):
#   no_max_sub       softmax without subtracting the max logit
#   kx_ky_swapped    tap k read as 3*kx + ky instead of 3*ky + kx
#   clamped_taps     edge taps clamped to the image instead of zero-padded
#   ij_transposed    fine pixel (i, j) written (and its gradient read) at (j, i)
#   halo_fwd/_bwd    the taps at w0 - 1 and w0 + TW of a coarse row segment [w0, w0 + TW) read as 0, with the forward's
#                    TW = 512/f or the backward's TW = 256/f (the halo that stage_taps loads)
#   no_s             the softmax backward without its -s term
#   gather_flipped   dL/dflow gathered at y - 1 + ky instead of y + 1 - ky
#   no_f             dL/dflow without the factor f
#   all_pixels       the loss and the metrics divided by the pixel count instead of the valid count
#   epe_first        the EPE taken from the first prediction instead of the last
UPSAMPLE_MUTANTS = ("no_max_sub", "kx_ky_swapped", "clamped_taps", "ij_transposed", "halo_fwd", "halo_bwd", "no_s",
                    "gather_flipped", "no_f")
LOSS_MUTANTS = ("all_pixels", "epe_first")
FWD_TW = {2: 256, 4: 128, 8: 64}
BWD_TW = {2: 128, 4: 64, 8: 32}


def _softmax9(m, max_sub=True):
    """m [..., 9 on axis 1 ...]: softmax over axis 1 in the array's dtype, max-subtracted."""
    mx = m.max(axis=1, keepdims=True) if max_sub else np.zeros_like(m[:, :1])
    e = np.exp(m - mx)
    return e / e.sum(axis=1, keepdims=True)


def _taps(flow, f, dt, mutant=None):
    N, D, H, W = flow.shape
    fl = flow.astype(dt) * dt(f)
    pad = np.pad(fl, ((0, 0), (0, 0), (1, 1), (1, 1)), mode="edge" if mutant == "clamped_taps" else "constant")
    order = [(ky, kx) for kx in range(3) for ky in range(3)] if mutant == "kx_ky_swapped" else \
        [(ky, kx) for ky in range(3) for kx in range(3)]
    U = np.stack([pad[:, :, ky:ky + H, kx:kx + W] for ky, kx in order], axis=2)   # [N,D,9,H,W]
    if mutant in ("halo_fwd", "halo_bwd"):
        tw = (FWD_TW if mutant == "halo_fwd" else BWD_TW)[f]
        w = np.arange(W)
        U = U.copy()
        for k in range(9):
            lost = (w % tw == 0) if k % 3 == 0 else ((w + 1) % tw == 0) if k % 3 == 2 else np.zeros(W, bool)
            U[:, :, k, :, lost] = 0
    return U


def _weights(mask, f, dtype, mutant=None):
    N, _, H, W = mask.shape
    with np.errstate(invalid="ignore", over="ignore"):
        if dtype is None:
            return _softmax9(mask.astype(np.float64).reshape(N, 9, f, f, H, W))
        w = _softmax9(mask.astype(np.float32).reshape(N, 9, f, f, H, W), mutant != "no_max_sub")
        return w.astype(dtype).astype(np.float32)


def convex_upsample(flow, mask, f, dtype=None, mutant=None):
    """flow [N,D,H,W], mask [N,9f^2,H,W] -> out [N,D,fH,fW] (fp64 when dtype is None, else fp32)."""
    N, D, H, W = flow.shape
    dt = np.float64 if dtype is None else np.float32
    w = _weights(mask, f, dtype, mutant)                           # [N,9,f,f,H,W]
    U = _taps(flow, f, dt, None if mutant == "halo_bwd" else mutant)   # [N,D,9,H,W]
    out = np.zeros((N, D, f, f, H, W), dt)
    with np.errstate(invalid="ignore", over="ignore"):
        for k in range(9):
            out = out + w[:, None, k] * U[:, :, k, None, None]
    perm = (0, 1, 4, 3, 5, 2) if mutant == "ij_transposed" else (0, 1, 4, 2, 5, 3)
    return out.transpose(perm).reshape(N, D, f * H, f * W)


def convex_upsample_backward(flow, mask, f, grad_out, dtype=None, mutant=None):
    """-> (dflow [N,D,H,W], dmask [N,9f^2,H,W]) for dL/dout = grad_out."""
    N, D, H, W = flow.shape
    dt = np.float64 if dtype is None else np.float32
    w = _weights(mask, f, dtype, mutant)
    U = _taps(flow, f, dt, None if mutant == "halo_fwd" else mutant)
    perm = (0, 1, 5, 3, 2, 4) if mutant == "ij_transposed" else (0, 1, 3, 5, 2, 4)
    G = grad_out.astype(dt).reshape(N, D, H, f, W, f).transpose(perm)                    # [N,D,i,j,H,W]
    with np.errstate(invalid="ignore", over="ignore"):
        dW = np.zeros((N, 9, f, f, H, W), dt)
        for d in range(D):
            dW = dW + G[:, d, None] * U[:, d, :, None, None]
        if dtype is not None:
            dW = dW.astype(dtype).astype(np.float32)
        s = np.zeros((N, 1, f, f, H, W), dt)
        for k in range(9):
            s = s + dW[:, k:k + 1] * w[:, k:k + 1]
        dmask = w * dW if mutant == "no_s" else w * (dW - s)
        TS = (w[:, None] * G[:, :, None]).sum(axis=(3, 4))     # [N,D,9,H,W]
    dflow = np.zeros((N, D, H + 2, W + 2), dt)
    for k in range(9):
        ky, kx = divmod(k, 3)
        if mutant == "gather_flipped":
            ky = 2 - ky
        dflow[:, :, ky:ky + H, kx:kx + W] += TS[:, :, k]
    dflow = dflow[:, :, 1:-1, 1:-1]
    if mutant != "no_f":
        dflow = dflow * dt(f)
    out_dt = np.float64 if dtype is None else dtype
    return dflow, dmask.reshape(N, 9 * f * f, H, W).astype(out_dt)


def loss_weights(n_pred, gamma=0.9):
    g = gamma ** (15 / (n_pred - 1))
    return [g ** (n_pred - i - 1) for i in range(n_pred)]


def sequence_loss(preds, gt, valid, gamma=0.9):
    """fp64: (loss, {'train_epe', 'train_1px', 'train_3px'}, [dloss/dp_i], inf_in_valid)."""
    v = valid >= 0.5
    g = gt.astype(np.float64)
    inf = bool(np.isinf(g[v]).any())
    w = loss_weights(len(preds), gamma)
    n = int(v.sum())
    with np.errstate(invalid="ignore", divide="ignore"):
        means = [np.abs(p.astype(np.float64) - g)[v].sum() / n if n else np.nan for p in preds]
        loss = sum(wi * m for wi, m in zip(w, means))
        epe = np.abs(preds[-1].astype(np.float64) - g)[v]
        metrics = {'train_epe': epe.mean() if n else np.nan, 'train_1px': (epe < 1).mean() if n else np.nan,
                   'train_3px': (epe < 3).mean() if n else np.nan}
        grads = [np.where(v, np.sign(p.astype(np.float64) - g) * wi / max(n, 1), 0.0) for p, wi in zip(preds, w)]
    return loss, metrics, grads, inf


def sequence_loss_kernel(preds, gt, valid, gamma=0.9, mutant=None):
    """The sequence-loss kernel's op order in fp32 (fp64 partial sums, an fp32 reciprocal of the fp32 count):
    -> (loss, epe, px1, px3) as np.float32."""
    v = valid >= 0.5
    g = gt.astype(np.float32)
    n = v.size if mutant == "all_pixels" else int(v.sum())
    inv = np.float32(1) / np.float32(n)
    d = [(p.astype(np.float32) - g)[v] for p in preds]
    loss = np.float32(0)
    for wi, di in zip(loss_weights(len(preds), gamma), d):
        m = np.float32(np.float32(np.abs(di).astype(np.float64).sum()) * inv)
        loss = np.float32(loss + np.float32(np.float32(wi) * m))
    last = d[0] if mutant == "epe_first" else d[-1]
    ep = np.sqrt(last * last)
    epe = np.float32(np.float32(ep.astype(np.float64).sum()) * inv)
    return (loss, epe, np.float32(np.float32((ep < 1).sum()) * inv), np.float32(np.float32((ep < 3).sum()) * inv))
