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
before the softmax backward, dmask rounded to it.

Sequence loss over predictions p_i, ground truth g and the mask v = (valid >= 0.5):
    loss = sum_i gamma'^(P-1-i) mean_v |p_i - g|,  gamma' = gamma^(15/(P-1))
    EPE  = |p_last - g| over v;  metrics = mean EPE, mean(EPE < 1), mean(EPE < 3)
    dloss/dp_i = gamma'^(P-1-i) sign(p_i - g) / |v| on v, 0 elsewhere.
"""
import numpy as np


def _softmax9(m):
    """m [..., 9 on axis 1 ...]: softmax over axis 1 in the array's dtype, max-subtracted."""
    mx = m.max(axis=1, keepdims=True)
    e = np.exp(m - mx)
    return e / e.sum(axis=1, keepdims=True)


def _taps(flow, f, dt):
    N, D, H, W = flow.shape
    pad = np.zeros((N, D, H + 2, W + 2), dt)
    pad[:, :, 1:-1, 1:-1] = flow.astype(dt) * dt(f)
    return np.stack([pad[:, :, ky:ky + H, kx:kx + W] for ky in range(3) for kx in range(3)], axis=2)   # [N,D,9,H,W]


def _weights(mask, f, dtype):
    N, _, H, W = mask.shape
    with np.errstate(invalid="ignore", over="ignore"):
        if dtype is None:
            return _softmax9(mask.astype(np.float64).reshape(N, 9, f, f, H, W))
        w = _softmax9(mask.astype(np.float32).reshape(N, 9, f, f, H, W))
        return w.astype(dtype).astype(np.float32)


def convex_upsample(flow, mask, f, dtype=None):
    """flow [N,D,H,W], mask [N,9f^2,H,W] -> out [N,D,fH,fW] (fp64 when dtype is None, else fp32)."""
    N, D, H, W = flow.shape
    dt = np.float64 if dtype is None else np.float32
    w = _weights(mask, f, dtype)                                   # [N,9,f,f,H,W]
    U = _taps(flow, f, dt)                                         # [N,D,9,H,W]
    out = np.zeros((N, D, f, f, H, W), dt)
    with np.errstate(invalid="ignore", over="ignore"):
        for k in range(9):
            out = out + w[:, None, k] * U[:, :, k, None, None]
    return out.transpose(0, 1, 4, 2, 5, 3).reshape(N, D, f * H, f * W)


def convex_upsample_backward(flow, mask, f, grad_out, dtype=None):
    """-> (dflow [N,D,H,W], dmask [N,9f^2,H,W]) for dL/dout = grad_out."""
    N, D, H, W = flow.shape
    dt = np.float64 if dtype is None else np.float32
    w = _weights(mask, f, dtype)
    U = _taps(flow, f, dt)
    G = grad_out.astype(dt).reshape(N, D, H, f, W, f).transpose(0, 1, 3, 5, 2, 4)       # [N,D,i,j,H,W]
    with np.errstate(invalid="ignore", over="ignore"):
        dW = np.zeros((N, 9, f, f, H, W), dt)
        for d in range(D):
            dW = dW + G[:, d, None] * U[:, d, :, None, None]
        if dtype is not None:
            dW = dW.astype(dtype).astype(np.float32)
        s = np.zeros((N, 1, f, f, H, W), dt)
        for k in range(9):
            s = s + dW[:, k:k + 1] * w[:, k:k + 1]
        dmask = w * (dW - s)
        TS = (w[:, None] * G[:, :, None]).sum(axis=(3, 4))     # [N,D,9,H,W]
    dflow = np.zeros((N, D, H + 2, W + 2), dt)
    for k in range(9):
        ky, kx = divmod(k, 3)
        dflow[:, :, ky:ky + H, kx:kx + W] += TS[:, :, k]
    dflow = dflow[:, :, 1:-1, 1:-1] * dt(f)
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
