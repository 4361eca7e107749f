"""The disparity head of both training stages on sm_90a: convex flow upsampling (reference core/raft_stereo_human.py:69-81,
`FlowUpdateModule.upsample_flow`) and the sequence loss (lib/loss.py:8-33), forward and backward (csrc/flow_head.cu).

`convex_upsample(flow, mask, factor)` is the body of `upsample_flow` in one forward kernel and two backward kernels, in
place of the softmax / unfold / fp32 broadcast product / sum / permute chain.  It keeps the op chain's dtype boundaries:
the weights have the mask's dtype, products and sums are fp32, `mask.grad` has the mask's dtype and `flow.grad` is fp32.
CUDA fp32 flow with D in {1, 2}, an fp32 or fp16 mask and factor in {2, 4, 8} only; anything else raises.

`sequence_loss(flow_preds, flow_gt, valid, loss_gamma=0.9)` has the reference's signature and results with one host
synchronisation (one read of the stats and the inf flag) instead of about nine.  The predictions and `valid` are fp32;
`flow_gt` is fp32 or fp16 (the training cache stores the flow in fp16 and the loader hands it over unchanged; the op
chain promotes `pred - gt` to fp32, and so do the kernels).  Inputs it does not cover (CPU tensors, other dtypes such as
the fp64 flow of the uncached loader, C != 1, more than 32 predictions, a flow_gt that requires grad) go to the
reference's function, which is looked up in `lib.loss` when that module is importable.
"""
import ctypes as C
import sys

import torch

from . import _lib

FACTORS = (2, 4, 8)
_MASK_DTYPES = {torch.float32: 0, torch.float16: 1}
_GT_DTYPES = {torch.float32: 0, torch.float16: 1}


def _p(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


def upsample_supported(flow, mask, factor):
    """Whether `convex_upsample` runs these inputs natively (the patched `upsample_flow` calls the reference otherwise)."""
    if not (torch.is_tensor(flow) and torch.is_tensor(mask) and flow.is_cuda and mask.device == flow.device):
        return False
    if flow.dtype != torch.float32 or mask.dtype not in _MASK_DTYPES or factor not in FACTORS or flow.dim() != 4:
        return False
    N, D, H, W = flow.shape
    return D in (1, 2) and tuple(mask.shape) == (N, 9 * factor * factor, H, W)


class _ConvexUpsample(torch.autograd.Function):
    @staticmethod
    def forward(ctx, flow, mask, factor):
        N, D, H, W = (int(s) for s in flow.shape)
        fl, m = flow.detach().contiguous(), mask.detach().contiguous()
        out = torch.empty((N, D, factor * H, factor * W), dtype=torch.float32, device=flow.device)
        with torch.cuda.device(flow.device):
            rc = _lib.lib.gpsg_convex_upsample_forward(*_lib.device_stream(flow.device), _MASK_DTYPES[m.dtype], factor,
                                                       N, D, H, W, _p(fl), _p(m), _p(out))
        _lib.check(rc, "gpsg_convex_upsample_forward")
        ctx.save_for_backward(fl, m)
        ctx.factor = factor
        return out

    @staticmethod
    def backward(ctx, grad_out):
        fl, m = ctx.saved_tensors
        N, D, H, W = (int(s) for s in fl.shape)
        want_flow, want_mask = ctx.needs_input_grad[0], ctx.needs_input_grad[1]
        if not (want_flow or want_mask):
            return None, None, None
        g = grad_out.detach().to(torch.float32).contiguous()
        dmask = torch.empty_like(m) if want_mask else None
        dflow = torch.empty_like(fl) if want_flow else None
        ws = None
        if want_flow:
            nb = int(_lib.lib.gpsg_convex_upsample_backward_workspace_bytes(N, D, H, W))
            ws = torch.empty(nb // 4, dtype=torch.float32, device=fl.device)
        with torch.cuda.device(fl.device):
            rc = _lib.lib.gpsg_convex_upsample_backward(*_lib.device_stream(fl.device), _MASK_DTYPES[m.dtype], ctx.factor,
                                                        N, D, H, W, _p(fl), _p(m), _p(g), _p(dmask), _p(dflow), _p(ws))
        _lib.check(rc, "gpsg_convex_upsample_backward")
        return dflow, dmask, None


def convex_upsample(flow, mask, factor):
    """[N, D, H, W] fp32 flow and [N, 9*f^2, H, W] fp32 / fp16 mask -> [N, D, f*H, f*W] fp32: the convex combination of
    the 3x3 neighbourhood of f*flow under the softmax of the mask over its 9 taps (`upsample_flow`)."""
    if not upsample_supported(flow, mask, factor):
        raise RuntimeError(
            f"convex_upsample (gpsg): needs CUDA fp32 flow [N, 1|2, H, W], an fp32/fp16 mask [N, 9*f^2, H, W] on the same "
            f"device and f in {FACTORS}; got flow {tuple(flow.shape)} {flow.dtype} {flow.device}, mask "
            f"{tuple(mask.shape)} {mask.dtype} {mask.device}, f={factor}")
    return _ConvexUpsample.apply(flow, mask, factor)


def make_upsample_flow(orig):
    """`FlowUpdateModule.upsample_flow` on the fused kernels; inputs they do not cover, and calls under autocast (where
    the op chain's softmax changes dtype), go to `orig`, the reference's own method."""
    def upsample_flow(self, flow, mask):
        factor = 2 ** self.args.n_downsample
        if torch.is_autocast_enabled() or not upsample_supported(flow, mask, factor):
            return orig(self, flow, mask)
        return _ConvexUpsample.apply(flow, mask, factor)
    upsample_flow.__doc__ = orig.__doc__
    return upsample_flow


# ---- sequence loss -------------------------------------------------------------------------------------------------

def loss_weights(n_predictions, loss_gamma=0.9):
    """The per-prediction weights of lib/loss.py:18-21, in the reference's own float arithmetic (one prediction raises
    its ZeroDivisionError)."""
    adjusted_loss_gamma = loss_gamma ** (15 / (n_predictions - 1))
    return [adjusted_loss_gamma ** (n_predictions - i - 1) for i in range(n_predictions)]


def sequence_loss_supported(flow_preds, flow_gt, valid):
    if not (torch.is_tensor(flow_gt) and torch.is_tensor(valid)) or not 1 <= len(flow_preds) <= _lib.SEQ_LOSS_MAX_PRED:
        return False
    ts = list(flow_preds) + [valid]
    if not all(torch.is_tensor(t) and t.is_cuda and t.device == flow_gt.device and t.dtype == torch.float32 and
               t.shape == flow_gt.shape for t in ts):
        return False
    if not flow_gt.is_cuda or flow_gt.dtype not in _GT_DTYPES:
        return False
    return flow_gt.dim() >= 2 and flow_gt.shape[1] == 1 and not flow_gt.requires_grad


def _args(preds, gt, valid, weights, grads=None):
    a = _lib.SeqLossArgs()
    for i, p in enumerate(preds):
        a.pred[i] = p.data_ptr()
        a.weight[i] = weights[i]
        if grads is not None:
            a.grad[i] = grads[i].data_ptr()
    a.gt, a.valid, a.numel, a.n_pred = gt.data_ptr(), valid.data_ptr(), gt.numel(), len(preds)
    a.gt_dtype = _GT_DTYPES[gt.dtype]
    return a


class _SequenceLoss(torch.autograd.Function):
    """(gt, valid, weights, *preds) -> (loss 0-dim, stats[6]); only the loss is differentiable."""

    @staticmethod
    def forward(ctx, gt, valid, weights, *preds):
        dev = gt.device
        gt, valid = gt.detach().contiguous(), valid.detach().contiguous()
        ps = [p.detach().contiguous() for p in preds]
        stats = torch.empty(6, dtype=torch.float32, device=dev)
        ws = torch.empty(int(_lib.lib.gpsg_sequence_loss_workspace_bytes()) // 8, dtype=torch.float64, device=dev)
        with torch.cuda.device(dev):
            rc = _lib.lib.gpsg_sequence_loss_forward(*_lib.device_stream(dev), _args(ps, gt, valid, weights), _p(stats),
                                                     _p(ws))
        _lib.check(rc, "gpsg_sequence_loss_forward")
        ctx.save_for_backward(gt, valid, stats, *ps)
        ctx.weights = weights
        ctx.mark_non_differentiable(stats)
        return stats[0].clone(), stats

    @staticmethod
    def backward(ctx, grad_loss, _grad_stats):
        gt, valid, stats, *ps = ctx.saved_tensors
        g = grad_loss.detach().to(torch.float32).reshape(1).contiguous()    # read on the device: no sync
        grads = [torch.empty_like(p) for p in ps]
        with torch.cuda.device(gt.device):
            rc = _lib.lib.gpsg_sequence_loss_backward(*_lib.device_stream(gt.device),
                                                      _args(ps, gt, valid, ctx.weights, grads), _p(g), _p(stats))
        _lib.check(rc, "gpsg_sequence_loss_backward")
        return (None, None, None, *grads)


def _reference_sequence_loss():
    mod = sys.modules.get("lib.loss")
    if mod is None:
        import importlib
        mod = importlib.import_module("lib.loss")
    from . import patch
    return patch.original(mod, "sequence_loss")


def sequence_loss(flow_preds, flow_gt, valid, loss_gamma=0.9):
    """lib/loss.py:8-33 with the same signature and results: (0-dim fp32 flow_loss with gradient to every prediction,
    {'train_epe', 'train_1px', 'train_3px'} as Python floats).  valid >= 0.5 selects the pixels; an inf in flow_gt at a
    valid pixel raises AssertionError; an empty valid set gives NaN.  The loss's reductions run in a fixed order (bit-
    reproducible) and the prediction gradients are bit-identical to the op chain's on the GPU."""
    if not sequence_loss_supported(flow_preds, flow_gt, valid):
        return _reference_sequence_loss()(flow_preds, flow_gt, valid, loss_gamma)
    weights = loss_weights(len(flow_preds), loss_gamma)
    loss, stats = _SequenceLoss.apply(flow_gt, valid, weights, *flow_preds)
    epe, px1, px3, inf, _ = stats[1:].tolist()             # the one host synchronisation
    assert not inf
    return loss, {'train_epe': epe, 'train_1px': px1, 'train_3px': px3}
