"""Independent fp64 torch restatement of the fused photometric loss (TEST INFRASTRUCTURE ONLY).

Restates `0.8 L1 + 0.2 (1 - SSIM)` (reference train_stage2.py:70-72, lib/loss.py:35-72) from its maths, in
differentiable fp64 CPU torch, so that the gradients w.r.t. the image and the ground truth come from autograd rather
than from a hand-written backward:

  * moments  mu1 = w * x, mu2 = w * y, E[x^2] = w * x^2, E[y^2] = w * y^2, E[xy] = w * xy, with `*` the zero-padded
    11x11 correlation and w the reference's window: the fp32 outer product of the fp32 1-D Gaussian whose bit patterns
    `loss_oracle.window_1d()` holds;
  * S = (2 mu1 mu2 + C1)(2 s12 + C2) / ((mu1^2 + mu2^2 + C1)(s11 + s22 + C2)), s11 = E[x^2] - mu1^2, s22 likewise,
    s12 = E[xy] - mu1 mu2, C1 = 0.01^2, C2 = 0.03^2;
  * L1 = mean |x - y|, SSIM = mean S, both over all planes * H * W elements.

`dmaps` gives the three per-pixel partials the CUDA forward stores for its backward (dS/dmu1 at fixed E[.], dS/dE[x^2],
dS/dE[xy]), by autograd of the per-pixel S w.r.t. the moments.  `grad_from_dmaps` is the closed form the backward
evaluates from them; `mutant=` perturbs it (and the forward) the way a wrong kernel would, so the tests can show that
the per-element bounds of `bounds` reject each such kernel.

Error bound.  Let eps_q = 2^-24 (1 + (E_q[x^2] + E_q[y^2]) / B2_q), B2 = s11 + s22 + C2, B1 = mu1^2 + mu2^2 + C1.  In
fp32 the moments carry errors of a few ulps of E[x^2] + E[y^2], which the cancellation in s11, s22, s12 turns into a
relative error of order eps_q in B2 and A2 = 2 s12 + C2; |S| <= 1, |A1| <= B1 and |A2| <= B2 then bound every derived
quantity at q by eps_q times its natural scale:
    S: 1,   dS/dE[x^2]: 1/B2,   dS/dE[xy]: 2/B2,   dS/dmu1: 2 (|mu1| + |mu2|) (1/B1 + 1/B2).
The backward sum  sum_q w(q-p) (dmu1_q + 2 x_p ds11_q + y_p ds12_q)  cancels as well, so its error is bounded by the
window sum of eps_q times those scales, with |x_p| and |y_p| as the weights of the last two.  The L1 sign is exact on
the same fp32 inputs; the final products add a few ulps of the w_l1 term.

C_BOUND is the constant in front of the gradient bound, C_DMAPS the one in front of the per-pixel partials and of the
values (a single pixel's partials do not average their rounding errors over a window, so they need more room).  Both
were fixed from fp32 evaluations on the CPU: the reference's own fp32 autograd chain stays within a quarter of the
gradient bound on every element of every case tests/test_loss_torch64_cpu.py runs (at most 0.17 of it), and an fp32
121-tap conv2d forward reaches 0.41 of the partials' bound."""
import torch
import torch.nn.functional as F

from oracle.loss_oracle import window_1d

F64 = torch.float64
C1, C2 = 0.01 ** 2, 0.03 ** 2
EPS = 2.0 ** -24
C_BOUND = 32.0                 # gradients w.r.t. img and gt
C_DMAPS = 128.0                # per-pixel partials, loss, L1 and SSIM values
TILE = 32                      # the CUDA kernels' output tile (csrc/loss.cu), for the halo mutants
MUTANTS = ("window_shift", "dss_xy_swapped", "n_per_plane", "sign0_plus", "halo_bwd", "halo_fwd")


class Window:
    """The reference's 11x11 window w2 = fp32(w w^T) (`_1D.mm(_1D.t()).float()`, w = `loss_oracle.window_1d()`) as a
    zero-padded correlation of [P,H,W] planes.  w2 is applied as the exact fp64 separable product w w^T plus the exact
    remainder D = w2 - w w^T (|D| <= 2^-24 w2), the latter in fp32: the result is the fp64 correlation with w2 to
    ~2^-48 relative, at a fraction of the cost of an fp64 11x11 conv2d.  `shift` moves every tap one column right."""

    def __init__(self, shift=False):
        w = torch.from_numpy(window_1d()).to(F64)
        w2 = torch.outer(w.float(), w.float()).to(F64)
        d = w2 - torch.outer(w, w)                                  # exact: w_i w_j has 48 significant bits
        wh = w
        if shift:
            wh, d = torch.roll(w, 1), torch.roll(d, 1, dims=1)
        self.wv, self.wh, self.d32 = w.reshape(1, 1, 11, 1), wh.reshape(1, 1, 1, 11), d.float()[None, None]
        self.w2 = torch.outer(w, wh) + d

    def __call__(self, a):
        a = a[:, None]
        sep = F.conv2d(F.conv2d(a, self.wh, padding=(0, 5)), self.wv, padding=(5, 0))
        return (sep + F.conv2d(a.float(), self.d32, padding=5).to(F64))[:, 0]


def window_2d(dtype=F64):
    """[11,11]: the reference's window in `dtype`."""
    return Window().w2.to(dtype)


def planes_of(t):
    """[..., H, W] -> [P, H, W]."""
    return t.reshape(-1, t.shape[-2], t.shape[-1])


def tiled(blur):
    """`blur` with every input outside the output pixel's 32x32 tile read as zero: a kernel whose halo is lost."""
    def tile_blur(a):
        out = torch.zeros_like(a)
        H, W = a.shape[-2:]
        for y0 in range(0, H, TILE):
            for x0 in range(0, W, TILE):
                out[:, y0:y0 + TILE, x0:x0 + TILE] = blur(a[:, y0:y0 + TILE, x0:x0 + TILE])
        return out
    return tile_blur


def blur_for(mutant=None, stage="fwd"):
    """The correlation a kernel with bug `mutant` applies in its forward (`stage="fwd"`) or backward (`"bwd"`)."""
    bl = Window(shift=mutant == "window_shift")
    return tiled(bl) if mutant == "halo_" + stage else bl


def moments(x, y, blur):
    """x, y [P,H,W] -> (mu1, mu2, E[x^2], E[y^2], E[xy])."""
    return blur(x), blur(y), blur(x * x), blur(y * y), blur(x * y)


def ssim_from_moments(mu1, mu2, exx, eyy, exy):
    s11, s22, s12 = exx - mu1 * mu1, eyy - mu2 * mu2, exy - mu1 * mu2
    return ((2 * mu1 * mu2 + C1) * (2 * s12 + C2)) / ((mu1 * mu1 + mu2 * mu2 + C1) * (s11 + s22 + C2))


def forward(img, gt, w_l1=0.8, w_ssim=0.2, mutant=None):
    """-> dict(loss, l1, ssim: 0-dim; ssim_map [P,H,W]; ssim_per_image [B] for [B,C,H,W] inputs; moments), fp64 and
    differentiable w.r.t. img / gt where they require grad."""
    x, y = planes_of(img.to(F64)), planes_of(gt.to(F64))
    mom = moments(x, y, blur_for(mutant))
    S = ssim_from_moments(*mom)
    n = S[0].numel() if mutant == "n_per_plane" else S.numel()
    l1 = (x - y).abs().sum() / n
    ss = S.sum() / n
    out = {"loss": w_l1 * l1 + w_ssim * (1.0 - ss), "l1": l1, "ssim": ss, "ssim_map": S, "moments": mom}
    if img.dim() == 4:
        out["ssim_per_image"] = S.reshape(img.shape[0], -1).sum(1) / (n // img.shape[0])
    return out


def forward_and_grads(img, gt, w_l1=0.8, w_ssim=0.2):
    """`forward` (detached) and the autograd d loss / d img, d loss / d gt (fp64, in the input shape)."""
    x = img.detach().to(F64).requires_grad_(True)
    y = gt.detach().to(F64).requires_grad_(True)
    out = forward(x, y, w_l1, w_ssim)
    g = torch.autograd.grad(out["loss"], (x, y))
    out = {k: (tuple(t.detach() for t in v) if k == "moments" else v.detach()) for k, v in out.items()}
    return out, g[0], g[1]


def dmaps(mom):
    """The kernel's three per-pixel partials for d/d img from the moments (mu1, mu2, E[x^2], E[y^2], E[xy]): [3,P,H,W] =
    (dS/dmu1 at fixed E[.], dS/dE[x^2], dS/dE[xy]), by autograd of sum S (S at q depends only on the moments at q)
    w.r.t. the moment maps; and the same three for d/d gt (w.r.t. mu2, E[y^2], E[xy])."""
    m = [t.detach().requires_grad_(True) for t in mom]
    g = torch.autograd.grad(ssim_from_moments(*m).sum(), m)
    return torch.stack([g[0], g[2], g[4]]), torch.stack([g[1], g[3], g[4]])


def grad_from_dmaps(img, gt, dm, w_l1=0.8, w_ssim=0.2, mutant=None):
    """Closed form of d loss / d img from its partials dm:
    (w_l1 sign(x - y) - w_ssim sum_q w(q-p) (dmu1_q + 2 x_p ds11_q + y_p ds12_q)) / N.  For d/d gt pass (gt, img)."""
    x, y = planes_of(img.detach().to(F64)), planes_of(gt.detach().to(F64))
    bl = blur_for(mutant, "bwd")
    c = [bl(dm[k]) for k in range(3)]
    if mutant == "dss_xy_swapped":
        dss = c[0] + 2 * y * c[1] + x * c[2]
    else:
        dss = c[0] + 2 * x * c[1] + y * c[2]
    sgn = torch.sign(x - y)
    if mutant == "sign0_plus":
        sgn = torch.where(x == y, torch.ones_like(sgn), sgn)
    n = x[0].numel() if mutant == "n_per_plane" else x.numel()
    return ((w_l1 * sgn - w_ssim * dss) / n).reshape(img.shape)


def mutant_outputs(img, gt, w_l1, w_ssim, mutant):
    """What a kernel with bug `mutant` would return, in fp64: the keys of `forward` plus dmaps_img, dmaps_gt, grad_img,
    grad_gt."""
    out = forward(img, gt, w_l1, w_ssim, mutant)
    out["dmaps_img"], out["dmaps_gt"] = dmaps(out.pop("moments"))
    out["grad_img"] = grad_from_dmaps(img, gt, out["dmaps_img"], w_l1, w_ssim, mutant)
    out["grad_gt"] = grad_from_dmaps(gt, img, out["dmaps_gt"], w_l1, w_ssim, mutant)
    return out


def bounds(img, gt, mom, w_l1=0.8, w_ssim=0.2, g=1.0):
    """Per-element bounds on the fp32 results, from the fp64 moments `mom` of (img, gt):
      grad    C_BOUND |g| (w_ssim sum_q w(q-p) eps_q (a_q + 2 (|x_p| + |y_p|) / B2_q) + w_l1 2^-24 [x_p != y_p]) / N,
              a_q the natural scale of dS/dmu1 (the same for d/d img and d/d gt, the scales being symmetric);
      dmaps   C_DMAPS eps_q times each partial's natural scale;
      values  SSIM: C_DMAPS mean eps_q plus the fp32 summation (4 sequential adds, a 32-lane tree, the final rounding);
              L1: a few ulps of mean |x - y|; the loss: their weighted sum and its own roundings."""
    x, y = planes_of(img.detach().to(F64)), planes_of(gt.detach().to(F64))
    mu1, mu2, exx, eyy, exy = mom
    B1 = mu1 * mu1 + mu2 * mu2 + C1
    B2 = (exx - mu1 * mu1) + (eyy - mu2 * mu2) + C2
    eps = EPS * (1.0 + (exx + eyy) / B2)
    a = 2 * (mu1.abs() + mu2.abs()) * (1 / B1 + 1 / B2)
    blur = Window()
    n = x.numel()
    ssim_part = blur(eps * a) + 2 * (x.abs() + y.abs()) * blur(eps / B2)
    grad = (C_BOUND * abs(g) * (w_ssim * ssim_part + w_l1 * EPS * (x != y).to(F64)) / n).reshape(img.shape)
    dm = C_DMAPS * eps * torch.stack([a, 1 / B2, 2 / B2])
    l1 = (x - y).abs().mean()
    t_ss = C_DMAPS * eps.mean() + 32 * EPS
    t_l1 = 32 * EPS * l1
    out = {"grad_img": grad, "grad_gt": grad, "dmaps_img": dm, "dmaps_gt": dm, "ssim": t_ss, "l1": t_l1,
           "loss": w_l1 * t_l1 + w_ssim * t_ss + 4 * EPS * (w_l1 * l1 + w_ssim)}
    if img.dim() == 4:
        out["ssim_per_image"] = C_DMAPS * eps.reshape(img.shape[0], -1).mean(1) + 32 * EPS
    return out


def reference_fp32(img, gt, w_l1=0.8, w_ssim=0.2):
    """The reference's own fp32 chain in its op order (depthwise 11x11 conv2d of x, y, x*x, y*y, x*y; pow(2) and
    products; the SSIM quotient; means), with autograd: -> (loss, grad_img, grad_gt), fp32, on [B,C,H,W] inputs."""
    x = img.detach().to(torch.float32).requires_grad_(True)
    y = gt.detach().to(torch.float32).requires_grad_(True)
    C = x.shape[-3]
    w = window_2d(torch.float32)[None, None].expand(C, 1, 11, 11).contiguous()
    conv = lambda t: F.conv2d(t, w, padding=5, groups=C)
    mu1, mu2 = conv(x), conv(y)
    mu1_sq, mu2_sq, mu1_mu2 = mu1.pow(2), mu2.pow(2), mu1 * mu2
    sigma1_sq = conv(x * x) - mu1_sq
    sigma2_sq = conv(y * y) - mu2_sq
    sigma12 = conv(x * y) - mu1_mu2
    S = ((2 * mu1_mu2 + C1) * (2 * sigma12 + C2)) / ((mu1_sq + mu2_sq + C1) * (sigma1_sq + sigma2_sq + C2))
    loss = w_l1 * torch.abs(x - y).mean() + w_ssim * (1.0 - S.mean())
    gx, gy = torch.autograd.grad(loss, (x, y))
    return loss.detach(), gx, gy
