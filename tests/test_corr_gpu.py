"""GPU parity of the sm_90a correlation sampler: golden vectors from the reference's CorrBlock1D,
the CPU oracle at larger sizes, fp16 volumes (stage-2 AMP), edge cases.  Through the drop-in
`corr_sampler` module (== C-ABI via ctypes)."""
import os

import numpy as np
import pytest
import torch

from gps_gaussian_b200 import _lib, synth
from oracle.corr_oracle import CorrOracle

pytestmark = pytest.mark.gpu
G = np.load(os.path.join(os.path.dirname(__file__), "golden", "corr_golden.npz"))


def _cuda(a, dtype=torch.float32):
    return torch.from_numpy(np.ascontiguousarray(a)).to("cuda", dtype)


def test_sampler_forward_backward_golden():
    import corr_sampler
    coords = _cuda(G["coords"])
    for i in range(4):
        vol = _cuda(G[f"level{i}"])
        out, = corr_sampler.forward(vol, coords[:, [0]] / 2 ** i, 4)
        assert out.shape == (2, 9, 3, 40) and out.dtype == torch.float32
        assert np.abs(out.cpu().numpy() - G["out"][:, 9 * i:9 * i + 9]).max() < 2e-5     # fp32 coords/2^i and weights
        gv, = corr_sampler.backward(vol, coords[:, [0]] / 2 ** i, _cuda(G["grad_out"][:, 9 * i:9 * i + 9]), 4)
        assert gv.shape == vol.shape
        assert np.abs(gv.cpu().numpy() - G[f"grad_level{i}"]).max() < 2e-5


def test_corr_block_fast_matches_reference_block_golden():
    """Mirrored CorrBlockFast1D(fmap1, fmap2)(coords) == reference CorrBlock1D output (golden), incl. autograd."""
    from gps_gaussian_b200.corr import CorrBlockFast1D
    f1 = _cuda(G["fmap1"]).requires_grad_(True)
    f2 = _cuda(G["fmap2"]).requires_grad_(True)
    blk = CorrBlockFast1D(f1, f2, num_levels=4, radius=4)
    out = blk(_cuda(G["coords"]))
    assert out.shape == (2, 36, 3, 40)
    assert np.abs(out.detach().cpu().numpy() - G["out"]).max() < 5e-5
    (out * _cuda(G["grad_out"])).sum().backward()
    assert f1.grad is not None and torch.isfinite(f1.grad).all() and float(f1.grad.abs().sum()) > 0


@pytest.mark.parametrize("dtype,tol", [(torch.float32, 1e-5), (torch.float16, 4e-3)])
def test_sampler_vs_oracle_large(dtype, tol):
    """BASELINE-size feature maps: [2,192,128,128] -> volume [2,128,128,128] (level 0) and a pooled level."""
    import corr_sampler
    f1, f2, coords = synth.corr_inputs(2, 16, 128, 128)
    o = CorrOracle("f32")
    pyr = o.pyramid(f1, f2, 3)
    for i in (0, 2):
        volq = _cuda(pyr[i], dtype)
        ref_in = volq.float().cpu().numpy()                       # oracle sees the same (quantised) values
        cx = (coords[:, 0] / np.float32(2 ** i)).astype(np.float32)
        out, = corr_sampler.forward(volq, _cuda(coords) / 2 ** i, 4)
        assert out.dtype == dtype
        want = o.sample_fwd(ref_in, cx, 4)
        assert np.abs(out.float().cpu().numpy() - want).max() < tol * max(1.0, np.abs(want).max())
        go = np.random.default_rng(i).standard_normal(want.shape).astype(np.float32)
        goq = _cuda(go, dtype)
        gv, = corr_sampler.backward(volq, _cuda(coords) / 2 ** i, goq, 4)
        wantg = o.sample_bwd(ref_in.shape, cx, goq.float().cpu().numpy(), 4)
        assert np.abs(gv.float().cpu().numpy() - wantg).max() < tol * max(1.0, np.abs(wantg).max())


def test_sampler_edge_cases():
    import corr_sampler
    o = CorrOracle("f32")
    rng = np.random.default_rng(0)
    # odd sizes, radius != 4, everything out of range, integer coords, non-contiguous coords channel
    vol = rng.standard_normal((1, 3, 5, 7)).astype(np.float32)
    coords = np.stack([rng.uniform(-20, 30, (1, 3, 5)), np.zeros((1, 3, 5))], 1).astype(np.float32)
    coords[0, 0, 0, :3] = [-100.0, 3.0, 1e6]
    for r in (1, 4, 6):
        out, = corr_sampler.forward(_cuda(vol), _cuda(coords), r)
        assert np.abs(out.cpu().numpy() - o.sample_fwd(vol, coords[:, 0], r)).max() < 1e-5
        go = rng.standard_normal(out.shape).astype(np.float32)
        gv, = corr_sampler.backward(_cuda(vol), _cuda(coords), _cuda(go), r)
        assert np.abs(gv.cpu().numpy() - o.sample_bwd(vol.shape, coords[:, 0], go, r)).max() < 1e-5
    # empty batch
    out, = corr_sampler.forward(torch.zeros(0, 3, 5, 7, device="cuda"), torch.zeros(0, 1, 3, 5, device="cuda"), 4)
    assert out.shape == (0, 9, 3, 5)


def test_autograd_sampler_linear_and_adjoint():
    """<S(v), g> == <v, S^T(g)>: forward and backward are exact adjoints (size-independent property)."""
    from gps_gaussian_b200.corr import CorrSampler
    gen = torch.Generator("cuda").manual_seed(0)
    vol = torch.randn(2, 32, 64, 48, device="cuda", generator=gen, requires_grad=True)
    coords = torch.rand(2, 1, 32, 64, device="cuda", generator=gen) * 60 - 6
    out = CorrSampler.apply(vol, coords, 4)
    g = torch.randn(out.shape, device="cuda", generator=gen)
    (out * g).sum().backward()
    lhs = float((out.detach().double() * g.double()).sum())
    rhs = float((vol.detach().double() * vol.grad.double()).sum())
    assert abs(lhs - rhs) < 1e-3 * max(1.0, abs(lhs))


def _unfused_block(f1, f2, coords, levels=4, r=4):
    """The reference's op sequence (core/corr.py:31-61) with torch ops + the per-level sampler: einsum, /sqrt(D),
    avg_pool2d, CorrSampler per level, cat."""
    import torch.nn.functional as F
    from gps_gaussian_b200.corr import CorrSampler
    B, D, H, W1 = f1.shape
    W2 = f2.shape[3]
    corr = torch.einsum('aijk,aijh->ajkh', f1, f2).reshape(B, H, W1, 1, W2).contiguous() / torch.sqrt(torch.tensor(D).float())
    corr = corr.reshape(B * H * W1, 1, 1, W2)
    outs = []
    for i in range(levels):
        lvl = corr.view(B, H, W1, -1)
        outs.append(CorrSampler.apply(lvl, coords[:, [0]] / 2 ** i, r))
        corr = F.avg_pool2d(corr, [1, 2], stride=[1, 2])
    return torch.cat(outs, 1)


@pytest.mark.parametrize("shape", [(2, 24, 3, 40), (1, 192, 5, 128), (2, 17, 2, 150)])
def test_fused_block_matches_unfused_incl_fmap_grads(shape):
    """Fused build+pyramid and fused 4-level lookup == the reference's op-by-op sequence (fp32), outputs and d/dfmap."""
    from gps_gaussian_b200.corr import CorrBlockFast1D
    B, D, H, W = shape
    f1n, f2n, cn = synth.corr_inputs(B, D, H, W, seed=5)
    g = torch.randn(B, 36, H, W, device="cuda", generator=torch.Generator("cuda").manual_seed(1))
    res = []
    for fused in (True, False):
        f1 = _cuda(f1n).requires_grad_(True); f2 = _cuda(f2n).requires_grad_(True)
        out = CorrBlockFast1D(f1, f2, num_levels=4, radius=4)(_cuda(cn)) if fused else _unfused_block(f1, f2, _cuda(cn))
        (out * g).sum().backward()
        res.append((out.detach(), f1.grad, f2.grad))
    for a, b in zip(*res):
        assert a.shape == b.shape
        assert float((a - b).abs().max()) < 2e-4 * max(1.0, float(b.abs().max()))


@pytest.mark.parametrize("dtype,tol", [(torch.float32, 2e-5), (torch.float16, 3e-3)])
def test_fused_pyramid_build_vs_oracle(dtype, tol):
    from gps_gaussian_b200.corr import CorrBlockFast1D
    f1n, f2n, _ = synth.corr_inputs(2, 192, 6, 128, seed=3)
    f1, f2 = _cuda(f1n, dtype), _cuda(f2n, dtype)
    blk = CorrBlockFast1D(f1, f2, num_levels=4, radius=4)
    o = CorrOracle("f64")
    pyr = o.pyramid(f1.float().cpu().numpy(), f2.float().cpu().numpy(), 4)       # oracle sees the quantised inputs
    for i in range(4):
        got = blk.corr_pyramid[i]
        assert got.shape == (2, 6, 128, 1, 128 >> i) and got.dtype == dtype
        assert np.abs(got.squeeze(3).float().cpu().numpy() - pyr[i]).max() < tol * max(1.0, np.abs(pyr[i]).max())


@pytest.mark.parametrize("dtype,tol", [(torch.float32, 2e-5), (torch.float16, 4e-3)])
@pytest.mark.parametrize("shape", [(1, 192, 4, 128, 128), (2, 70, 3, 33, 150), (1, 5, 1, 1, 1)])
def test_build_backward_kernel_vs_fp64_contractions(dtype, tol, shape):
    """gpsg_corr_build_backward: dF1 = F2 g^T / sqrt(D), dF2 = F1 g / sqrt(D) vs fp64 einsum (W1 != W2, ragged tiles)."""
    import ctypes as C
    from gps_gaussian_b200 import _lib
    B, D, H, W1, W2 = shape
    gen = torch.Generator("cuda").manual_seed(11)
    f1 = torch.randn(B, D, H, W1, device="cuda", generator=gen).to(dtype)
    f2 = torch.randn(B, D, H, W2, device="cuda", generator=gen).to(dtype)
    g = torch.randn(B, H, W1, W2, device="cuda", generator=gen).to(dtype)
    d1, d2 = torch.full_like(f1, float("nan")), torch.full_like(f2, float("nan"))
    p = lambda t: C.c_void_p(t.data_ptr())
    rc = _lib.lib.gpsg_corr_build_backward(0, C.c_void_p(torch.cuda.current_stream().cuda_stream),
                                           0 if dtype == torch.float32 else 1, B, D, H, W1, W2, p(f1), p(f2), p(g), p(d1), p(d2))
    _lib.check(rc, "gpsg_corr_build_backward")
    r1 = torch.einsum("bhxy,bdhy->bdhx", g.double(), f2.double()) / D ** 0.5
    r2 = torch.einsum("bhxy,bdhx->bdhy", g.double(), f1.double()) / D ** 0.5
    for got, ref in ((d1, r1), (d2, r2)):
        assert torch.isfinite(got).all()
        assert float((got.double() - ref).abs().max()) < tol * max(1.0, float(ref.abs().max()))


@pytest.mark.parametrize("shape", [(2, 192, 6, 128, 128), (1, 64, 3, 152, 48), (1, 32, 2, 264, 128), (1, 256, 2, 64, 64),
                                   (1, 16, 1, 8, 16)])
def test_fp16_tcgen05_build_matches_ffma_kernel_and_oracle(shape):
    """fp16 volumes take the wgmma kernel (corr_tc.cu); GPSG_CORR_BUILD=ffma forces the FFMA kernel.  Both follow the
    same rounding chain, so every pyramid level agrees to one fp16 ulp of the level's magnitude (different fp32 summation
    order), and both match the fp64 oracle on the quantised inputs.  Shapes: ragged M tiles (W1 = 152, 264), N < 128."""
    from gps_gaussian_b200.corr import CorrBlockFast1D
    B, D, H, W1, W2 = shape
    gen = torch.Generator("cuda").manual_seed(7)
    f1 = torch.randn(B, D, H, W1, device="cuda", generator=gen).half()
    f2 = torch.randn(B, D, H, W2, device="cuda", generator=gen).half()
    tc = [v.clone() for v in CorrBlockFast1D(f1, f2, num_levels=4, radius=4).corr_pyramid]
    _lib.set_corr_build("ffma")
    try:
        ff = [v.clone() for v in CorrBlockFast1D(f1, f2, num_levels=4, radius=4).corr_pyramid]
    finally:
        _lib.set_corr_build("wgmma")
    pyr = CorrOracle("f64").pyramid(f1.float().cpu().numpy(), f2.float().cpu().numpy(), 4)
    for l in range(4):
        a, b = tc[l].squeeze(3).float(), ff[l].squeeze(3).float()
        assert a.shape == (B, H, W1, W2 >> l) and tc[l].dtype == torch.float16
        scale = max(1.0, float(b.abs().max()))
        assert float((a - b).abs().max()) <= 2.0 ** -10 * scale * 2, l                  # <= 1 ulp at the top binade
        assert float(((a - b).abs() > 0).float().mean()) < 0.02, l                     # and almost always bit-identical
        assert np.abs(a.cpu().numpy() - pyr[l]).max() < 3e-3 * max(1.0, np.abs(pyr[l]).max()), l


def test_tcgen05_build_falls_back_for_unsupported_shapes():
    """D not a multiple of 16, W2 > 128, W2 % 16 != 0 or misaligned views use the FFMA kernel: same results as ever."""
    from gps_gaussian_b200.corr import CorrBlockFast1D
    gen = torch.Generator("cuda").manual_seed(8)
    for (B, D, H, W1, W2) in [(1, 24, 2, 40, 40), (1, 32, 2, 64, 160), (1, 32, 1, 24, 24)]:
        f1 = torch.randn(B, D, H, W1, device="cuda", generator=gen).half()
        f2 = torch.randn(B, D, H, W2, device="cuda", generator=gen).half()
        got = CorrBlockFast1D(f1, f2, num_levels=2, radius=4).corr_pyramid[0].squeeze(3).float()
        ref = torch.einsum("bdhx,bdhy->bhxy", f1.double(), f2.double()) / D ** 0.5
        assert float((got.double() - ref).abs().max()) < 3e-3 * max(1.0, float(ref.abs().max()))


@pytest.mark.parametrize("shape", [(2, 192, 4, 128, 128), (1, 64, 2, 152, 48), (1, 32, 2, 264, 128), (1, 256, 1, 64, 64),
                                   (1, 16, 1, 8, 16), (1, 48, 3, 72, 112)])
def test_fp16_tcgen05_build_backward_matches_ffma_kernel_and_fp64(shape):
    """gpsg_corr_build_backward in fp16: wgmma kernels (K-major and MN-major g operand) vs the FFMA kernels
    (GPSG_CORR_BUILD=ffma) vs fp64 contractions; ragged M tiles and K padded to 16 (W1 = 152, 264, 72, 8)."""
    import ctypes as C
    from gps_gaussian_b200 import _lib
    B, D, H, W1, W2 = shape
    gen = torch.Generator("cuda").manual_seed(13)
    f1 = torch.randn(B, D, H, W1, device="cuda", generator=gen).half()
    f2 = torch.randn(B, D, H, W2, device="cuda", generator=gen).half()
    g = torch.randn(B, H, W1, W2, device="cuda", generator=gen).half()
    p = lambda t: C.c_void_p(t.data_ptr())

    def run():
        d1, d2 = torch.full_like(f1, float("nan")), torch.full_like(f2, float("nan"))
        rc = _lib.lib.gpsg_corr_build_backward(0, C.c_void_p(torch.cuda.current_stream().cuda_stream), 1, B, D, H, W1, W2,
                                               p(f1), p(f2), p(g), p(d1), p(d2))
        _lib.check(rc, "gpsg_corr_build_backward")
        torch.cuda.synchronize()
        return d1, d2

    tc = run()
    _lib.set_corr_build("ffma")
    try:
        ff = run()
    finally:
        _lib.set_corr_build("wgmma")
    r1 = torch.einsum("bhxy,bdhy->bdhx", g.double(), f2.double()) / D ** 0.5
    r2 = torch.einsum("bhxy,bdhx->bdhy", g.double(), f1.double()) / D ** 0.5
    for a, b_, ref in ((tc[0], ff[0], r1), (tc[1], ff[1], r2)):
        assert torch.isfinite(a).all()
        scale = max(1.0, float(ref.abs().max()))
        assert float((a.double() - ref).abs().max()) < 4e-3 * scale
        assert float((a.float() - b_.float()).abs().max()) <= 2.0 ** -9 * scale       # same value up to one fp16 ulp
