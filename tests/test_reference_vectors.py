"""Consumer of tools/dump_reference_vectors.py: when tests/golden/raster_reference_*.npz / corr_reference_*.npz exist
(recorded from the REAL diff-gaussian-rasterization / corr_sampler on a machine that has them), the CPU oracle and the
sm_90a kernels are pinned to them: radii bit-exact, RGB <= 1e-4 abs, gradients <= 1e-3 rel (BASELINE.json north_star).
Until then the rasterizer oracle stays "parity unpinned" (DESIGN.md section 2) and these tests skip; the checking code
itself is exercised on the CPU against vectors synthesised from the oracle (so it cannot rot)."""
import glob
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
sys.path.insert(0, os.path.join(ROOT, "tools"))
from dump_reference_vectors import RASTER_CASES  # noqa: E402
from gps_gaussian_b200 import synth  # noqa: E402
from helpers import GRAD_TOL, RGB_TOL, grad_err, oracle_forward  # noqa: E402

RASTER_FILES = sorted(glob.glob(os.path.join(GOLDEN, "raster_reference_*.npz")))
CORR_FILES = sorted(glob.glob(os.path.join(GOLDEN, "corr_reference_*.npz")))
no_vectors = pytest.mark.skipif(not RASTER_FILES, reason="no vectors recorded from the real diff-gaussian-rasterization yet "
                                "(tools/dump_reference_vectors.py); the rasterizer oracle is parity-unpinned until then")


def _scene(case):
    kw = dict(RASTER_CASES[case])
    return synth.random_cube_scene(kw.pop("P"), kw.pop("res"), **kw)


def check_against_vectors(vec, color, radii, grads):
    """vec: mapping with the arrays written by dump_reference_vectors.dump_raster; color/radii/grads: the implementation
    under test.  Flip-affected pixels / Gaussians are bounded the way the two oracles differ from each other."""
    assert np.array_equal(np.asarray(radii, np.int32), vec["radii"])
    d = np.abs(np.asarray(color, np.float64) - vec["color"]).max(0)
    assert (d > RGB_TOL).mean() < 5e-4 and d.max() < 1.2e-2, ((d > RGB_TOL).mean(), d.max())
    for k in ("dL_dmeans3D", "dL_dcolors", "dL_dopacity", "dL_dscales", "dL_drots"):
        per = grad_err(np.asarray(grads[k]).reshape(vec[k].shape), vec[k])
        assert (per > GRAD_TOL).sum() <= max(2, int(1e-3 * per.size)) and per.max() < 5e-2, (k, float(per.max()))


def _oracle_outputs(sc, dtype="f32"):
    o, st = oracle_forward(sc, dtype)
    g = np.random.default_rng(0).standard_normal(st["color"].shape).astype(np.float32)
    gr = o.backward(st, g.astype(o.np))
    return st, g, gr


def test_checker_plumbing_on_synthesised_vectors():
    """No real vectors needed: vectors synthesised from the fp64 oracle, checked with the fp32 oracle as the implementation."""
    sc = _scene("wide_cloud")
    st64, g, gr64 = _oracle_outputs(sc, "f64")
    vec = dict(color=st64["color"], radii=st64["radii"], grad_out=g,
               **{k: gr64[k].reshape(-1, gr64[k].shape[-1]) if gr64[k].ndim > 1 else gr64[k].reshape(-1, 1)
                  for k in ("dL_dmeans3D", "dL_dcolors", "dL_dopacity", "dL_dscales", "dL_drots")})
    st32, _, gr32 = _oracle_outputs(sc, "f32")
    check_against_vectors(vec, st32["color"], st32["radii"], gr32)
    bad = dict(gr32, dL_dscales=gr32["dL_dscales"] * 1.01)
    with pytest.raises(AssertionError):
        check_against_vectors(vec, st32["color"], st32["radii"], bad)


@no_vectors
@pytest.mark.parametrize("path", RASTER_FILES or ["-"])
def test_cpu_oracle_matches_the_real_extension(path):
    vec = np.load(path)
    sc = _scene(str(vec["case"]))
    o, st = oracle_forward(sc, "f32")
    gr = o.backward(st, vec["grad_out"].astype(np.float32))
    check_against_vectors(vec, st["color"], st["radii"], gr)


@no_vectors
@pytest.mark.gpu
@pytest.mark.parametrize("path", RASTER_FILES or ["-"])
def test_device_matches_the_real_extension(path):
    import torch
    from gps_gaussian_b200.introspect import RasterCall
    vec = np.load(path)
    sc = _scene(str(vec["case"]))
    rc = RasterCall(sc)
    rc.forward()
    got = rc.backward(torch.from_numpy(vec["grad_out"]).cuda(), want_cov3D=False)
    check_against_vectors(vec, rc.color.cpu().numpy(), rc.radii.cpu().numpy(),
                          {k: v.cpu().numpy() for k, v in got.items() if v is not None})


@pytest.mark.skipif(not CORR_FILES, reason="no vectors recorded from the real corr_sampler (the sampler is pinned by CorrBlock1D instead)")
@pytest.mark.gpu
@pytest.mark.parametrize("path", CORR_FILES or ["-"])
def test_device_sampler_matches_the_real_extension(path):
    import torch
    import corr_sampler
    vec = np.load(path)
    v, c = torch.from_numpy(vec["volume"]).cuda(), torch.from_numpy(vec["coords"]).cuda()
    out, = corr_sampler.forward(v, c, int(vec["radius"]))
    assert np.abs(out.cpu().numpy() - vec["out"]).max() < 1e-5
    gv, = corr_sampler.backward(v, c, torch.from_numpy(vec["grad_out"]).cuda(), int(vec["radius"]))
    assert np.abs(gv.cpu().numpy() - vec["grad_volume"]).max() < 1e-5
