"""CPU: the per-Gaussian rounding bound of the rasterizer backward (oracle/raster_bounds.py), validated on the fp32 oracle.

gpsg_oracle.c built in fp32 is itself an fp32 implementation of the same backward, with a serial sum over each
Gaussian's pixels.  So on the fp32 forward state it must lie within the bound of the fp64 backward run on the same state
(summation depth = the number of its terms) for every Gaussian outside the exemption set -- on every scene shape the GPU
file uses.  The bound must also be tight enough to catch small errors on small gradients that the max-normalised
helpers.assert_grad_parity accepts.

The constants were fixed from operation counts (gpsg_oracle.c MAG_*, raster_bounds.C_CHAIN / C_ROT) before any ratio was
looked at; the bound is u * Mag with u = 2^-24, no extra factor.
"""
import numpy as np
import pytest

from gps_gaussian_b200 import synth
from helpers import assert_grad_parity, oracle_forward, record
from oracle import raster_bounds as rb
from oracle.raster_oracle import RasterOracle

WIDE = dict(width=250, height=40, focal=(240.0, 190.0), principal=(118.0, 23.0))
TALL = dict(width=40, height=250, focal=(150.0, 260.0), principal=(21.0, 130.0))
KEYS = ("dL_dmean2D", "dL_dconic", "dL_dopacity", "dL_dcolors", "dL_dmeans3D", "dL_dscales", "dL_drots", "dL_dcov3D")
# Planted errors go into an element under 1e-3 of its tensor's max whose Mag / |grad| is small.  Mag / |grad| < 100 is
# not met by any element here: with random-sign dL/dpix every gradient is a sum of cancelling terms, and Mag carries at
# least MAG_TERM (16) times their absolute sum.  So the limit is 1000 (a relative error of 1e-3 then exceeds u * Mag by
# >= 16x); the chosen elements have Mag / |grad| of about 110-170 and are reported with their ratios.
PLANT_MAG_MAX = 1000.0
FLIP_MAG_MAX = 1e6       # ... and a sign flip (error 2 |grad|) exceeds it by >= 33x


def _setup(sc, seed):
    o32, base = oracle_forward(sc, "f32")
    st = rb.fp64_state(base, base["final_T"], base["n_contrib"])
    g = np.random.default_rng(seed).standard_normal((3, sc["H"], sc["W"])).astype(np.float32)
    want = RasterOracle("f64").backward_mag(st, g)
    got = RasterOracle("f32").backward(dict(base), g)
    shared, own, _ = rb.exempt_sets(st, 8)
    return base, st, g, want, got, shared | own


SCENES = {
    "C1": lambda: synth.random_cube_scene(10_000, 256),
    "250x40": lambda: synth.random_cube_scene(1500, 64, spread=0.6, scale_mul=4.0, bg=(0.3, 0.6, 0.9), seed=13,
                                              **dict(WIDE, scale_modifier=0.7)),
    "40x250": lambda: synth.random_cube_scene(1500, 64, spread=0.6, scale_mul=4.0, seed=13, **dict(TALL, scale_modifier=1.6)),
    "300x8": lambda: synth.random_cube_scene(1000, 64, spread=0.6, scale_mul=2.0, bg=(0.2, 0.2, 0.2), seed=13, width=300,
                                             height=8, focal=(300.0, 50.0), principal=(150.0, 4.5)),
    "saturated": lambda: synth.random_cube_scene(3000, 64, spread=0.3, scale_mul=10.0, bg=(0.3, 0.6, 0.9), seed=13),
    "mod0.6": lambda: synth.random_cube_scene(4000, 128, seed=3, bg=(0.1, 0.2, 0.3), scale_modifier=0.6),
}


def _cov3d_precomp_scene():
    sc = synth.random_cube_scene(3000, 128, seed=5)
    _, ref = oracle_forward(sc, "f32", render=False)
    return dict(sc, cov3D_precomp=ref["cov3D"].copy(), scales=None, rots=None)


@pytest.mark.parametrize("name", list(SCENES) + ["cov3D_precomp"])
def test_fp32_oracle_backward_is_within_the_bound(name):
    sc = _cov3d_precomp_scene() if name == "cov3D_precomp" else SCENES[name]()
    base, st, g, want, got, exempt = _setup(sc, 3)
    if name == "saturated":
        r = base["ranges"].astype(np.int64)
        assert int((r[:, 1] - r[:, 0]).max()) > 2000                     # lists of 2k+ entries, many pixels saturate
    B = rb.grad_bounds(st, want, want["nterm"])
    rec = dict(P=int(st["P"]), exempt=int(exempt.sum()), visible=int((st["radii"] > 0).sum()))
    for k in KEYS:
        if name == "cov3D_precomp" and k in ("dL_dscales", "dL_drots"):
            continue
        r = rb.ratios(got[k], want[k], B[k])
        rec[k] = float(r[~exempt].max())
        assert rec[k] <= 1.0, (name, k, rec[k], int(np.argmax(np.where(exempt, 0, r))))
    record(f"bounds_cpu:{name}", **rec)
    assert exempt.size < 5000 or exempt.mean() < 0.5, rec                 # as helpers.assert_grad_parity


def test_mag_dominates_the_gradient_and_is_zero_for_culled():
    sc = synth.random_cube_scene(2000, 130, seed=9, spread=3.0, bg=(0.2, 0.3, 0.4))
    base, st, g, want, got, exempt = _setup(sc, 1)
    M = want["mag"]
    for k, s in rb.COLS.items():
        assert (M[:, s] >= np.abs(want[k]).reshape(st["P"], -1)).all(), k
        assert (want["absum"][:, s] >= np.abs(want[k]).reshape(st["P"], -1) * (1 - 1e-12)).all(), k
    B = rb.grad_bounds(st, want, want["nterm"])
    culled = st["radii"] <= 0
    assert culled.sum() > 100
    for k in KEYS:
        assert float(np.abs(B[k].reshape(st["P"], -1)[culled]).max()) == 0.0, k
        assert (B[k] >= 0).all()
    assert int(want["nterm"][culled].max()) == 0


def _pick(want_k, bound_k, exempt, rng_pick=None, qmax=PLANT_MAG_MAX):
    """A non-exempt element whose magnitude is under 1e-3 of the tensor max and whose bound is small against it."""
    w = np.abs(want_k).reshape(want_k.shape[0], -1)
    b = bound_k.reshape(w.shape) / rb.U
    with np.errstate(divide="ignore", invalid="ignore"):
        q = np.where(w > 0, b / w, np.inf)
    ok = (w > 0) & (w < 1e-3 * w.max()) & (q < qmax) & ~exempt[:, None]
    if rng_pick is not None:
        ok &= rng_pick[:, None]
    idx = np.argwhere(ok)
    assert len(idx), "no element to plant an error in"
    return tuple(idx[np.argmin(q[ok])])


def test_planted_errors_fail_the_bound_and_pass_the_max_normalised_check():
    sc = synth.random_cube_scene(10_000, 256)
    base, st, g, want, got, exempt = _setup(sc, 0)
    depth = rb.device_depth(base, want["nterm"])
    B = rb.grad_bounds(st, want, depth)
    # the deepest list position of a tile: a Gaussian that sits in one tile only, last in that tile's list, and that
    # some pixel evaluated -- its whole dL_dcolors is the term at that position
    deepest = np.zeros(st["P"], bool)
    for t in range(base["ranges"].shape[0]):
        s, e = (int(v) for v in base["ranges"][t])
        if e > s:
            deepest[base["_vals_full"][e - 1]] = True
    deepest &= (base["tiles_touched"] == 1) & (want["nterm"] > 0)
    plants = []
    i, _ = _pick(want["dL_dopacity"][:, None], B["dL_dopacity"], exempt)
    plants.append(("dL_dopacity", i, None, lambda v: v * (1 + 1e-3)))
    i, c = _pick(want["dL_drots"], B["dL_drots"], exempt, qmax=FLIP_MAG_MAX)
    plants.append(("dL_drots", i, c, lambda v: -v))
    i, c = _pick(want["dL_dcolors"], B["dL_dcolors"], exempt, rng_pick=deepest)
    plants.append(("dL_dcolors", i, c, lambda v: v * (1 + 1e-3)))
    fp32_keys = (("dL_dmeans3D", "dL_dmeans3D"), ("dL_dcolors", "dL_dcolors"), ("dL_dopacity", "dL_dopacity"),
                 ("dL_dscales", "dL_dscales"), ("dL_drots", "dL_drots"))
    for k, i, c, f in plants:
        bad = {kk: np.array(want[kk], copy=True) for kk, _ in fp32_keys}
        if c is None:
            bad[k][i] = f(bad[k][i])
        else:
            bad[k][i, c] = f(bad[k][i, c])
        r = rb.ratios(bad[k], want[k], B[k])
        record("bounds_cpu:planted", tensor=k, gaussian=int(i), ratio=float(r[i]),
               rel_to_max=float(np.abs(want[k]).reshape(st["P"], -1)[i].max() / np.abs(want[k]).max()))
        assert r[i] > 1.0, (k, i, r[i])                                  # the bound catches it
        # the max-normalised check accepts the same gradients
        assert_grad_parity("planted", sc, bad, base, base["final_T"], base["n_contrib"], g, keys=fp32_keys)
