"""Shared helpers for the parity tests (oracle = checker only).

Parity accounting (VERDICT r1 weak #1/#2).  A.4/A.6 take three hard decisions per evaluated (pixel, Gaussian) pair:
`power > 0`, `alpha < 1/255`, `test_T < 1e-4`.  Two correct fp32 implementations can disagree on one only where the
tested value sits within rounding distance of its threshold.  `RasterOracle.margins` measures that distance, so the old
"x % of pixels may exceed 1e-4" budgets become statements that are checked exactly:

  image      every pixel NOT near a threshold: |gpu - oracle| <= 1e-4 (north_star), n_contrib identical, final_T to 1e-5;
             every pixel over 1e-4 IS near a threshold, and moves by at most one flipped contribution (<= 1.2e-2).
  gradients  the backward replays the forward's decisions (final_T, n_contrib are inputs of A.6), so it is compared with
             the oracle's backward run on the SAME forward decisions (the device's final_T / n_contrib / tile lists).  What
             is left are `alpha < 1/255` / `power > 0` re-evaluations.  Three classes of Gaussians:
               clean   not evaluated by any pixel that has such a near decision:   <= 1e-3 (max-normalised, north_star)
               shared  evaluated by such a pixel, own decision not near (a neighbour's flip rescales its T / accumulated
                       colour there by ~1/255):                                      <= 5e-3
               own     its own alpha/power is the near one (a flip adds/removes its whole contribution at that pixel): <= 5e-2
             Against the fp32 oracle (same precision as the device; eps = rounding of the device's approximations) `clean`
             is > 95 % of a C2 scene and agrees to ~1e-6.  Against the fp64 oracle the fp32 rounding of the projected
             means (6e-5 px at 1000-px coordinates => 1e-4 relative on alpha) must be inside eps, so eps_alpha = 1e-3 there
             and `clean` shrinks; the bound on each class is the same.
The counts are appended to $GPSG_PARITY_LOG (json lines) when that variable is set.
"""
import json
import os

import numpy as np

from oracle.raster_oracle import RasterOracle

RGB_TOL = 1e-4       # abs, BASELINE.json north_star
GRAD_TOL = 1e-3      # rel (max-normalised), BASELINE.json north_star
FLIP_CAP = 1.2e-2    # one flipped contribution: alpha*T*c with test_T ~ 1e-4, alpha <= 0.99  =>  T*alpha <= ~1e-2
SHARED_TOL = 5e-3    # class `shared` (see above)
TAINT_CAP = 5e-2     # class `own`
EPS_ALPHA_F64 = 1e-3 # fp32 rounding of means2D / conic seen from an fp64 replay


def oracle_forward(sc, dtype="f32", nthreads=8, render=True):
    o = RasterOracle(dtype)
    return o, o.forward(sc["means3D"], sc["colors"], sc["opacity"], sc.get("scales"), sc.get("rots"), sc["view"],
                        sc["proj"], sc["tanfovx"], sc["tanfovy"], sc["W"], sc["H"], sc["bg"],
                        scale_mod=sc.get("scale_modifier", 1.0), cov3D_precomp=sc.get("cov3D_precomp"),
                        nthreads=nthreads, render=render)


def near_plane_scene(sc, seed=0):
    """`sc` with its Gaussians moved to view-space depths on both sides of the z = 0.2 cull plane (some a relative 1e-7 or
    less from it, some exactly on it), inside the field of view.  Returns (scene, view-space z in fp64)."""
    rng = np.random.default_rng(seed)
    P = sc["means3D"].shape[0]
    d = np.concatenate([[0.0, 1e-8, -1e-8, 3e-8, -3e-8, 1e-7, -1e-7], rng.choice([-1, 1], P) * 10.0 ** rng.uniform(-7, 0, P)])
    z = np.clip(0.2 + d[:P], 0.01, None)
    E = sc["cam"]["E"]
    xy = rng.uniform(-0.4, 0.4, (P, 2)) * np.array([sc["tanfovx"], sc["tanfovy"]]) * z[:, None]
    X = ((np.concatenate([xy, z[:, None]], 1) - E[:, 3]) @ E[:, :3]).astype(np.float32)
    z_view = X.astype(np.float64) @ E[2, :3] + E[2, 3]             # of the fp32-rounded positions
    return dict(sc, means3D=X), z_view


def rel_err(a, b):
    """max |a-b| / max|b|  (normalised max error; b is the reference)."""
    a = np.asarray(a, np.float64); b = np.asarray(b, np.float64)
    d = np.abs(a - b).max() if a.size else 0.0
    s = np.abs(b).max() if b.size else 0.0
    return d / s if s > 0 else d


def record(tag, **kv):
    path = os.environ.get("GPSG_PARITY_LOG")
    if path:
        os.makedirs(os.path.dirname(os.path.abspath(path)), exist_ok=True)
        with open(path, "a") as f:
            f.write(json.dumps(dict(case=tag, **kv)) + "\n")


def _threads():
    return min(os.cpu_count() or 8, 64)


def assert_image_parity(tag, color, final_T, n_contrib, oracle, ref):
    """color [3,H,W], final_T [H,W], n_contrib [H,W] from the device vs the fp32 oracle state `ref` (same tile lists)."""
    m = oracle.margins(ref, nthreads=_threads())
    near = m["near"]
    d = np.abs(np.asarray(color, np.float64) - ref["color"]).max(0)
    over = d > RGB_TOL
    far_max = float(d[~near].max()) if (~near).any() else 0.0
    nc_bad = n_contrib.reshape(near.shape) != ref["n_contrib"]
    dT = np.abs(np.asarray(final_T, np.float64).reshape(near.shape) - ref["final_T"])
    rec = dict(pixels=int(near.size), near=int(near.sum()), over_tol=int(over.sum()), over_tol_not_near=int((over & ~near).sum()),
               max_err_not_near=far_max, max_err=float(d.max()), n_contrib_mismatch=int(nc_bad.sum()),
               n_contrib_mismatch_not_near=int((nc_bad & ~near).sum()), eps=m["eps"])
    record(tag + ":image", **rec)
    assert far_max <= RGB_TOL, rec                          # the north_star bound, on every pixel it can hold for
    assert not (over & ~near).any(), rec                    # => every pixel over tolerance has a near-threshold decision
    assert float(d.max()) <= FLIP_CAP, rec                  # and moved by at most one flipped contribution
    assert not (nc_bad & ~near).any(), rec
    assert float(dT[~near].max() if (~near).any() else 0.0) <= 1e-5, rec
    assert near.mean() < 0.02, rec                          # the exemption is a thin set
    return rec


def forced_backward(sc, dtype, base, final_T, n_contrib, g):
    """Oracle backward in `dtype` on its own continuous per-Gaussian state but the DISCRETE decisions of the forward under
    test: visible set + tile lists of `base` (fp32 oracle state, bit-identical to the device's) and the device's final_T /
    n_contrib -- exactly the inputs A.6 replays.  Returns (oracle, state, grads)."""
    o, st = oracle_forward(sc, dtype, render=False)
    st = dict(st)
    st["radii"], st["ranges"], st["_vals_full"] = base["radii"], base["ranges"], base["_vals_full"]
    st["final_T"] = np.ascontiguousarray(np.asarray(final_T).reshape(sc["H"], sc["W"]), o.np)
    st["n_contrib"] = np.ascontiguousarray(np.asarray(n_contrib).reshape(sc["H"], sc["W"]), np.uint32)
    return o, st, o.backward(st, np.asarray(g, o.np))


def grad_err(got, want):
    """per-Gaussian max error normalised by the tensor's max magnitude."""
    want = np.asarray(want, np.float64)
    got = np.asarray(got, np.float64).reshape(want.shape[0], -1)
    want = want.reshape(want.shape[0], -1)
    return np.abs(got - want).max(1) / max(np.abs(want).max(), 1e-30)


GRAD_KEYS = (("dL_dmeans3D", "dL_dmeans3D"), ("dL_dcolors", "dL_dcolors"), ("dL_dopacity", "dL_dopacity"),
             ("dL_dscales", "dL_dscales"), ("dL_drots", "dL_drots"), ("dL_dmeans2D", "dL_dmean2D"), ("dL_dcov3D", "dL_dcov3D"))


def assert_grad_parity(tag, sc, got, base, final_T, n_contrib, g, dtypes=("f32", "f64"), keys=GRAD_KEYS):
    """got: dict of numpy gradient arrays from the device (names of the C-ABI)."""
    rec_all = {}
    for dt in dtypes:
        o, st, want = forced_backward(sc, dt, base, final_T, n_contrib, g)
        # T decisions are not re-taken in the backward (eps_T = 0); see the module docstring for the three classes
        eps = dict(T=0.0) if dt == "f32" else dict(T=0.0, alpha=EPS_ALPHA_F64)
        m = o.margins(st, eps=eps, nthreads=_threads())
        own, shared = m["taint_own"], m["taint"] & ~m["taint_own"]
        clean = ~m["taint"]
        for k_got, k_ref in keys:
            if got.get(k_got) is None:
                continue
            a = np.asarray(got[k_got])
            if k_got == "dL_dmeans2D":
                a = a[:, :2]                                  # [P,3] with z unused vs the oracle's NDC-scaled [P,2]
            per = grad_err(a, want[k_ref])
            mx = lambda msk: float(per[msk].max()) if msk.any() else 0.0
            rec = dict(P=int(per.size), clean=int(clean.sum()), shared=int(shared.sum()), own=int(own.sum()),
                       near_pixels=int(m["near"].sum()), over_tol=int((per > GRAD_TOL).sum()),
                       over_tol_clean=int(((per > GRAD_TOL) & clean).sum()), max_err_clean=mx(clean), max_err_shared=mx(shared),
                       max_err_own=mx(own), eps_alpha=m["eps"]["alpha"])
            rec_all[(dt, k_got)] = rec
            record(f"{tag}:grad:{dt}:{k_got}", **rec)
            assert rec["max_err_clean"] <= GRAD_TOL, (dt, k_got, rec)
            assert rec["max_err_shared"] <= SHARED_TOL, (dt, k_got, rec)
            assert rec["max_err_own"] <= TAINT_CAP, (dt, k_got, rec)
        if dt == "f32":
            # the exemption stays a minority (C2: 3 %; 2048^2 render of 512^2 sources, splats 4x larger: 38 %)
            assert clean.size < 5000 or clean.mean() > 0.5, (dt, float(clean.mean()))
    return rec_all
