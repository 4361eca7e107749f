"""GPU: every aux-mode gradient element within its own fp32 rounding bound of an fp64 backward on the device's own state.

The aux backward is linear in (g_rgb, g_D, g_A), and each part is a colour backward of the oracle (see
test_raster_aux_gpu.py): the colour image; the depth image, colours (z, 0, 0) over a black background, whose colour
gradient is dL/dz; the alpha image, black Gaussians over the background (-1, 0, 0).  So the fp64 truth is the sum of three
oracle_render_backward_mag runs on the device's forward state (raster_bounds.fp64_state) plus dL/dz times the view
matrix's third row in dL/dmeans3D, and the bound of each element is the sum of the three parts' bounds
(raster_bounds.grad_bounds), with
  * the depth term charged through the projection chain: |view row| * (bound of dL/dz) + the rounding of the fma that
    adds it, 2u * (|dL/dmeans3D| + |view row| |dL/dz|);
  * the extra replay operations of aux mode charged: per term the device does up to four more fp32 operations than a
    colour replay (the fourth channel's accum_rec update and fma, the g_A subtraction in the background term), against a
    per-term rounding weight of at least MAG_TERM = 16 in every part, so each part's compositing bound is scaled by 20/16.
Gaussians with a near-threshold decision are exempt, as in test_raster_grad_bounds_gpu.py.  The planted errors of the
issue (the depth term dropped from dL/dmeans3D, g_A with the wrong sign, g_D scaled by 1 + 1e-3) are each shown to fail
the bound on the device."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from gps_gaussian_b200 import synth
from gps_gaussian_b200.introspect import RasterCall
from helpers import SHARED_TOL, TAINT_CAP, grad_err, oracle_forward, record
from oracle import raster_bounds as rb
from oracle.raster_oracle import RasterOracle

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KEYS = (("dL_dmeans2D", "dL_dmean2D"), ("dL_dcolors", "dL_dcolors"), ("dL_dopacity", "dL_dopacity"),
        ("dL_dmeans3D", "dL_dmeans3D"), ("dL_dscales", "dL_dscales"), ("dL_drots", "dL_drots"), ("dL_dcov3D", "dL_dcov3D"))
AUX_OPS = 20.0 / 16.0


def _np(t):
    return t.detach().cpu().numpy()


def _threads():
    return min(os.cpu_count() or 8, 64)


class _AuxTruth:
    def __init__(self, sc, seed):
        self.sc = sc
        self.rc = RasterCall(sc)
        H, W = sc["H"], sc["W"]
        self.depth = torch.empty((H, W), device="cuda")
        self.alpha = torch.empty((H, W), device="cuda")
        self.rc.forward(out_depth=self.depth, out_alpha=self.alpha)
        torch.cuda.synchronize()
        dst = self.rc.state()
        _, self.ref = oracle_forward(sc, "f32", render=False)
        assert np.array_equal(_np(dst["point_list"]).view(np.uint32), self.ref["vals"])
        st = rb.fp64_state(self.ref, _np(dst["final_T"]), _np(dst["n_contrib"]).view(np.uint32))
        rng = np.random.default_rng(seed)
        self.g = rng.standard_normal((3, H, W)).astype(np.float32)
        self.gD = rng.standard_normal((H, W)).astype(np.float32)
        self.gA = rng.standard_normal((H, W)).astype(np.float32)
        P = st["P"]
        z = np.asarray(st["depth"], np.float64)
        o = RasterOracle("f64")
        zero = np.zeros((H, W), np.float32)
        parts = [(st, self.g),
                 (dict(st, inputs=dict(st["inputs"], colors=np.stack([z, np.zeros(P), np.zeros(P)], 1), bg=np.zeros(3))),
                  np.stack([self.gD, zero, zero])),
                 (dict(st, inputs=dict(st["inputs"], colors=np.zeros((P, 3)), bg=np.array([-1.0, 0.0, 0.0]))),
                  np.stack([self.gA, zero, zero]))]
        wants, bounds = [], []
        for s, g in parts:
            w = o.backward_mag(s, g)
            wants.append(w)
            bounds.append({k: AUX_OPS * v for k, v in rb.grad_bounds(s, w, rb.device_depth(self.ref, w["nterm"])).items()})
        vrow = np.asarray(st["inputs"]["view"], np.float64).reshape(16)[[2, 6, 10]]
        vis = (st["radii"] > 0)[:, None]
        self.dz = wants[1]["dL_dcolors"][:, 0] * vis[:, 0]
        self.vrow = vrow
        self.want = {k: sum(w[k] for w in wants) for k in wants[0] if k.startswith("dL_") and k != "dL_dcolors"}
        self.want["dL_dcolors"] = wants[0]["dL_dcolors"]
        self.want["dL_dmeans3D"] = self.want["dL_dmeans3D"] + self.dz[:, None] * vrow[None]
        self.bounds = {k: sum(b[k] for b in bounds) for k in bounds[0] if k != "dL_dcolors"}
        self.bounds["dL_dcolors"] = bounds[0]["dL_dcolors"]
        dzb = bounds[1]["dL_dcolors"][:, 0]
        self.bounds["dL_dmeans3D"] = self.bounds["dL_dmeans3D"] + vis * (
            np.abs(vrow)[None] * dzb[:, None]
            + 2 * rb.U * (np.abs(self.want["dL_dmeans3D"]) + np.abs(vrow)[None] * np.abs(self.dz)[:, None]))
        self.shared, self.own, _ = rb.exempt_sets(st, _threads())

    def device_grads(self, deterministic=False, gD=None, gA=None):
        cu = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
        got = self.rc.backward(cu(self.g), want_cov3D=True, deterministic=deterministic,
                               grad_depth=cu(self.gD if gD is None else gD), grad_alpha=cu(self.gA if gA is None else gA))
        torch.cuda.synchronize()
        return {k: _np(v) for k, v in got.items() if v is not None}

    def worst(self, got, keys=KEYS):
        """Worst error-to-bound ratio over the non-exempt Gaussians, per tensor."""
        clean = ~(self.shared | self.own)
        out = {}
        for k_got, k_ref in keys:
            if got.get(k_got) is None:
                continue
            a = got[k_got][:, :2] if k_got == "dL_dmeans2D" else got[k_got]
            r = rb.ratios(a, self.want[k_ref], self.bounds[k_ref])
            out[k_got] = float(r[clean].max()) if clean.any() else 0.0
            per = grad_err(a, self.want[k_ref])
            mx = lambda msk: float(per[msk].max()) if msk.any() else 0.0
            out[k_got + ":shared_own"] = (mx(self.shared), mx(self.own))
        return out

    def check(self, tag, got, keys=KEYS):
        w = self.worst(got, keys)
        record(f"{tag}:aux_grad_bound", **{k: v for k, v in w.items() if ":" not in k})
        for k, v in w.items():
            if ":" in k:
                assert v[0] <= SHARED_TOL and v[1] <= TAINT_CAP, (tag, k, v)
            else:
                assert v <= 1.0, (tag, k, v)
        return w


def _check_scene(tag, sc, seed, planted=False, keys=KEYS):
    t = _AuxTruth(sc, seed)
    t.check(tag, t.device_grads(), keys)
    det = t.device_grads(deterministic=True)
    t.check(tag + ":det", det, keys)
    if planted:
        bad = t.device_grads(gA=-t.gA)                                        # g_A with the wrong sign
        assert max(v for k, v in t.worst(bad, keys).items() if ":" not in k) > 1.0, tag
        bad = t.device_grads(gD=t.gD * np.float32(1 + 1e-3))                  # g_D scaled by 1 + 1e-3
        assert max(v for k, v in t.worst(bad, keys).items() if ":" not in k) > 1.0, tag
        good = t.device_grads()                                               # the depth term dropped from dL/dmeans3D
        good["dL_dmeans3D"] = good["dL_dmeans3D"] - t.dz[:, None] * t.vrow[None]
        assert t.worst(good, keys)["dL_dmeans3D"] > 1.0, tag
    return t


def test_c1_aux_within_the_bound_and_planted_errors_fail_it():
    _check_scene("C1", synth.random_cube_scene(10_000, 256), 0, planted=True)


@pytest.mark.parametrize("res,P,spread,mul,bg,cam", [
    (100, 1500, 0.5, 4.0, (0.3, 0.6, 0.9), {}),
    (64, 300, 0.3, 10.0, (0.3, 0.6, 0.9), {}),
    (64, 1500, 0.6, 4.0, (0.3, 0.6, 0.9), dict(width=250, height=40, focal=(240.0, 190.0), principal=(118.0, 23.0),
                                               scale_modifier=0.7)),
    (64, 1500, 0.6, 4.0, (0.0, 0.0, 0.0), dict(width=40, height=250, focal=(150.0, 260.0), principal=(21.0, 130.0),
                                               scale_modifier=1.6)),
    (64, 3000, 3.0, 5.0, (0.0, 0.0, 0.0), dict(width=120, height=48, focal=(70.0, 52.0), principal=(66.0, 20.0),
                                               scale_modifier=1.3)),
    (48, 30000, 0.25, 1.0, (0.0, 0.0, 0.0), {}),
], ids=["100-1500", "64-300-saturated-bg", "250x40-mod0.7", "40x250-mod1.6", "120x48-clamp-mod1.3", "48-30000-radix-tile"])
def test_edge_shapes_aux_within_the_bound(res, P, spread, mul, bg, cam):
    sc = synth.random_cube_scene(P, res, spread=spread, scale_mul=mul, bg=bg, seed=13, **cam)
    _check_scene(f"edge-{res}-{P}", sc, 3, planted=(P == 1500 and not cam))


def test_cov3d_precomp_aux_within_the_bound():
    sc = synth.random_cube_scene(3000, 128, seed=5)
    _, ref = oracle_forward(sc, "f32", render=False)
    _check_scene("cov3D_precomp", dict(sc, cov3D_precomp=ref["cov3D"].copy(), scales=None, rots=None), 1,
                 keys=tuple(k for k in KEYS if k[0] not in ("dL_dscales", "dL_drots")))


def test_c2_aux_within_the_bound():
    _check_scene("C2", synth.stereo_pair_scene(1024), 5)


_DET_SCRIPT = r"""
import sys, numpy as np, torch
sys.path.insert(0, sys.argv[1]); sys.path.insert(0, sys.argv[1] + "/tests")
from gps_gaussian_b200 import synth
from gps_gaussian_b200.introspect import RasterCall
sc = synth.random_cube_scene(10_000, 256, seed=int(sys.argv[2]))
rc = RasterCall(sc)
d = torch.empty(sc["H"], sc["W"], device="cuda"); a = torch.empty_like(d)
rc.forward(out_depth=d, out_alpha=a)
rng = np.random.default_rng(1)
g = torch.from_numpy(rng.standard_normal((3, sc["H"], sc["W"])).astype(np.float32)).cuda()
gD = torch.from_numpy(rng.standard_normal((sc["H"], sc["W"])).astype(np.float32)).cuda()
gA = torch.from_numpy(rng.standard_normal((sc["H"], sc["W"])).astype(np.float32)).cuda()
out = rc.backward(g, want_cov3D=True, deterministic=True, grad_depth=gD, grad_alpha=gA)
np.savez(sys.argv[3], depth=d.cpu().numpy(), alpha=a.cpu().numpy(), color=rc.color.cpu().numpy(),
         **{k: v.cpu().numpy() for k, v in out.items() if v is not None})
"""


def test_deterministic_aux_backward_bitwise_equal_on_radix_and_bucket_binning(tmp_path):
    """GPSG_BINNING=radix against the default tile-bucket path: the aux forward outputs and the deterministic aux
    gradients are bit-identical (each run in its own process: the binning switch is read once per process)."""
    res = {}
    for name, binning in (("bucket", None), ("radix", "radix")):
        env = dict(os.environ)
        env.pop("GPSG_BINNING", None)
        if binning:
            env["GPSG_BINNING"] = binning
        path = str(tmp_path / f"{name}.npz")
        r = subprocess.run([sys.executable, "-c", _DET_SCRIPT, ROOT, "7", path], env=env, cwd=ROOT, capture_output=True,
                           text=True, timeout=600)
        assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
        res[name] = np.load(path)
    a, b = res["bucket"], res["radix"]
    assert sorted(a.files) == sorted(b.files)
    for k in a.files:
        assert np.array_equal(a[k].view(np.uint32), b[k].view(np.uint32)), k
