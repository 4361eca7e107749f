"""Dataset renderer on the GPU (csrc/mesh_render.cu): bit parity with the serial oracle on a procedural body and an
adversarial mesh, geometry checked with the reference's own `depth2pts`, the unmodified `prepare_data/render_data.py`
through the `taichi_three` stand-in, and one stage-1 training step on what it rendered."""
import math
import os
import pickle

import numpy as np
import pytest
import torch

import mesh_reference as mr
from gps_gaussian_b200 import harness, synth_mesh

pytestmark = pytest.mark.gpu
needs_ref = pytest.mark.skipif(harness.staged_reference() is None, reason="oracle/_ref is not staged")


def _u32(a):
    return np.ascontiguousarray(np.asarray(a, np.float32)).view(np.uint32)


def _device_render(cams, ld, lc, verts, faces, uvs=None, face_uvs=None, tex=None):
    from gps_gaussian_b200 import mesh_render
    t = lambda a, dt: None if a is None else torch.from_numpy(np.ascontiguousarray(a, dt)).cuda()
    outs = mesh_render.render(t(verts, np.float32), t(faces, np.int32), [c.render_camera() for c in cams], ld, lc,
                              t(uvs, np.float32), t(face_uvs, np.int32), t(tex, np.float32))
    torch.cuda.synchronize()
    return [tuple(x.cpu().numpy() for x in o) for o in outs]


def _assert_parity(cams, ld, lc, verts, faces, uvs=None, face_uvs=None, tex=None):
    got = _device_render(cams, ld, lc, verts, faces, uvs, face_uvs, tex)
    for cam, g in zip(cams, got):
        want = mr.oracle_render(cam, ld, lc, verts, faces, uvs, face_uvs, tex)
        for name, a, b in zip(("img", "zbuf", "mask"), g, want):
            assert a.shape == b.shape, name
            bad = _u32(a) != _u32(b)
            assert not bad.any(), (name, cam.res, int(bad.sum()), np.argwhere(bad)[:5].tolist())
    return got


def _texture(img_bgr):
    """render_data.py's texture transform (:102-104) and StaticModel's /255, as the stand-in uploads it."""
    return np.ascontiguousarray(img_bgr[:, :, ::-1]).swapaxes(0, 1)[:, ::-1, :].astype(np.float32) / 255


def test_parity_procedural_body_1024_and_2048():
    obj, tex_img = synth_mesh.procedural_scan(120_000, 1024, seed=7)
    f = obj["f"]
    assert len(f) >= 100_000
    cams = [mr.ring_camera(37.0), mr.ring_camera(37.0, hr=True), mr.ring_camera(211.5)]
    ld, lc = mr.lights(seed=3)
    args = (obj["vi"], f[:, :, 0], obj["vt"], f[:, :, 1], _texture(tex_img))
    got = _assert_parity(cams, ld, lc, *args)
    for (img, zbuf, mask), cam in zip(got, cams):
        assert mask[..., 0].sum() > 0.05 * cam.res[0] * cam.res[1] and img.max() > 0.1
    again = _device_render(cams, ld, lc, *args)
    for a, b in zip(got, again):
        assert all(x.tobytes() == y.tobytes() for x, y in zip(a, b))


def _square_or_not(res):
    from taichi_three import Camera
    cam = Camera(res=res)
    cam.set_intrinsic(0.8 * min(res), 0.8 * min(res), res[0] * 0.5, res[1] * 0.5 + 25)
    cam.set(pos=[0.0, 1.13, 1.98], target=[0.0, 0.85, 0.0])
    cam._init()
    return cam


@pytest.mark.parametrize("variant", ["textured", "no_vt", "no_texture", "nonfinite"])
def test_parity_adversarial_mesh(variant):
    verts, faces, uvs, fu = mr.adversarial_mesh(seed=11)
    tex = np.random.default_rng(2).uniform(0, 1, (37, 53, 3)).astype(np.float32)
    ld, lc = mr.lights(seed=5)
    if variant == "no_vt":
        uvs = fu = None
    if variant == "no_texture":
        tex = None
    if variant == "nonfinite":
        # NaN and infinite uvs, and a negative light colour that drives sqrt(mix(blue, orange, c)) below zero: NaN
        # colours must come out as the same canonical NaN on both sides
        uvs = uvs.copy()
        uvs[::7] = np.nan
        uvs[3::11, 0] = np.inf
        uvs[5::13, 1] = -np.inf
        lc = lc.copy()
        lc[0] = -2.0
    cams = [mr.ring_camera(0.0), _square_or_not((640, 480)), _square_or_not((480, 640))]
    got = _assert_parity(cams, ld, lc, verts, faces, uvs, fu, tex)
    if variant == "nonfinite":
        assert all(np.isnan(img).any() for img, _, _ in got)
    # the reference clamps the bbox end N.x to [0, res1]: with res0 > res1 the columns x >= res1 are never drawn, while
    # the full-screen faces cover every other pixel but row and column 0
    for (img, zbuf, mask), cam in zip(got, cams):
        m = mask[..., 0] > 0
        W, H = cam.res
        assert m[1:, 1:min(W, H)].mean() > 0.99 and not m[:, H:].any()
        assert not m[0, :].any() and not m[:, 0].any()
    # both raster paths are taken: faces bigger and smaller than one 16x16 tile
    rast = mr.ring_camera(0.0)
    A = _screen(rast, verts[faces])
    area = np.ptp(A[..., 0], axis=1) * np.ptp(A[..., 1], axis=1)
    assert (area > 4096).any() and (area[np.isfinite(area)] < 100).sum() > 1000
    again = _device_render(cams, ld, lc, verts, faces, uvs, fu, tex)
    for a, b in zip(got, again):
        assert all(x.tobytes() == y.tobytes() for x, y in zip(a, b))


def _screen(cam, pts):
    R = np.array(cam._dev_inv_rot, np.float64).reshape(3, 3)
    p = (pts.astype(np.float64) - np.array(cam._dev_pos)) @ R.T
    fx, fy, cx, cy = cam._dev_K
    with np.errstate(all="ignore"):
        return np.stack([(fx * p[..., 0] + cx * p[..., 2]) / np.abs(p[..., 2]),
                         (fy * p[..., 1] + cy * p[..., 2]) / np.abs(p[..., 2])], -1)


def _standin_render(obj, tex, angles, res=(1024, 1024)):
    """Render through the stand-in's Scene / StaticModel / Camera like render_data.py does; returns per angle
    (extrinsic, intrinsic, zbuf, img, mask) in image layout."""
    import taichi_three as t3
    scene = t3.Scene()
    model = t3.StaticModel(2 * len(obj["f"]), obj=obj, tex=tex)
    scene.add_model(model)
    cam = t3.Camera(res=res)
    scene.add_camera(cam)
    scene.add_lights(t3.Lights([t3.Light([0, 0, 1], color=[1.0, 1.0, 1.0])]))
    out = []
    for a in angles:
        ref = mr.ring_camera(a, res)
        cam.set_intrinsic(*ref._dev_K)
        cam.set(pos=ref.eye, target=ref.target)
        cam._init()
        scene.render()
        out.append((cam.export_extrinsic(), cam.export_intrinsic(), cam.zbuf.to_numpy().swapaxes(0, 1),
                    cam.img.to_numpy().swapaxes(0, 1), cam.mask.to_numpy().swapaxes(0, 1)))
    return out


@needs_ref
def test_sphere_geometry_through_reference_depth2pts():
    harness.add_reference_to_path()
    from lib.human_loader import depth2pts
    centre, r = np.array([0.0, 0.85, 0.0]), 0.4
    nlat, nlon = 96, 192
    v, f, t = synth_mesh.uv_sphere(tuple(centre), r, nlat, nlon)
    obj = {"vi": v, "vt": t, "vn": None, "f": np.stack([f, f], -1)}
    views = _standin_render(obj, None, [0.0, 22.5])
    pts = []
    for E, K, zbuf, _, mask in views:
        depth = (zbuf * 2.0 ** 15).astype(np.uint16).astype(np.float32) / 2.0 ** 15      # render_data.save + read_depth
        m = mask[..., 0] > 0
        assert m.sum() > 50_000 and (depth[m] > 0).all()
        P = depth2pts(torch.from_numpy(depth), torch.FloatTensor(E), torch.FloatTensor(K)).numpy()[m].astype(np.float64)
        # bound: (1) depth2pts reads pixel (x, y) at (x + 0.5, y + 0.5), the rasterizer sampled it at (x, y): a lateral
        # offset of sqrt(2)/2 px, i.e. sqrt(2)/2 * z / f in space; (2) the chord error of the facets, at most
        # r (1 - cos(dtheta)) with dtheta = pi / nlat, and the screen-affine depth of a facet, at most dz^2 / (4 z_min)
        # with dz <= r dtheta; (3) uint16 truncation of the inverse depth, 2^-15, i.e. z^2 2^-15 / (1 - z 2^-15) in depth
        # along a ray at most 1.3 times as long; (4) fp32 arithmetic of depth2pts
        z_max, z_min, fpx = 2.0 + r, 2.0 - r, K[0, 0]
        dth = math.pi / nlat
        bound = (math.sqrt(2) / 2 * z_max / fpx + r * (1 - math.cos(dth)) + (r * dth) ** 2 / (4 * z_min)
                 + 1.3 * z_max ** 2 * 2.0 ** -15 / (1 - z_max * 2.0 ** -15) + 1e-5)
        err = np.abs(np.linalg.norm(P - centre, axis=1) - r)
        assert err.max() <= bound, (float(err.max()), bound)
        pts.append(P)
    # every masked point of view 0 lies on the sphere, so it projects inside view 1's silhouette
    E1, K1, _, _, mask1 = views[1]
    q = (K1 @ (E1[:, :3] @ pts[0].T + E1[:, 3:])).T
    uv = q[:, :2] / q[:, 2:]
    m1 = mask1[..., 0] > 0
    xi, yi = np.floor(uv[:, 0]).astype(int), np.floor(uv[:, 1]).astype(int)
    inside = m1[np.clip(yi, 0, 1023), np.clip(xi, 0, 1023)]
    # the sample offset of (1) and the bound above move a projection by under 2 px near the silhouette
    grown = m1.copy()
    for dy in (-2, -1, 0, 1, 2):
        for dx in (-2, -1, 0, 1, 2):
            grown |= np.roll(np.roll(m1, dy, 0), dx, 1)
    assert inside.mean() > 0.98 and grown[np.clip(yi, 0, 1023), np.clip(xi, 0, 1023)].all()


# ---- the unmodified script --------------------------------------------------------------------------------------

# The val scan has more than twice the faces of the train scan, so the script's StaticRenderer outgrows its capacity N
# on the second scan: change_all() rebuilds the scene with a new StaticModel of the previous obj and texture, and
# modify_model() then swaps the new scan in and calls _init() (render_data.py:43-77).
SCANS = {"train": ("0001", 12_000), "val": ("0002", 40_000)}


def _scan_tree(root, tex_size=512):
    import cv2
    for k, (phase, (sid, n_faces)) in enumerate(SCANS.items()):
        obj, tex = synth_mesh.procedural_scan(n_faces, tex_size, seed=100 + k)
        d = os.path.join(root, "PATH", "TO", "THuman2.0", phase, sid)
        synth_mesh.write_obj(os.path.join(d, f"{sid}.obj"), obj)
        cv2.imwrite(os.path.join(d, "material0.jpeg"), tex)
        p = os.path.join(root, "PATH", "TO", "THuman2.0", "THuman2.0_Smpl_X_Paras", sid)
        os.makedirs(p, exist_ok=True)
        with open(os.path.join(p, "smplx_param.pkl"), "wb") as fh:
            pickle.dump({"global_orient": np.array([[0.05, 0.4 * (k + 1), -0.02]], np.float32)}, fh)
    return root


def _run_script(workdir):
    """`python <ref>/prepare_data/render_data.py` as a user runs it: the script's own directory, which holds the
    reference's `taichi_three`, comes first on sys.path, and GPSG_PATCH=1's import finder must still pick the stand-in."""
    import subprocess
    import sys
    _scan_tree(workdir)
    script = os.path.join(harness.staged_reference(), "prepare_data", "render_data.py")
    p = subprocess.run([sys.executable, script], cwd=workdir, env=harness.script_env(patch=True), text=True,
                       capture_output=True, timeout=1800)
    assert p.returncode == 0, p.stdout[-3000:] + p.stderr[-6000:]
    # StaticRenderer.change_all() prints 'init': once for the first scan, once when the second outgrows N
    assert p.stdout.splitlines().count("init") == 2, p.stdout[-2000:]
    return os.path.join(workdir, "PATH", "TO", "SAVE", "RENDERED", "DATA")


@pytest.fixture(scope="module")
def rendered(tmp_path_factory):
    if harness.staged_reference() is None:
        pytest.skip("oracle/_ref is not staged")
    return _run_script(str(tmp_path_factory.mktemp("render_a")))


@needs_ref
def test_render_data_script_runs_unmodified(rendered, tmp_path):
    import cv2
    for phase, (sid, _) in SCANS.items():
        for pid in range(16):
            name = f"{sid}_{pid:03d}"
            for vid in range(5):
                img = cv2.imread(os.path.join(rendered, phase, "img", name, f"{vid}.jpg"))
                assert img.shape == (1024, 1024, 3) and img.dtype == np.uint8
                hr = os.path.join(rendered, phase, "img", name, f"{vid}_hr.jpg")
                assert os.path.exists(hr) == (vid >= 2)
                if vid >= 2:
                    assert cv2.imread(hr).shape == (2048, 2048, 3)
                depth = cv2.imread(os.path.join(rendered, phase, "depth", name, f"{vid}.png"), cv2.IMREAD_UNCHANGED)
                mask = cv2.imread(os.path.join(rendered, phase, "mask", name, f"{vid}.png"), cv2.IMREAD_UNCHANGED)
                assert depth.shape == (1024, 1024) and depth.dtype == np.uint16
                assert mask.shape == (1024, 1024, 3) and mask.dtype == np.uint8
                on = mask[..., 0] == 255
                assert on.mean() > 0.03 and (depth[on] > 0).all() and (depth[~on] == 0).all()
                for kind, shape in (("intrinsic", (3, 3)), ("extrinsic", (3, 4))):
                    a = np.load(os.path.join(rendered, phase, "parm", name, f"{vid}_{kind}.npy"))
                    assert a.shape == shape and a.dtype == np.float64
    # a second run with the script's own seed writes the same bytes
    other = _run_script(str(tmp_path / "render_b"))
    files = sorted(os.path.relpath(os.path.join(d, f), rendered) for d, _, fs in os.walk(rendered) for f in fs)
    assert len(files) == 2 * 16 * (8 + 5 + 5 + 10)          # img (+3 _hr), depth, mask, parm
    for rel in files:
        with open(os.path.join(rendered, rel), "rb") as a, open(os.path.join(other, rel), "rb") as b:
            assert a.read() == b.read(), rel


@needs_ref
def test_rendered_data_trains_stage1(rendered):
    import shutil
    root = os.path.join(os.path.dirname(rendered), "train_root")
    shutil.copytree(rendered, root)
    cfg = harness.load_cfg(root, stage=1, src_res=1024, num_steps=3, batch_size=2)
    st = harness.Stage1State(cfg)
    data = st.batch(0)
    flow, valid = data["lmain"]["flow"], data["lmain"]["valid"]
    assert float(valid.sum()) > 1000 and float((flow.abs() * valid).sum()) > 0
    out = harness.stage1_step(st, data)
    assert math.isfinite(float(out["loss"])) and math.isfinite(float(out["grad_norm"]))
