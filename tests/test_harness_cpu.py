"""Harness items of SURVEY.md 8f-4 on the CPU, pinned to what the UNMODIFIED reference produced: the `yacs` stand-in rebuilds
the reference's own config (default tree of `config/stereo_human_config.py` + `config/stage2.yaml`, recorded in
tests/golden/harness_golden.npz by tests/golden/make_harness_golden.py), the synthetic dataset writer produces exactly the files
the reference's own `StereoHumanDataset` was recorded reading, and the flow it returned unprojects onto the analytic surface.
The C3 harness builds the reference's own model and batch from the tree the oracle recipe staged in oracle/_ref.
The import hook and `patch.install()` are checked on stand-in modules with the reference's module names and import structure."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DROPIN = os.path.join(ROOT, "gps-gaussian_b200", "dropin")
G = np.load(os.path.join(ROOT, "tests", "golden", "harness_golden.npz"))
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
from make_harness_golden import RES, dataset_fingerprint  # noqa: E402

# the reference's module layout as the patch sees it: core.corr defines the two classes, core.raft_stereo_human copies one
# of them with `from core.corr import ...` (core/raft_stereo_human.py:6), lib.GaussianRender defines pts2render
STANDINS = {
    "core/__init__.py": "",
    "core/corr.py": "class CorrSampler:\n    pass\n\n\nclass CorrBlockFast1D:\n    pass\n",
    "core/raft_stereo_human.py": "from core.corr import CorrBlockFast1D\n",
    "lib/__init__.py": "",
    "lib/GaussianRender.py": "def pts2render(data, bg_color):\n    return data\n",
}


def _write_standins(root):
    for rel, text in STANDINS.items():
        path = os.path.join(str(root), rel)
        os.makedirs(os.path.dirname(path), exist_ok=True)
        with open(path, "w") as f:
            f.write(text)
    return str(root)


def test_yacs_standin_loads_the_reference_config(tmp_path):
    if DROPIN not in sys.path:
        sys.path.insert(0, DROPIN)
    import yacs.config
    from yacs.config import CfgNode
    assert yacs.config.__file__.startswith(DROPIN)                  # ours, not an installed yacs
    c = CfgNode(json.loads(str(G["config_defaults_json"])))          # the tree ConfigStereoHuman() builds
    yml = tmp_path / "stage2.yaml"
    yml.write_text(str(G["stage2_yaml"]))
    c.defrost()                                                      # ConfigStereoHuman.load
    c.merge_from_file(str(yml))
    c.freeze()
    cfg = c.clone()                                                  # ConfigStereoHuman.get_cfg
    assert json.loads(json.dumps(cfg)) == json.loads(str(G["config_merged_json"]))
    assert cfg.batch_size == 2 and cfg.restore_ckpt is None and abs(cfg.wdecay - 1e-5) < 1e-12      # 'None' / '1e-5' decoded
    assert cfg.raft.mixed_precision is True and cfg.raft.hidden_dims == [96, 96, 96] and cfg.dataset.use_hr_img is True
    assert cfg.raft.corr_implementation == "reg_cuda" and cfg.dataset.znear == 0.01                 # defaults survive
    with pytest.raises(AttributeError):
        cfg.exp_name = "x"                                                                          # frozen after load
    cfg.defrost()
    cfg.exp_name = "x"
    cfg.record.ckpt_path = "p"                                                                      # train_stage2.py:192-199
    cfg.freeze()
    assert json.loads(json.dumps(cfg))["record"]["ckpt_path"] == "p"                                # lib/train_recoder.py:24
    with pytest.raises(KeyError):
        cfg.clone().merge_from_list(["no.such.key", 1])


def test_synthetic_dataset_is_read_by_the_reference_loader(tmp_path):
    from gps_gaussian_b200 import synth_dataset
    from oracle import unproject_oracle
    names = synth_dataset.write_dataset(str(tmp_path), n_train=2, n_val=1, res=RES, hr=True)
    # the writer still produces the files the reference loader was recorded reading: identical lossless content (masks,
    # depth maps, calibration) and JPEG images whose decoded 8x8-block means agree within 2/255 (codec versions may differ)
    digest, jpgs = dataset_fingerprint(str(tmp_path))
    assert digest == str(G["dataset_lossless_digest"])
    k_all = sorted(int(k[len("dataset_jpg"):-len("_blocks")]) for k in G.files if k.startswith("dataset_jpg") and k.endswith("_blocks"))
    assert len(k_all) == len(jpgs) > 0
    for k, (shape, items) in zip(k_all, sorted(jpgs.items())):
        assert [rel for rel, _ in items] == json.loads(str(G[f"dataset_jpg{k}_names_json"]))
        assert np.abs(np.stack([t for _, t in items]) - G[f"dataset_jpg{k}_blocks"]).max() <= 2.0
    assert names["train"] == json.loads(str(G["names_train_json"])) == json.loads(str(G["sample_list_json"]))
    for v in ("lmain", "rmain"):
        assert tuple(G[f"{v}_img_shape"]) == (3, RES, RES) and tuple(G[f"{v}_mask_shape"]) == (3, RES, RES)
        assert G[f"{v}_flow"].shape == (1, RES, RES) and G[f"{v}_valid"].shape == (1, RES, RES)
        lo, hi = G[f"{v}_img_range"]
        assert float(G[f"{v}_valid"].mean()) > 0.1 and -1.0 <= lo and hi <= 1.0
    assert tuple(G["novel_img_shape"]) == (3, 2 * RES, 2 * RES) and int(G["novel_width"]) == 2 * RES     # _hr image of view 3
    # flow (reference rectification + stereo_pts2flow) -> depth -> points (our oracle of flow2depth + depth2pc):
    # every valid point must lie on the capsule that was rendered (radius of sample 0, axis x = z = 0).
    radii = np.random.default_rng(synth_dataset.synth.SEED)
    r0 = 0.425 * float(radii.uniform(0.9, 1.05))
    for v in ("lmain", "rmain"):
        g = lambda k: G[f"{v}_{k}"].astype(np.float64)
        flow, valid = g("flow")[None], g("valid")[None]
        depth, xyz, pv = unproject_oracle.unproject(flow, np.repeat(valid, 3, 1), g("intr")[None], g("extr")[None],
                                                    g("ref_intr")[None], g("Tf_x").reshape(1))
        pts = xyz[0][pv[0]]
        mid = pts[(pts[:, 1] > r0 + 0.05) & (pts[:, 1] < 1.8 - r0 - 0.05)]            # cylinder part of the capsule
        assert mid.shape[0] > 200
        rad = np.sqrt(mid[:, 0] ** 2 + mid[:, 2] ** 2)
        assert abs(np.median(rad) - r0) < 0.01 and np.percentile(np.abs(rad - r0), 90) < 0.03, (np.median(rad), r0)
    # the test-time path (test_view_interp.py): original calibration for get_novel_calib
    assert tuple(G["test_lmain_intr_ori_shape"]) == (3, 3) and tuple(G["test_rmain_extr_ori_shape"]) == (3, 4)
    assert int(G["test_novel_height"]) == 2 * RES


def test_import_hook_rebinds_the_reference_entry_points(tmp_path):
    """GPSG_PATCH=1 + dropin/ on PYTHONPATH: `sitecustomize` installs the post-import hook, the reference's
    `from core.corr import CorrBlockFast1D` / `from lib.GaussianRender import pts2render` resolve to the fused paths;
    without the variable nothing is touched."""
    ref = _write_standins(tmp_path / "ref")
    code = ("import core.raft_stereo_human as r, core.corr as c\n"
            "from lib.GaussianRender import pts2render\n"
            "print(r.CorrBlockFast1D.__module__, c.CorrSampler.__module__, pts2render.__module__)\n")
    out = {}
    for flag in ("0", "1"):
        env = dict(os.environ, PYTHONPATH=os.pathsep.join([DROPIN, ref, ROOT]), GPSG_PATCH=flag)
        p = subprocess.run([sys.executable, "-c", code], env=env, cwd=str(tmp_path), capture_output=True, text=True)
        assert p.returncode == 0, p.stderr[-2000:]
        out[flag] = p.stdout.split()
    assert out["0"] == ["core.corr", "core.corr", "lib.GaussianRender"]
    assert out["1"] == ["gps_gaussian_b200.corr", "gps_gaussian_b200.corr", "gps_gaussian_b200.GaussianRender"]


@pytest.mark.skipif(not os.path.isfile(os.path.join(ROOT, "oracle", "_ref", "train_stage2.py")),
                    reason="oracle/_ref not staged (run __graft_entry__.build() where the original project is checked out)")
def test_c3_harness_builds_the_reference_model_and_batch_on_cpu(tmp_path):
    """Plumbing of gps_gaussian_b200.harness without a GPU: staging, config, the reference's loader + model (the
    pure-PyTorch 'reg' correlation path), one forward.  The GPU half is tests/test_c3_gpu.py."""
    import torch
    from gps_gaussian_b200 import harness, synth_dataset
    assert harness.staged_reference() == os.path.join(ROOT, "oracle", "_ref")
    for name in ("train_stage2.py", "core/corr.py", "lib/GaussianRender.py", "gaussian_renderer/__init__.py"):
        assert os.path.isfile(os.path.join(harness.REF_STAGED, name))     # the tree the oracle recipe staged
    root = str(tmp_path / "data")
    synth_dataset.write_dataset(root, n_train=2, n_val=1, res=128, hr=True)
    cfg = harness.load_cfg(root, src_res=128, num_steps=3, batch_size=2, corr_implementation="reg")
    assert cfg.stage1_ckpt is None and cfg.num_steps == 3 and cfg.dataset.data_root == root
    st = harness.C3State(cfg, device="cpu")
    data = st.batch(0)
    assert tuple(data["lmain"]["img"].shape) == (2, 3, 128, 128) and tuple(data["novel_view"]["img"].shape) == (2, 3, 256, 256)
    data, flow_loss, metrics = st.model(data, is_train=True)
    assert tuple(data["lmain"]["xyz"].shape) == (2, 128 * 128, 3) and data["rmain"]["pts_valid"].dtype == torch.bool
    assert bool(torch.isfinite(flow_loss)) and "train_epe" in metrics


def test_patch_install_and_uninstall_in_process(tmp_path):
    """`patch.install()` rebinds modules that are ALREADY imported (incl. the `from core.corr import ...` copy held by
    core.raft_stereo_human); `patch.uninstall()` puts the reference's own objects back."""
    from gps_gaussian_b200 import patch
    ref = _write_standins(tmp_path / "ref")
    names = ("core", "core.corr", "core.raft_stereo_human", "lib", "lib.GaussianRender")
    saved = {n: sys.modules.pop(n) for n in names if n in sys.modules}
    sys.path.insert(0, ref)
    try:
        import core.corr
        import core.raft_stereo_human
        import lib.GaussianRender
        orig = (core.corr.CorrBlockFast1D, core.corr.CorrSampler, core.raft_stereo_human.CorrBlockFast1D,
                lib.GaussianRender.pts2render)
        assert all(o.__module__ in ("core.corr", "lib.GaussianRender") for o in orig)
        patch.install()
        try:
            assert patch.active()
            assert core.corr.CorrBlockFast1D.__module__ == "gps_gaussian_b200.corr"
            assert core.raft_stereo_human.CorrBlockFast1D is core.corr.CorrBlockFast1D
            assert lib.GaussianRender.pts2render.__module__ == "gps_gaussian_b200.GaussianRender"
            patch.install()                                               # idempotent
        finally:
            patch.uninstall()
        assert not patch.active()
        assert (core.corr.CorrBlockFast1D, core.corr.CorrSampler, core.raft_stereo_human.CorrBlockFast1D,
                lib.GaussianRender.pts2render) == orig
    finally:
        sys.path.remove(ref)
        for n in names:
            sys.modules.pop(n, None)
        sys.modules.update(saved)
