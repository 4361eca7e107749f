"""Stage-1 training and the real-data script on hardware: the reference's OWN depth-only model, optimisation step and
entry scripts against the drop-ins, with the `taichi` stand-in running the validation preview on csrc/point_splat.cu.

  (a) train_stage1.py:56-74 executed statement for statement (fp32 RAFT, GradScaler disabled): finite loss, finite
      gradients that reach the RAFT update block;
  (b) the fp32 disparity after 3 GRU iterations through `corr_implementation='reg_cuda'` (our `corr_sampler` on an fp32
      volume) equals the reference's pure-PyTorch 'reg', under a bound derived below;
  (c) `train_stage1.py` (3 steps, one eval with its preview JPEG), then `train_stage2.py` warm-started from its
      checkpoint, then `test_real_data.py` on that checkpoint, as subprocesses -- with and without GPSG_PATCH=1.
"""
import glob
import math
import os

import pytest
import torch

from gps_gaussian_b200 import harness

pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(harness.staged_reference() is None,
                                 reason="oracle/_ref not staged (run __graft_entry__.build() where the original project is checked out)")]

RES = 256
N_VAL = 2           # train_stage1.py's eval draws from int(len(val_loader) / val_boost) batches of 2: one sample gives 0


@pytest.fixture(scope="module")
def dataset(tmp_path_factory):
    from gps_gaussian_b200 import synth_dataset
    root = str(tmp_path_factory.mktemp("stage1data"))
    synth_dataset.write_dataset(root, n_train=2, n_val=N_VAL, res=RES, hr=True)
    return root


def _state(dataset, corr=None, seed=1314):
    cfg = harness.load_cfg(dataset, stage=1, src_res=RES, num_steps=3, batch_size=2)
    assert not cfg.raft.mixed_precision                                            # config/stage1.yaml: fp32
    if corr is not None:
        cfg.defrost()
        cfg.raft.corr_implementation = corr
        cfg.freeze()
    return harness.Stage1State(cfg, seed=seed)


def test_stage1_step_finite_and_raft_gets_gradients(dataset):
    st = _state(dataset)
    assert not st.scaler.is_enabled()
    out = harness.stage1_step(st, st.batch(0))
    assert math.isfinite(float(out["loss"])) and math.isfinite(float(out["grad_norm"]))
    with_grad = [(n, p) for n, p in st.model.named_parameters() if p.grad is not None]
    assert all(bool(torch.isfinite(p.grad).all()) for _, p in with_grad)
    raft = sum(p.numel() for n, p in with_grad if n.startswith("raft_stereo."))
    assert raft > 1_000_000
    upd = float(sum(p.grad.abs().sum() for p in st.model.raft_stereo.update_module.parameters() if p.grad is not None))
    assert upd > 0
    print(f"stage-1 step: flow_loss {float(out['flow_loss']):.4f}, grad norm {float(out['grad_norm']):.4e}, "
          f"{raft} RAFT parameters with gradients")


def test_stage1_flow_reg_cuda_equals_reg_fp32(dataset, monkeypatch):
    """Same seed => same weights; same batch; only the correlation lookup differs, both in fp32.  TF32 is off for this
    comparison (PyTorch runs cuDNN convolutions in TF32 by default, whose 10-bit mantissa would re-round any fp32
    difference to 2^-11, as coarse as fp16), so every op of both runs is fp32."""
    harness.add_reference_to_path()
    import core.corr
    shapes = []
    plain = core.corr.CorrBlock1D.corr

    def corr_recording_shape(fmap1, fmap2):
        out = plain(fmap1, fmap2)
        shapes.append(tuple(out.shape))
        return out
    monkeypatch.setattr(core.corr.CorrBlock1D, "corr", staticmethod(corr_recording_shape))
    monkeypatch.setattr(torch.backends.cudnn, "allow_tf32", False)
    monkeypatch.setattr(torch.backends.cuda.matmul, "allow_tf32", False)
    flows = {}
    for corr in ("reg", "reg_cuda"):
        st = _state(dataset, corr=corr)
        data = st.batch(0)
        with torch.no_grad():
            data, flow_loss, _ = st.model(data, is_train=True)
        flows[corr] = (torch.cat([data["lmain"]["flow_pred"], data["rmain"]["flow_pred"]]), float(flow_loss))
        del st
    assert flows["reg"][0].dtype == torch.float32 and flows["reg_cuda"][0].dtype == torch.float32
    a, b = flows["reg"][0].double(), flows["reg_cuda"][0].double()
    err = float((a - b).abs().max())
    mag = float(a.abs().max())
    # Stage 2's bound, 5e-3 * max(1, |flow|), covers lookups of an fp16 volume: every value rounded to 2^-11 relative.
    # Here both runs build the same fp32 volume (core/corr.py einsum) and differ only in the lookup.  'reg' interpolates
    # with grid_sample, which maps x in [0, W2-1] to [-1, 1] and back; that round trip moves x by up to ~4 ulps of W2, i.e.
    # a relative error of 4 * W2 * 2^-24 in the interpolated value.  Scale stage 2's bound by that ratio.
    W2 = shapes[0][-1]
    bound = 5e-3 * (4 * W2 * 2.0 ** -24) / 2.0 ** -11 * max(1.0, mag)
    print(f"stage-1 fp32 flow after 3 iters: max|reg|={mag:.3f}px, max|reg - reg_cuda|={err:.3e}px (bound {bound:.3e}, "
          f"W2={W2}); flow_loss {flows['reg'][1]:.6f} vs {flows['reg_cuda'][1]:.6f}")
    assert bound < 5e-3 * max(1.0, mag)
    assert err < bound, (err, bound)
    assert abs(flows["reg"][1] - flows["reg_cuda"][1]) < bound


def _same_bytes(work, names):
    for name in names:
        with open(os.path.join(work, name), "rb") as a, open(os.path.join(harness.REF_STAGED, name), "rb") as b:
            assert a.read() == b.read(), name


@pytest.mark.parametrize("patched", [False, True])
def test_stage1_stage2_real_data_scripts_run_unmodified(dataset, tmp_path, patched):
    import cv2
    work = harness.make_workdir(str(tmp_path / "work"), dataset, src_res=RES, num_steps=3, batch_size=2,
                                stage1=dict(src_res=RES, num_steps=3, batch_size=2))
    _same_bytes(work, ("train_stage1.py", "train_stage2.py", "test_real_data.py", "lib/TaichiRender.py", "lib/utils.py",
                       "core/corr.py"))
    # stage 1: 3 steps, eval (and preview) at step 2
    p = harness.run_script(work, "train_stage1.py", patch=patched, timeout=1500)
    assert p.returncode == 0, p.stdout[-3000:] + p.stderr[-6000:]
    assert "FINISHED TRAINING" in p.stdout
    exp1 = glob.glob(os.path.join(work, "experiments", "GPS-GS_stage1_*"))
    assert len(exp1) == 1
    ckpt1 = glob.glob(os.path.join(exp1[0], "ckpt", "*_final.pth"))
    assert len(ckpt1) == 1
    shows = glob.glob(os.path.join(exp1[0], "show", "*.jpg"))
    assert [os.path.basename(f) for f in shows] == ["2.jpg"], shows
    im = cv2.imread(shows[0])
    drawn = float((im.max(2) > 8).mean())
    print(f"stage-1 preview {im.shape}: mean {im.mean():.2f}, {drawn:.3f} of pixels drawn")
    assert im.shape == (RES, RES, 3) and im.mean() > 1.0 and drawn > 0.01
    # stage 2 warm-started from the stage-1 checkpoint (train_stage2.py:50-52)
    with open(os.path.join(work, "config", "stage2.yaml"), "w") as f:
        f.write(harness.stage2_yaml(dataset, src_res=RES, num_steps=3, batch_size=2, stage1_ckpt=ckpt1[0]))
    q = harness.run_script(work, "train_stage2.py", patch=patched, timeout=1500)
    assert q.returncode == 0, q.stdout[-3000:] + q.stderr[-6000:]
    assert "FINISHED TRAINING" in q.stdout and "Using checkpoint from stage1" in q.stderr
    ckpt2 = glob.glob(os.path.join(work, "experiments", "GPS-GS_stage2_*", "ckpt", "*_final.pth"))
    assert len(ckpt2) == 1
    sd = torch.load(ckpt2[0], map_location="cpu")
    assert sd["total_steps"] == 3 and all(bool(torch.isfinite(v).all()) for v in sd["network"].values() if v.is_floating_point())
    # the real-data script on that checkpoint: one novel view per sample
    r = harness.run_script(work, "test_real_data.py", ["--test_data_root", os.path.join(dataset, "val"), "--ckpt_path",
                                                       ckpt2[0], "--src_view", "0", "1"], patch=patched, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-6000:]
    imgs = sorted(glob.glob(os.path.join(work, "test_out", "*_novel.jpg")))
    assert len(imgs) == N_VAL, imgs
    for f in imgs:
        im = cv2.imread(f)
        assert im.shape == (2 * RES, 2 * RES, 3) and im.mean() > 1.0
