"""Generate tests/golden/harness_golden.npz from the REFERENCE's own config class and dataset loader.

Run with GPSG_REFERENCE naming a checkout of the original project:  python tests/golden/make_harness_golden.py
Records (i) the default config tree `config/stereo_human_config.py:ConfigStereoHuman` builds, the text of `config/stage2.yaml`
and the merged config, built with this repository's `yacs` stand-in; (ii) what `lib/human_loader.py:StereoHumanDataset`
returns for the synthetic dataset `synth_dataset.write_dataset(res=96)` writes, with a fingerprint of the files it read
(`dataset_fingerprint`: lossless files by decoded content, JPEG files by 8x8-block means of their decoded pixels)."""
import hashlib
import json
import os
import sys
import tempfile
from types import SimpleNamespace

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
RES = 96


JPEG_BLOCK = 8


def dataset_fingerprint(root):
    """What the loader reads from a dataset, independent of how an image codec library encodes it: (sha256 over the
    relative path and DECODED content of every lossless file -- .png pixels, .npy arrays -- in sorted order, the sorted
    relative paths of the .jpg files, their decoded pixels as 8x8-block means [n, h/8, w/8, 3] float32).  JPEG is lossy,
    so its pixels are compared within a tolerance rather than hashed."""
    import cv2
    h = hashlib.sha256()
    jpgs, thumbs = [], []
    for d, _, files in sorted(os.walk(root)):
        for f in sorted(files):
            p = os.path.join(d, f)
            rel = os.path.relpath(p, root)
            if f.endswith(".jpg"):
                img = cv2.imread(p, cv2.IMREAD_UNCHANGED).astype(np.float32)
                hh, ww = img.shape[0] // JPEG_BLOCK, img.shape[1] // JPEG_BLOCK
                jpgs.append(rel)
                thumbs.append(img[:hh * JPEG_BLOCK, :ww * JPEG_BLOCK].reshape(hh, JPEG_BLOCK, ww, JPEG_BLOCK, -1).mean((1, 3)))
                continue
            a = cv2.imread(p, cv2.IMREAD_UNCHANGED) if f.endswith(".png") else np.load(p) if f.endswith(".npy") else None
            assert a is not None, rel
            h.update(rel.encode())
            h.update(str((a.dtype.str, a.shape)).encode())
            h.update(np.ascontiguousarray(a).tobytes())
    by_shape = {}
    for rel, t in zip(jpgs, thumbs):
        by_shape.setdefault(t.shape, []).append((rel, t))
    return h.hexdigest(), by_shape


def loader_options(root):
    return SimpleNamespace(data_root=root, test_data_root=None, use_processed_data=False, source_id=[0, 1],
                           train_novel_id=[2, 3, 4], val_novel_id=[3], src_res=RES, use_hr_img=True, bg_color=[0, 0, 0],
                           znear=0.01, zfar=100.0, trans=[0.0, 0.0, 0.0], scale=1.0)


def main():
    ref = os.environ["GPSG_REFERENCE"]
    for p in (ref, os.path.join(ROOT, "gps-gaussian_b200", "dropin"), ROOT):
        sys.path.insert(0, p)
    from gps_gaussian_b200 import synth_dataset
    from config.stereo_human_config import ConfigStereoHuman
    from lib.human_loader import StereoHumanDataset
    out = {}
    c = ConfigStereoHuman()
    out["config_defaults_json"] = json.dumps(c.get_cfg())
    with open(os.path.join(ref, "config", "stage2.yaml")) as f:
        out["stage2_yaml"] = f.read()
    c.load(os.path.join(ref, "config", "stage2.yaml"))
    out["config_merged_json"] = json.dumps(c.get_cfg())

    with tempfile.TemporaryDirectory() as root:
        names = synth_dataset.write_dataset(root, n_train=2, n_val=1, res=RES, hr=True)
        digest, jpgs = dataset_fingerprint(root)
        out["dataset_lossless_digest"] = digest
        for k, (shape, items) in enumerate(sorted(jpgs.items())):
            out[f"dataset_jpg{k}_names_json"] = json.dumps([rel for rel, _ in items])
            out[f"dataset_jpg{k}_blocks"] = np.stack([t for _, t in items])
        opt = loader_options(root)
        ds = StereoHumanDataset(opt, phase="train")
        out["sample_list_json"] = json.dumps(list(ds.sample_list))
        out["names_train_json"] = json.dumps(list(names["train"]))
        item = ds.get_item(0, novel_id=[3])
        for v in ("lmain", "rmain"):
            d = item[v]
            for k in ("flow", "valid", "intr", "extr", "ref_intr", "Tf_x"):
                out[f"{v}_{k}"] = np.asarray(d[k].numpy(), np.float32)
            out[f"{v}_img_shape"] = np.array(d["img"].shape)
            out[f"{v}_img_range"] = np.array([float(d["img"].min()), float(d["img"].max())], np.float32)
            out[f"{v}_mask_shape"] = np.array(d["mask"].shape)
        out["novel_img_shape"] = np.array(item["novel_view"]["img"].shape)
        out["novel_width"] = np.array(int(item["novel_view"]["width"]))
        opt.test_data_root = os.path.join(root, "val")
        t = StereoHumanDataset(opt, phase="test").get_test_item(0, source_id=[0, 1])
        out["test_lmain_intr_ori_shape"] = np.array(t["lmain"]["intr_ori"].shape)
        out["test_rmain_extr_ori_shape"] = np.array(t["rmain"]["extr_ori"].shape)
        out["test_novel_height"] = np.array(int(t["novel_view"]["height"]))
    np.savez_compressed(os.path.join(HERE, "harness_golden.npz"), **out)


if __name__ == "__main__":
    main()
