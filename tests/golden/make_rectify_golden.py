"""Generate tests/golden/rectify_golden.npz from cv2 and the REFERENCE's own loader functions.

    python tests/golden/make_rectify_golden.py          (after __graft_entry__.build() has staged oracle/_ref)

For each case, the inputs (images, masks, K, extrinsics, the pts2depth depth of both views), the cv2.stereoRectify
results and what StereoHumanDataset.get_rectified_stereo_data and stereo_to_dict_tensor (lib/human_loader.py:245-366)
return for them, called unbound on a stand-in `self` that carries only opt.src_res.  Cases (tests/rectify_cases.py):
  ring      : seeded ring pair at 22.5 deg, own K per view, soft mask edges, inverse depth on a zero background;
  wide      : 60 deg with a tilt, so the maps leave the source image;
  nonsquare : 96 x 160 input, 128 x 128 output, no pts (the loader's depth2pts needs square depth);
  empty     : an all-zero mask, with pts.
"""
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))
from gps_gaussian_b200 import harness  # noqa: E402
import rectify_cases  # noqa: E402

CASES = {  # name: (seed, Hin, Win, src_res, angle, tilt, empty mask, with pts)
    "ring": (11, 96, 96, 96, 22.5, 0.0, False, True),
    "wide": (12, 96, 96, 96, 60.0, 8.0, False, True),
    "nonsquare": (13, 96, 160, 128, 22.5, 0.0, False, False),
    "empty": (14, 64, 64, 64, 22.5, 0.0, True, True),
}


def main():
    harness.add_reference_to_path()
    from lib import human_loader as hl
    out = {}
    for name, (seed, Hin, Win, res, angle, tilt, empty, with_pts) in CASES.items():
        views = rectify_cases.pair(seed, Hin, Win, angle=angle, tilt=tilt, empty=empty)
        rng = np.random.default_rng(seed + 100)
        data = []
        for img, mask, K, E in views:
            pts = hl.depth2pts(torch.FloatTensor(rectify_cases.inv_depth(Hin, rng)), torch.FloatTensor(E),
                               torch.FloatTensor(K)) if with_pts else None
            data.append((img, mask, K, E, pts))
        me = types.SimpleNamespace(opt=types.SimpleNamespace(src_res=res))
        st = hl.StereoHumanDataset.get_rectified_stereo_data(me, data[0], data[1])
        item = hl.StereoHumanDataset.stereo_to_dict_tensor(me, st, name)
        R0, R1, P0, P1 = rectify_cases.stereo_rectify(views[0][2], views[0][3], views[1][2], views[1][3], res)
        p = f"{name}/"
        for k in range(2):
            img, mask, K, E, pts = data[k]
            out.update({p + f"in_img{k}": img, p + f"in_mask{k}": mask, p + f"K{k}": K, p + f"E{k}": E})
            if with_pts:
                cam = st["camera"]
                d = hl.pts2depth(torch.FloatTensor(pts), torch.FloatTensor(cam[f"extr{k}"]), torch.FloatTensor(cam[f"intr{k}"]))
                out[p + f"depth{k}"] = d.numpy()
                out[p + f"flow{k}"], out[p + f"valid{k}"] = st[f"flow{k}"], st[f"valid{k}"]
            out[p + f"img{k}"], out[p + f"mask{k}"] = st[f"img{k}"], st[f"mask{k}"]
            view = item["lmain" if k == 0 else "rmain"]
            out[p + f"img_t{k}"], out[p + f"mask_t{k}"] = view["img"].numpy(), view["mask"].numpy()
        for key, v in (("R0", R0), ("R1", R1), ("P0", P0), ("P1", P1), ("Tf_x", st["camera"]["Tf_x"]),
                       ("src_res", np.array(res))):
            out[p + key] = v
        print(name, {k: (v.dtype, v.shape) for k, v in st.items() if k != "camera"})
    np.savez_compressed(os.path.join(HERE, "rectify_golden.npz"), **out)


if __name__ == "__main__":
    main()
