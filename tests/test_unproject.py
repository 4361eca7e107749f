"""Fused unprojection (reference lib/utils.py:87-119 via lib/network.py:64-69): oracle vs the reference's golden
vectors on CPU; the sm_90a kernels vs golden + oracle on the GPU."""
import os

import numpy as np
import pytest
import torch

from oracle.unproject_oracle import unproject, unproject_backward

G = np.load(os.path.join(os.path.dirname(__file__), "golden", "unproject_golden.npz"))


def test_oracle_matches_reference_golden():
    depth, xyz, valid = unproject(G["flow"], G["mask"], G["intr"], G["extr"], G["ref_intr"], G["tf_x"])
    assert np.abs(depth - G["depth"]).max() < 1e-12
    assert np.array_equal(valid, G["valid"])
    v = G["valid"]
    assert np.abs(xyz[v] - G["xyz"][v]).max() < 1e-9                                   # invalid pixels have z = 1e8 garbage
    dflow = unproject_backward(G["depth"], G["mask"], G["intr"], G["extr"], G["tf_x"], G["g_xyz"], G["g_depth"])
    sc = np.abs(G["d_flow"]).max()
    assert np.abs(dflow - G["d_flow"])[G["valid"].reshape(G["d_flow"].shape)].max() < 1e-9 * sc


@pytest.mark.gpu
def test_kernel_matches_golden_and_autograd():
    from gps_gaussian_b200.unproject import unproject_view
    T = lambda k: torch.tensor(G[k], dtype=torch.float32, device="cuda")
    view = {"flow_pred": T("flow").requires_grad_(True), "mask": T("mask"), "intr": T("intr"), "extr": T("extr"),
            "ref_intr": T("ref_intr"), "Tf_x": T("tf_x")}
    depth, xyz, valid = unproject_view(view)
    assert depth.shape == (2, 1, 24, 24) and xyz.shape == (2, 576, 3) and valid.dtype == torch.bool
    assert np.array_equal(valid.cpu().numpy(), G["valid"])
    assert np.abs(depth.detach().cpu().numpy() - G["depth"]).max() < 1e-5 * np.abs(G["depth"]).max()
    v = G["valid"]
    assert np.abs(xyz.detach().cpu().numpy()[v] - G["xyz"][v]).max() < 2e-5 * np.abs(G["xyz"][v]).max()
    ((xyz * T("g_xyz")).sum() + (depth * T("g_depth")).sum()).backward()
    got = view["flow_pred"].grad.cpu().numpy()
    vm = G["valid"].reshape(G["d_flow"].shape)
    assert np.abs(got - G["d_flow"])[vm].max() < 1e-4 * np.abs(G["d_flow"][vm]).max()


@pytest.mark.gpu
def test_kernel_feeds_rasterizer_like_the_reference_pipeline():
    """flow2xyz(data) on a synthetic pair reproduces the xyz / pts_valid maps that synth.py derives with the same
    depth2pc arithmetic, at BASELINE size (1024^2)."""
    from gps_gaussian_b200 import synth
    from gps_gaussian_b200.unproject import flow2xyz
    S = 1024
    sc = synth.stereo_pair_scene(S, keep_maps=True)
    data = {}
    for name, vw in zip(("lmain", "rmain"), sc["views"]):
        z = vw["depth"]                                    # metric depth; the pipeline's "depth" is 1/z where valid
        inv = np.where(z > 0, 1.0 / np.maximum(z, 1e-6), 0.0).astype(np.float32)
        K = vw["K"].astype(np.float32)
        E = np.vstack([vw["E"], [0, 0, 0, 1]]).astype(np.float32)
        # choose Tf_x = -1, ref_intr = intr  =>  depth = flow * mask
        data[name] = {"flow_pred": torch.tensor(inv)[None, None].cuda(), "mask": torch.ones(1, 3, S, S, device="cuda"),
                      "intr": torch.tensor(K)[None].cuda(), "extr": torch.tensor(E)[None].cuda(),
                      "ref_intr": torch.tensor(K)[None].cuda(), "Tf_x": torch.tensor([1.0], device="cuda")}
    flow2xyz(data)
    for name, vw in zip(("lmain", "rmain"), sc["views"]):
        valid = data[name]["pts_valid"][0].cpu().numpy()
        assert np.array_equal(valid, vw["valid"])
        got = data[name]["xyz"][0].cpu().numpy()[valid]
        assert np.abs(got - vw["xyz"][valid]).max() < 1e-4
