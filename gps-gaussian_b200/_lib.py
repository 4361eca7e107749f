"""ctypes binding of libgpsg_sm90.so (the C ABI declared in include/gpsg.h).

There is NO fallback: if the shared library is missing this module raises at import time --
a product path that silently ran on the CPU oracle or on eager PyTorch would void every parity
claim.  Build it with `python gps-gaussian_b200/build.py` (or `__graft_entry__.build()`).
GPSG_LIB_PATH, if set, names another build of the same library to load (an instrumented variant, tools/sort_phases.py).
"""
import ctypes as C
import os
import threading

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("GPSG_LIB_PATH") or os.path.join(_HERE, "lib", "libgpsg_sm90.so")


class GpsgError(RuntimeError):
    pass


class RasterSettings(C.Structure):
    """GpsgRasterSettings (include/gpsg.h) == the 12 fields of GaussianRasterizationSettings."""
    _fields_ = [("image_height", C.c_int32), ("image_width", C.c_int32), ("tanfovx", C.c_float),
                ("tanfovy", C.c_float), ("bg", C.c_float * 3), ("scale_modifier", C.c_float),
                ("viewmatrix", C.c_float * 16), ("projmatrix", C.c_float * 16), ("sh_degree", C.c_int32),
                ("campos", C.c_float * 3), ("prefiltered", C.c_int32), ("debug", C.c_int32)]


class GeomView(C.Structure):
    _fields_ = [("depths", C.c_void_p), ("means2D", C.c_void_p), ("conic_opacity", C.c_void_p),
                ("tiles_touched", C.c_void_p), ("point_offsets", C.c_void_p)]


class BinningView(C.Structure):
    _fields_ = [("point_list_keys", C.c_void_p), ("point_list", C.c_void_p), ("slabA", C.c_void_p), ("block_lists", C.c_void_p)]


class ImageView(C.Structure):
    _fields_ = [("final_T", C.c_void_p), ("n_contrib", C.c_void_p), ("ranges", C.c_void_p), ("block_counts", C.c_void_p)]


ALLOC_FN = C.CFUNCTYPE(C.c_void_p, C.c_void_p, C.c_size_t)

if not os.path.exists(LIB_PATH):
    raise ImportError(
        f"{LIB_PATH} not found: the CUDA extension is not built. Run `python gps-gaussian_b200/build.py` "
        "(nvcc, sm_90a). There is deliberately no CPU / PyTorch fallback.")

lib = C.CDLL(LIB_PATH)

_vp, _i, _i64, _sz = C.c_void_p, C.c_int, C.c_int64, C.c_size_t
lib.gpsg_last_error.restype = C.c_char_p
lib.gpsg_last_error.argtypes = []
lib.gpsg_version.restype = _i
_pp = C.POINTER(C.c_void_p)
_rs = C.POINTER(RasterSettings)
lib.gpsg_rasterize_forward.restype = _i
lib.gpsg_rasterize_forward.argtypes = [_rs, _i, _vp, _i, _i] + [_vp] * 11 + [
    ALLOC_FN, _vp, ALLOC_FN, _vp, ALLOC_FN, _vp, C.POINTER(C.c_int32), _i]
lib.gpsg_rasterize_forward_maps_begin.restype = _i
lib.gpsg_rasterize_forward_maps_begin.argtypes = [_rs, _i, _vp, _i] + [_pp] * 6 + [
    _vp, ALLOC_FN, _vp, ALLOC_FN, _vp, _vp, _i]
lib.gpsg_rasterize_forward_maps_finish.restype = _i
lib.gpsg_rasterize_forward_maps_finish.argtypes = [_rs, _i, _vp, _i] + [_pp] * 6 + [_vp] * 6 + [
    ALLOC_FN, _vp, _vp, C.POINTER(C.c_int32)]
lib.gpsg_rasterize_forward_planned.restype = _i
lib.gpsg_rasterize_forward_planned.argtypes = [_rs, _i, _vp, _i] + [_vp] * 12 + [_i64, _vp, _vp, _i]
lib.gpsg_rasterize_forward_maps_planned.restype = _i
lib.gpsg_rasterize_forward_maps_planned.argtypes = [_rs, _i, _vp, _i] + [_pp] * 6 + [_vp] * 6 + [_i64, _vp, _vp, _i]
lib.gpsg_rasterize_backward_workspace_bytes.restype = _sz
lib.gpsg_rasterize_backward_workspace_bytes.argtypes = [_i, _i64, _i, _i]
lib.gpsg_rasterize_backward.restype = _i
lib.gpsg_rasterize_backward.argtypes = [_rs, _i, _vp, _i, _i, C.c_int32] + [_vp] * 23 + [_i]
lib.gpsg_rasterize_backward_maps_workspace_bytes.restype = _sz
lib.gpsg_rasterize_backward_maps_workspace_bytes.argtypes = [_i, _i64, _i, _i]
lib.gpsg_rasterize_backward_maps.restype = _i
lib.gpsg_rasterize_backward_maps.argtypes = [_rs, _i, _vp, _i, C.c_int32] + [_pp] * 6 + [_vp] * 7 + [_pp] * 5 + [_vp, _i]
lib.gpsg_mark_visible.restype = _i
lib.gpsg_mark_visible.argtypes = [_i, _vp, _i, _vp, C.POINTER(C.c_float), _vp]
lib.gpsg_geom_view.restype = _i
lib.gpsg_geom_view.argtypes = [_vp, _i, C.POINTER(GeomView)]
lib.gpsg_binning_view.restype = _i
lib.gpsg_binning_view.argtypes = [_vp, _i64, C.POINTER(BinningView)]
lib.gpsg_image_view.restype = _i
lib.gpsg_image_view.argtypes = [_vp, _i, _i, C.POINTER(ImageView)]
lib.gpsg_corr_sampler_forward.restype = _i
lib.gpsg_corr_sampler_forward.argtypes = [_i, _vp, _i, _i, _i, _i, _i, _vp, _i64, _i64, _i64, _vp, _i64, _i, _vp]
lib.gpsg_corr_sampler_backward.restype = _i
lib.gpsg_corr_sampler_backward.argtypes = [_i, _vp, _i, _i, _i, _i, _i, _vp, _i64, _vp, _i, _vp]

lib.gpsg_raster_geom_bytes.restype = _sz
lib.gpsg_raster_geom_bytes.argtypes = [_i]
lib.gpsg_raster_binning_bytes.restype = _sz
lib.gpsg_raster_binning_bytes.argtypes = [_i64]
lib.gpsg_raster_image_bytes.restype = _sz
lib.gpsg_raster_image_bytes.argtypes = [_i, _i]
lib.gpsg_corr_build_pyramid.restype = _i
lib.gpsg_corr_build_pyramid.argtypes = [_i, _vp, _i, _i, _i, _i, _i, _i, _vp, _vp, C.POINTER(C.c_void_p), _i]
lib.gpsg_corr_build_backward.restype = _i
lib.gpsg_corr_build_backward.argtypes = [_i, _vp, _i, _i, _i, _i, _i, _i, _vp, _vp, _vp, _vp, _vp]
lib.gpsg_corr_lookup_pyramid_forward.restype = _i
lib.gpsg_corr_lookup_pyramid_forward.argtypes = [_i, _vp, _i, _i, _i, _i, C.POINTER(C.c_void_p), C.POINTER(C.c_int32), _i,
                                                 _vp, _i64, _i, _vp]
lib.gpsg_corr_lookup_pyramid_backward.restype = _i
lib.gpsg_corr_lookup_pyramid_backward.argtypes = [_i, _vp, _i, _i, _i, _i, C.POINTER(C.c_void_p), C.POINTER(C.c_int32), _i,
                                                  _vp, _i64, _i, _vp]
lib.gpsg_unproject_forward.restype = _i
lib.gpsg_unproject_forward.argtypes = [_i, _vp, _i, _i, _vp, _vp, _i64, _vp, _vp, _i, _vp, _vp, _vp, _vp, _vp]
lib.gpsg_unproject_backward.restype = _i
lib.gpsg_unproject_backward.argtypes = [_i, _vp, _i, _i, _vp, _vp, _i64, _vp, _vp, _i, _vp, _vp, _vp, _vp, _vp]
lib.gpsg_l1_ssim_workspace_bytes.restype = _sz
lib.gpsg_l1_ssim_workspace_bytes.argtypes = [_i, _i, _i]
lib.gpsg_l1_ssim_forward.restype = _i
lib.gpsg_l1_ssim_forward.argtypes = [_i, _vp, _i, _i, _i, _vp, _vp, C.c_float, C.c_float, _vp, _vp, _vp]
lib.gpsg_l1_ssim_backward.restype = _i
lib.gpsg_l1_ssim_backward.argtypes = [_i, _vp, _i, _i, _i, _vp, _vp, _vp, C.c_float, C.c_float, _vp, _vp]
lib.gpsg_point_splat_workspace_bytes.restype = _sz
lib.gpsg_point_splat_workspace_bytes.argtypes = [_i, _i]
lib.gpsg_point_splat.restype = _i
lib.gpsg_point_splat.argtypes = [_i, _vp, _i, _i, _i, _i64, _vp, _vp, _vp, _vp, _vp]


class RectifyCamera(C.Structure):
    """GpsgRectifyCamera (include/gpsg.h): source K, rectifying R and P[:3,:3], fp64 row-major."""
    _fields_ = [("K", C.c_double * 9), ("R", C.c_double * 9), ("P", C.c_double * 9)]


class RectifyPlanes(C.Structure):
    """GpsgRectifyPlanes (include/gpsg.h): one view's device pointers, NULL where absent."""
    _fields_ = [(n, C.c_void_p) for n in ("img", "mask", "depth", "img_out", "mask_out", "depth_out", "img_tensor",
                                          "mask_tensor")]


MESH_MAX_CAMERAS = 8      # GPSG_MESH_MAX_CAMERAS (include/gpsg.h)
MESH_MAX_LIGHTS = 16      # GPSG_MESH_MAX_LIGHTS (include/gpsg.h)


class Mesh(C.Structure):
    """GpsgMesh (include/gpsg.h), passed by value: device pointers of the mesh and its texture, NULL where absent."""
    _fields_ = [("verts", C.c_void_p), ("face_verts", C.c_void_p), ("uvs", C.c_void_p), ("face_uvs", C.c_void_p),
                ("tex", C.c_void_p), ("num_verts", C.c_int32), ("num_faces", C.c_int32), ("num_uvs", C.c_int32),
                ("tex_w", C.c_int32), ("tex_h", C.c_int32)]


class MeshCamera(C.Structure):
    """GpsgMeshCamera (include/gpsg.h): res, intrinsics, position, trans^-1 (row-major) and the device outputs."""
    _fields_ = [("width", C.c_int32), ("height", C.c_int32), ("fx", C.c_float), ("fy", C.c_float), ("cx", C.c_float),
                ("cy", C.c_float), ("pos", C.c_float * 3), ("inv_rot", C.c_float * 9), ("img", C.c_void_p),
                ("zbuf", C.c_void_p), ("mask", C.c_void_p)]


class MeshScene(C.Structure):
    """GpsgMeshScene (include/gpsg.h), passed by value: the cameras of one render and the lights."""
    _fields_ = [("cameras", MeshCamera * MESH_MAX_CAMERAS), ("light_dir", (C.c_float * 3) * MESH_MAX_LIGHTS),
                ("light_color", (C.c_float * 3) * MESH_MAX_LIGHTS), ("num_cameras", C.c_int32),
                ("num_lights", C.c_int32)]


lib.gpsg_mesh_render_workspace_bytes.restype = _sz
lib.gpsg_mesh_render_workspace_bytes.argtypes = [_i, _i64]
lib.gpsg_mesh_render.restype = _i
lib.gpsg_mesh_render.argtypes = [_i, _vp, Mesh, MeshScene, _vp, _sz]
lib.gpsg_rectify_remap.restype = _i
lib.gpsg_rectify_remap.argtypes = [_i, _vp, C.POINTER(RectifyCamera), _i, _i, _i, _i, _i, _i, C.POINTER(RectifyPlanes)]
lib.gpsg_rectify_flow.restype = _i
lib.gpsg_rectify_flow.argtypes = [_i, _vp, _i, _i, _i, C.c_double, C.c_double, C.c_double, _pp, _pp, _pp, _pp]
class SeqLossArgs(C.Structure):
    """GpsgSeqLossArgs (include/gpsg.h), passed by value: prediction / gradient pointers and fp32 weights."""
    _fields_ = [("pred", C.c_void_p * 32), ("grad", C.c_void_p * 32), ("weight", C.c_float * 32), ("gt", C.c_void_p),
                ("valid", C.c_void_p), ("numel", C.c_int64), ("n_pred", C.c_int), ("gt_dtype", C.c_int)]


SEQ_LOSS_MAX_PRED = 32    # GPSG_SEQ_LOSS_MAX_PRED (include/gpsg.h)
# GpsgGsHeadWeights field order (include/gpsg.h)
GS_HEAD_PARAMS = ("out_w", "out_b", "rot_w1", "rot_b1", "rot_w2", "rot_b2", "scale_w1", "scale_b1", "scale_w2",
                  "scale_b2", "opacity_w1", "opacity_b1", "opacity_w2", "opacity_b2")
lib.gpsg_convex_upsample_forward.restype = _i
lib.gpsg_convex_upsample_forward.argtypes = [_i, _vp, _i, _i, _i, _i, _i, _i, _vp, _vp, _vp]
lib.gpsg_convex_upsample_backward_workspace_bytes.restype = _sz
lib.gpsg_convex_upsample_backward_workspace_bytes.argtypes = [_i, _i, _i, _i]
lib.gpsg_convex_upsample_backward.restype = _i
lib.gpsg_convex_upsample_backward.argtypes = [_i, _vp, _i, _i, _i, _i, _i, _i, _vp, _vp, _vp, _vp, _vp, _vp]
lib.gpsg_sequence_loss_workspace_bytes.restype = _sz
lib.gpsg_sequence_loss_workspace_bytes.argtypes = []
lib.gpsg_sequence_loss_forward.restype = _i
lib.gpsg_sequence_loss_forward.argtypes = [_i, _vp, SeqLossArgs, _vp, _vp]
lib.gpsg_sequence_loss_backward.restype = _i
lib.gpsg_sequence_loss_backward.argtypes = [_i, _vp, SeqLossArgs, _vp, _vp]


class GsHeadWeights(C.Structure):
    """GpsgGsHeadWeights (include/gpsg.h), passed by value: the 14 device pointers of the regressor tail's weights."""
    _fields_ = [(n, C.c_void_p) for n in GS_HEAD_PARAMS]


lib.gpsg_gs_head_workspace_bytes.restype = _sz
lib.gpsg_gs_head_workspace_bytes.argtypes = [_i, _i, _i]
lib.gpsg_gs_head_forward.restype = _i
lib.gpsg_gs_head_forward.argtypes = [_i, _vp, _i, _i, _i] + [_vp] * 6 + [GsHeadWeights, _vp]


class GsHeadGrads(C.Structure):
    """GpsgGsHeadGrads (include/gpsg.h), passed by value: the 14 device pointers of the tail's weight gradients."""
    _fields_ = [(n, C.c_void_p) for n in GS_HEAD_PARAMS]


lib.gpsg_gs_head_backward_workspace_bytes.restype = _sz
lib.gpsg_gs_head_backward_workspace_bytes.argtypes = [_i, _i, _i]
lib.gpsg_gs_head_backward.restype = _i
lib.gpsg_gs_head_backward.argtypes = [_i, _vp, _i, _i, _i] + [_vp] * 9 + [GsHeadWeights, GsHeadGrads, _vp]
# GpsgEncoderStemWeights field order (include/gpsg.h)
ENCODER_STEM_PARAMS = ("in_conv_w", "in_conv_b", "in_norm_w", "in_norm_b") + tuple(
    f"b{k}_{n}" for k in (1, 2) for n in ("conv1_w", "conv1_b", "norm1_w", "norm1_b", "conv2_w", "conv2_b", "norm2_w",
                                          "norm2_b"))
ENCODER_STEM_TF32, ENCODER_STEM_FP16 = 0, 1     # GPSG_ENCODER_STEM_TF32 / _FP16 (include/gpsg.h)


class EncoderStemWeights(C.Structure):
    """GpsgEncoderStemWeights (include/gpsg.h), passed by value: the 20 device pointers of the stem's parameters."""
    _fields_ = [(n, C.c_void_p) for n in ENCODER_STEM_PARAMS]


lib.gpsg_encoder_stem_workspace_bytes.restype = _sz
lib.gpsg_encoder_stem_workspace_bytes.argtypes = [_i, _i, _i, _i, _i]
lib.gpsg_encoder_stem_forward.restype = _i
lib.gpsg_encoder_stem_forward.argtypes = [_i, _vp, _i, _i, _i, _i, _i, _vp, EncoderStemWeights, _vp, _vp]
# GpsgDecoder1Weights field order (include/gpsg.h)
DECODER1_PARAMS = tuple(f"b0_{n}" for n in ("conv1_w", "conv1_b", "norm1_w", "norm1_b", "conv2_w", "conv2_b", "norm2_w",
                                            "norm2_b", "down_w", "down_b", "norm3_w", "norm3_b")) + tuple(
    f"b1_{n}" for n in ("conv1_w", "conv1_b", "norm1_w", "norm1_b", "conv2_w", "conv2_b", "norm2_w", "norm2_b"))


class Decoder1Weights(C.Structure):
    """GpsgDecoder1Weights (include/gpsg.h), passed by value: the 20 device pointers of decoder1's parameters."""
    _fields_ = [(n, C.c_void_p) for n in DECODER1_PARAMS]


lib.gpsg_decoder1_workspace_bytes.restype = _sz
lib.gpsg_decoder1_workspace_bytes.argtypes = [_i, _i, _i]
lib.gpsg_decoder1_forward.restype = _i
lib.gpsg_decoder1_forward.argtypes = [_i, _vp, _i, _i, _i, _vp, _vp, _vp, Decoder1Weights, _vp, _vp]


class Decoder23Weights(C.Structure):
    """GpsgDecoder23Weights (include/gpsg.h), passed by value: the 20 device pointers of decoder3's or decoder2's
    parameters, in GpsgDecoder1Weights' field order (`DECODER1_PARAMS`)."""
    _fields_ = [(n, C.c_void_p) for n in DECODER1_PARAMS]


lib.gpsg_decoder3_workspace_bytes.restype = _sz
lib.gpsg_decoder3_workspace_bytes.argtypes = [_i, _i, _i]
lib.gpsg_decoder3_forward.restype = _i
lib.gpsg_decoder3_forward.argtypes = [_i, _vp, _i, _i, _i, _vp, _vp, Decoder23Weights, _vp, _vp]
lib.gpsg_decoder2_workspace_bytes.restype = _sz
lib.gpsg_decoder2_workspace_bytes.argtypes = [_i, _i, _i]
lib.gpsg_decoder2_forward.restype = _i
lib.gpsg_decoder2_forward.argtypes = [_i, _vp, _i, _i, _i, _vp, _vp, _vp, Decoder23Weights, _vp, _vp]


class EncoderDownWeights(C.Structure):
    """GpsgEncoderDownWeights (include/gpsg.h), passed by value: the 20 device pointers of one down stage (res2 or res3),
    in GpsgDecoder1Weights' field order (`DECODER1_PARAMS`)."""
    _fields_ = [(n, C.c_void_p) for n in DECODER1_PARAMS]


lib.gpsg_encoder_down_workspace_bytes.restype = _sz
lib.gpsg_encoder_down_workspace_bytes.argtypes = [_i, _i, _i, _i, _i, _i]
lib.gpsg_encoder_down_forward.restype = _i
lib.gpsg_encoder_down_forward.argtypes = [_i, _vp, _i, _i, _i, _i, _i, _i, _vp, EncoderDownWeights, _vp, _vp]
UPDATE_PARAMS = ("convc1_w", "convc1_b", "convc2_w", "convc2_b", "convf1_w", "convf1_b", "convf2_w", "convf2_b",
                 "conv_w", "conv_b", "convz_w", "convz_b", "convr_w", "convr_b", "convq_w", "convq_b",
                 "fh_conv1_w", "fh_conv1_b", "fh_conv2_w", "fh_conv2_b", "mask0_w", "mask0_b", "mask2_w", "mask2_b")


class UpdateWeights(C.Structure):
    """GpsgUpdateWeights (include/gpsg.h), passed by value: the 24 device pointers of the update block's parameters."""
    _fields_ = [(n, C.c_void_p) for n in UPDATE_PARAMS]


lib.gpsg_update_workspace_bytes.restype = _sz
lib.gpsg_update_workspace_bytes.argtypes = [_i, _i, _i]
lib.gpsg_update_packed_bytes.restype = _sz
lib.gpsg_update_packed_bytes.argtypes = []
lib.gpsg_update_pack.restype = _i
lib.gpsg_update_pack.argtypes = [_i, _vp, UpdateWeights, _vp]
lib.gpsg_update_step.restype = _i
lib.gpsg_update_step.argtypes = [_i, _vp, _i, _i, _i, _i, _vp, _vp, _vp, _vp, _i64, _vp, _vp, _vp]
lib.gpsg_profile_enable.restype = _i
lib.gpsg_profile_enable.argtypes = [_i]
lib.gpsg_profile_read.restype = _i
lib.gpsg_profile_read.argtypes = [C.POINTER(C.c_float), C.POINTER(C.c_int32), C.POINTER(C.c_int32), _i]
lib.gpsg_profile_stage_name.restype = C.c_char_p
lib.gpsg_profile_stage_name.argtypes = [_i]

EXPORTED = ["gpsg_last_error", "gpsg_version", "gpsg_rasterize_forward", "gpsg_rasterize_forward_maps_begin",
            "gpsg_rasterize_forward_maps_finish", "gpsg_raster_geom_bytes", "gpsg_raster_binning_bytes",
            "gpsg_raster_image_bytes", "gpsg_rasterize_forward_planned", "gpsg_rasterize_forward_maps_planned",
            "gpsg_rasterize_backward_workspace_bytes", "gpsg_rasterize_backward",
            "gpsg_rasterize_backward_maps_workspace_bytes", "gpsg_rasterize_backward_maps", "gpsg_mark_visible",
            "gpsg_geom_view", "gpsg_binning_view", "gpsg_image_view", "gpsg_corr_sampler_forward",
            "gpsg_corr_sampler_backward", "gpsg_corr_build_pyramid", "gpsg_corr_build_backward",
            "gpsg_corr_lookup_pyramid_forward", "gpsg_corr_lookup_pyramid_backward", "gpsg_unproject_forward",
            "gpsg_unproject_backward", "gpsg_l1_ssim_workspace_bytes", "gpsg_l1_ssim_forward", "gpsg_l1_ssim_backward",
            "gpsg_set_corr_build", "gpsg_profile_enable", "gpsg_profile_read", "gpsg_profile_stage_name",
            "gpsg_point_splat_workspace_bytes", "gpsg_point_splat", "gpsg_rectify_remap", "gpsg_rectify_flow",
            "gpsg_convex_upsample_forward", "gpsg_convex_upsample_backward_workspace_bytes",
            "gpsg_convex_upsample_backward", "gpsg_sequence_loss_workspace_bytes", "gpsg_sequence_loss_forward",
            "gpsg_sequence_loss_backward", "gpsg_mesh_render_workspace_bytes", "gpsg_mesh_render", "gpsg_jpeg_parse",
            "gpsg_jpeg_decode_workspace_bytes", "gpsg_jpeg_decode", "gpsg_jpeg_encode_max_bytes",
            "gpsg_jpeg_encode_workspace_bytes", "gpsg_jpeg_encode", "gpsg_gs_head_workspace_bytes",
            "gpsg_gs_head_forward", "gpsg_gs_head_backward_workspace_bytes", "gpsg_gs_head_backward",
            "gpsg_encoder_stem_workspace_bytes", "gpsg_encoder_stem_forward", "gpsg_decoder1_workspace_bytes",
            "gpsg_decoder1_forward", "gpsg_decoder3_workspace_bytes", "gpsg_decoder3_forward",
            "gpsg_decoder2_workspace_bytes", "gpsg_decoder2_forward", "gpsg_encoder_down_workspace_bytes", "gpsg_encoder_down_forward",
            "gpsg_update_workspace_bytes", "gpsg_update_packed_bytes", "gpsg_update_pack", "gpsg_update_step"]

BWD_DETERMINISTIC = 1     # GPSG_BWD_DETERMINISTIC (include/gpsg.h)
FWD_ANTIALIAS = 1         # GPSG_FWD_ANTIALIAS (include/gpsg.h)


def forward_flags(antialiasing=False):
    """The `flags` word of the gpsg_rasterize_forward* entry points: GPSG_FWD_ANTIALIAS when `antialiasing`, else 0."""
    return FWD_ANTIALIAS if antialiasing else 0


def check(rc, what):
    if rc != 0:
        msg = lib.gpsg_last_error()
        raise GpsgError(f"{what} failed (code {rc}): {msg.decode() if msg else ''}")


# ---- torch-backed scratch allocator for the gpsg_alloc_fn callbacks ---------------------------
_tls = threading.local()


def _alloc_trampoline(user, nbytes):
    try:
        t = torch.empty(int(nbytes), dtype=torch.uint8, device=_tls.device)
        _tls.bufs[int(user or 0)] = t
        return t.data_ptr()
    except Exception:  # never let an exception cross the C boundary
        return None


ALLOC_CB = ALLOC_FN(_alloc_trampoline)


def begin_alloc(device):
    _tls.device = device
    _tls.bufs = {}


def end_alloc():
    bufs = _tls.bufs
    _tls.bufs = {}
    return bufs


def device_stream(device):
    """(device index, current stream handle) of a CUDA device: the first two arguments of every gpsg_* call."""
    device = torch.device(device)
    idx = device.index if device.index is not None else torch.cuda.current_device()
    return idx, C.c_void_p(torch.cuda.current_stream(idx).cuda_stream)


def _ptr(t):
    return C.c_void_p(t.data_ptr()) if (t is not None and t.numel() > 0) else None


def rasterize_forward(settings, out_color, radii, means3D, opacities, colors_precomp=None, shs=None, scales=None,
                      rotations=None, cov3D_precomp=None, out_depth=None, out_alpha=None, antialiasing=False):
    """One forward through the exact entry point gpsg_rasterize_forward: one host synchronisation, and the global radix
    fallback takes tile lists of any length.  Inputs are contiguous fp32 tensors on one CUDA device, absent ones None.
    Writes out_color [3,H,W] and radii [P]; returns (num_rendered, (geom, binning, image)), the buffers the backward
    reads.  out_depth / out_alpha ([H,W] fp32, both or neither): aux mode, which also writes the expected depth and the
    accumulated opacity.  antialiasing: the opacity-compensated screen-space filter (GPSG_FWD_ANTIALIAS); the backward of
    these buffers follows it without being told."""
    if (out_depth is None) != (out_alpha is None):
        raise ValueError("out_depth and out_alpha must be given together")
    dev = means3D.device
    idx, stream = device_stream(dev)
    n = C.c_int32(0)
    fn = lib.gpsg_rasterize_forward
    begin_alloc(dev)
    try:
        with torch.cuda.device(dev):
            rc = fn(
                C.byref(settings), idx, stream, int(means3D.shape[0]), int(shs.shape[1]) if shs is not None else 0,
                _ptr(means3D), _ptr(colors_precomp), _ptr(shs), _ptr(opacities), _ptr(scales), _ptr(rotations),
                _ptr(cov3D_precomp), _ptr(out_color), _ptr(out_depth), _ptr(out_alpha), _ptr(radii), ALLOC_CB, C.c_void_p(1),
                ALLOC_CB, C.c_void_p(2), ALLOC_CB, C.c_void_p(3), C.byref(n), forward_flags(antialiasing))
    finally:
        bufs = end_alloc()
    check(rc, fn.__name__)
    return int(n.value), (bufs.get(1), bufs.get(2), bufs.get(3))


def backward_flags(deterministic=None):
    """The `flags` word of the gpsg_rasterize_backward* entry points.  deterministic=None follows PyTorch's switch,
    torch.use_deterministic_algorithms(True), read when the backward runs (as PyTorch's own kernels read it); True / False
    force the mode.  Deterministic mode gives bit-identical gradients on reruns (include/gpsg.h)."""
    if deterministic is None:
        deterministic = torch.are_deterministic_algorithms_enabled()
    return BWD_DETERMINISTIC if deterministic else 0


def rasterize_backward(settings, num_rendered, bufs, radii, grad_color, means3D, opacities, colors_precomp=None,
                       shs=None, scales=None, rotations=None, cov3D_precomp=None, want_cov3D=False, deterministic=None,
                       grad_depth=None, grad_alpha=None):
    """Backward of `rasterize_forward` with the same inputs, its num_rendered, buffers and radii.  Returns the gradients
    dL_dmeans2D [P,3], dL_dcolors [P,3], dL_dopacity [P,1], dL_dmeans3D [P,3], dL_dscales [P,3], dL_drots [P,4],
    dL_dcov3D [P,6] and dL_dsh [P,M,3].  dL_dcolors is None on the SH path, dL_dsh is None without shs and dL_dcov3D
    is None unless want_cov3D.  `deterministic`: see `backward_flags`.  grad_depth / grad_alpha ([H,W], both or
    neither): the aux gradients; the buffers must then come from an aux forward."""
    if (grad_depth is None) != (grad_alpha is None):
        raise ValueError("grad_depth and grad_alpha must be given together")
    aux = grad_depth is not None
    flags = backward_flags(deterministic)
    dev = means3D.device
    P = int(means3D.shape[0])
    new = lambda *s: torch.empty(s, dtype=torch.float32, device=dev)
    out = dict(dL_dmeans2D=new(P, 3), dL_dcolors=new(P, 3) if colors_precomp is not None else None,
               dL_dopacity=new(P, 1), dL_dmeans3D=new(P, 3), dL_dscales=new(P, 3), dL_drots=new(P, 4),
               dL_dcov3D=new(P, 6) if want_cov3D else None,
               dL_dsh=new(P, int(shs.shape[1]), 3) if shs is not None else None)
    ws = torch.empty(int(lib.gpsg_rasterize_backward_workspace_bytes(P, num_rendered, flags, int(aux))), dtype=torch.uint8,
                     device=dev)
    f32 = lambda t: t.detach().to(torch.float32).contiguous()
    g = f32(grad_color)
    gaux = [f32(grad_depth), f32(grad_alpha)] if aux else [None, None]
    fn = lib.gpsg_rasterize_backward
    idx, stream = device_stream(dev)
    geom, binning, image = bufs
    with torch.cuda.device(dev):
        rc = fn(
            C.byref(settings), idx, stream, P, int(shs.shape[1]) if shs is not None else 0, num_rendered, _ptr(means3D),
            _ptr(colors_precomp), _ptr(shs), _ptr(opacities), _ptr(scales), _ptr(rotations), _ptr(cov3D_precomp),
            _ptr(radii), _ptr(geom), _ptr(binning), _ptr(image), _ptr(g), *[_ptr(t) for t in gaux], _ptr(out["dL_dmeans2D"]),
            _ptr(out["dL_dcolors"]), _ptr(out["dL_dopacity"]), _ptr(out["dL_dmeans3D"]), _ptr(out["dL_dcov3D"]),
            _ptr(out["dL_dsh"]), _ptr(out["dL_dscales"]), _ptr(out["dL_drots"]), _ptr(ws), flags)
    check(rc, fn.__name__)
    return out


lib.gpsg_set_corr_build.restype = _i
lib.gpsg_set_corr_build.argtypes = [_i]


def set_corr_build(kind="wgmma"):
    """'wgmma' (default: tensor-core kernels for fp16 volumes when the shape fits) or 'ffma'."""
    check(lib.gpsg_set_corr_build(1 if kind == "ffma" else 0), "gpsg_set_corr_build")


def profile_enable(on=True):
    """True / 1: CUDA events around every stage + launch counts; 2: launch counts only; False: off."""
    check(lib.gpsg_profile_enable(2 if on == 2 else (1 if on else 0)), "gpsg_profile_enable")


def profile_read():
    """{stage: dict(ms=total, calls=n, launches=k)} since the last read (synchronises)."""
    cap = 32
    ms, calls, launches = (C.c_float * cap)(), (C.c_int32 * cap)(), (C.c_int32 * cap)()
    n = lib.gpsg_profile_read(ms, calls, launches, cap)
    if n < 0:
        check(n, "gpsg_profile_read")
    return {lib.gpsg_profile_stage_name(i).decode(): dict(ms=float(ms[i]), calls=int(calls[i]), launches=int(launches[i]))
            for i in range(n)}
