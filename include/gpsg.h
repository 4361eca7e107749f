/*
 * gpsg.h -- C ABI of libgpsg_sm90.so: the H100 (sm_90a) splat rasterizer and 1-D stereo
 * correlation sampler behind GPS-Gaussian's hot path.
 *
 * The reference has no native code of its own; its FFI for this path is the pybind surface of
 * two third-party extensions it imports by name:
 *   - `diff_gaussian_rasterization._C`  (reference gaussian_renderer/__init__.py:14; called through
 *      GaussianRasterizer at :51-62)          -> rasterize_gaussians / rasterize_gaussians_backward /
 *                                                mark_visible
 *   - `corr_sampler`                    (reference core/corr.py:5-8; called at :22 and :28)
 *                                             -> forward / backward
 * Each entry point below replaces exactly one of those bound functions; plain pointers and sizes,
 * no torch/ATen types, no exceptions.  All pointers are DEVICE pointers unless marked host.
 * Every function returns 0 on success or a negative GPSG_E_* code; gpsg_last_error() gives the
 * message (thread-local).  All work is enqueued on `stream` (a cudaStream_t) of CUDA device `device`.
 */
#ifndef GPSG_H
#define GPSG_H
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#if defined(__GNUC__)
#define GPSG_API __attribute__((visibility("default")))
#else
#define GPSG_API
#endif

#define GPSG_OK 0
#define GPSG_E_INVALID (-1)   /* bad argument (shape / null / unsupported combination) */
#define GPSG_E_CUDA (-2)      /* a CUDA runtime call or kernel launch failed */
#define GPSG_E_ALLOC (-3)     /* an allocator callback returned NULL */
#define GPSG_E_CAPACITY (-4)  /* caller-provided workspace too small */

/* Mirrors diff_gaussian_rasterization.GaussianRasterizationSettings -- the 12 fields the reference
 * fills at gaussian_renderer/__init__.py:36-49.  Matrices are the 16 floats of the tensors the
 * reference passes (world_view_transform = W2V^T, full_proj_transform), i.e. the maths matrix is
 * M(r,c) = m[c*4+r].  Passed BY VALUE into kernels, so the tensors may live on host or device
 * (in training they stay in pinned host memory: reference train_stage2.py:155-157). */
typedef struct GpsgRasterSettings {
    int32_t image_height;
    int32_t image_width;
    float tanfovx;
    float tanfovy;
    float bg[3];
    float scale_modifier;
    float viewmatrix[16];
    float projmatrix[16];
    int32_t sh_degree;
    float campos[3];
    int32_t prefiltered;
    int32_t debug;
} GpsgRasterSettings;

/* Scratch allocator, the C form of upstream's `std::function<char*(size_t)>` resize callbacks over
 * torch byte tensors: must return a device pointer to >= `bytes` bytes (256-B aligned), valid until
 * the matching backward call has finished.  Called at most once per buffer per forward. */
typedef void* (*gpsg_alloc_fn)(void* user, size_t bytes);

GPSG_API const char* gpsg_last_error(void);
GPSG_API int gpsg_version(void);

/* ==== splat rasterizer: replaces _C.rasterize_gaussians / _C.rasterize_gaussians_backward (SURVEY.md Appendix A) ====
 * Conventions shared by the entry points below.
 *
 * Gaussians come in one of two forms.
 *   AoS: means3D[P,3] opacities[P]; exactly one of colors_precomp[P,3] / shs[P,sh_M,3]; either (scales[P,3],
 *     rotations[P,4]) or cov3D_precomp[P,6].
 *   maps (the fused map -> Gaussian ingest behind pts2render, reference lib/GaussianRender.py:5-39): the two source
 *     views' pixel-aligned maps are read in place instead of boolean-mask gathered (10 `nonzero` host syncs per sample)
 *     and concatenated.  Per view v in {0,1} (lmain, rmain), with S2 = pixels_per_view: valid[v][S2] (uint8/bool),
 *     xyz[v][S2,3], img[v][3,S2] in [-1,1] (colour = img*0.5+0.5), rot[v][4,S2], scale[v][3,S2], opacity[v][1,S2].
 *     Gaussian index = v*S2 + pixel, so P = 2*S2; invalid pixels are culled.  Pointer arguments of this form are HOST
 *     arrays of two device pointers.  Results (image, and gradients in map layout) equal the gather + render path.
 *
 * Outputs: out_color[3,H,W] and radii[P].  out_depth[H,W] and out_alpha[H,W] (fp32) are the aux outputs, both NULL or
 *   both set:
 *     alpha = 1 - T_final (accumulated opacity; exactly 1 - the transmittance the backward reads),
 *     depth = sum_i w_i z_i, w_i = alpha_i T_i the compositing weight and z_i the view-space depth of Gaussian i (the key
 *             the tile lists are sorted by).  Not normalised by alpha and without background (depth = 0 where nothing is
 *             drawn): depth is a fourth colour channel whose colour is z and whose background is 0.
 *   The colour image, radii and the saved buffers are bit-identical with and without the aux outputs, and the buffers
 *   have the same sizes (z is read from the geometry buffer).
 *
 * Forward flags (`flags` of gpsg_rasterize_forward, _maps_begin, _planned and _maps_planned):
 *   0: the upstream forward.
 *   GPSG_FWD_ANTIALIAS: opacity-compensated screen-space filter (upstream's `antialiasing` setting, the 2-D filter of
 *     Mip-Splatting).  The 0.3 px^2 dilation of the screen covariance stays, so the conics, radii, tile lists and sort
 *     keys are bit-identical to flags = 0; each splat's opacity is scaled by rho = sqrt(max(2.5e-5, det(Sigma2D) /
 *     det(Sigma2D + 0.3 I))), so its integrated alpha no longer grows with the dilation (sub-pixel splats no longer turn
 *     into >= 0.55 px blobs at full opacity).  The scaled opacity o * rho is what conic_opacity[P,4].w (gpsg_geom_view)
 *     holds and what the compositing uses.
 *   The forward records its flags in its image buffer, on the device and in stream order (no host synchronisation, so
 *   the planned forwards stay graph-capturable).  The backward reads them from the image buffer it is given, so it always
 *   differentiates the mode of the forward whose buffers it receives.  A reused planned image buffer carries the mode of
 *   its last forward.
 *   Unknown flag bits return GPSG_E_INVALID before any other argument is checked.
 *
 * Saved buffers: every forward leaves a geometry, a binning and an image buffer; the backward reads the three of the
 * forward it differentiates. */
#define GPSG_FWD_ANTIALIAS 1

/* ---- exact forward: replaces _C.rasterize_gaussians --------------------------------------------------------------
 * AoS Gaussians.  Scratch comes from the three callbacks (geometry / binning / image buffer, kept for the backward).
 * *num_rendered (HOST) receives the number of (tile, Gaussian) pairs.  One host synchronisation, as upstream, and tile
 * lists of any length (a global radix sort takes those too long for the in-CTA sort). */
GPSG_API int gpsg_rasterize_forward(const GpsgRasterSettings* settings, int device, void* stream, int P, int sh_M,
                                    const float* means3D, const float* colors_precomp, const float* shs,
                                    const float* opacities, const float* scales, const float* rotations,
                                    const float* cov3D_precomp, float* out_color, float* out_depth, float* out_alpha,
                                    int32_t* radii, gpsg_alloc_fn geom_alloc, void* geom_user,
                                    gpsg_alloc_fn binning_alloc, void* binning_user, gpsg_alloc_fn image_alloc,
                                    void* image_user, int32_t* num_rendered, int flags);

/* ---- exact forward of the maps, in two halves ---------------------------------------------------------------------
 * A BATCH of samples needs ONE host synchronisation (reference lib/GaussianRender.py:8 loops over the samples; upstream
 * synchronises once per sample to read num_rendered):
 *   _begin : projection (under `flags`), pairs-per-tile counts, tile ranges; allocates the geometry and image buffers
 *            through the callbacks (the caller keeps the pointers they returned) and enqueues a copy of 6 status words
 *            into `totals_host` (pinned host memory).  Does NOT synchronise.
 *   ... the caller synchronises `stream` once after the _begin calls of all samples ...
 *   _finish: sizes and allocates the binning buffer from totals_host, bins, sorts, composites into out_color (and the
 *            aux outputs when set); *num_rendered (HOST) receives the pair count.  The forward's mode is the one _begin
 *            recorded, so _finish takes no flags.
 * A batch of one is begin, one synchronisation, finish.  The saved buffers feed gpsg_rasterize_backward_maps. */
GPSG_API int gpsg_rasterize_forward_maps_begin(const GpsgRasterSettings* settings, int device, void* stream,
                                               int pixels_per_view, const uint8_t* const* valid, const float* const* xyz,
                                               const float* const* img, const float* const* rot,
                                               const float* const* scale, const float* const* opacity, int32_t* radii,
                                               gpsg_alloc_fn geom_alloc, void* geom_user, gpsg_alloc_fn image_alloc,
                                               void* image_user, uint32_t* totals_host /* >= 6 words, pinned */,
                                               int flags);
GPSG_API int gpsg_rasterize_forward_maps_finish(const GpsgRasterSettings* settings, int device, void* stream,
                                                int pixels_per_view, const uint8_t* const* valid,
                                                const float* const* xyz, const float* const* img,
                                                const float* const* rot, const float* const* scale,
                                                const float* const* opacity, float* out_color, float* out_depth,
                                                float* out_alpha, int32_t* radii, void* geom_buffer, void* image_buffer,
                                                gpsg_alloc_fn binning_alloc, void* binning_user,
                                                const uint32_t* totals_host, int32_t* num_rendered);

/* ---- sync-free ("planned") forwards: the serving loop (reference test_view_interp.py:39-47) ------------------------
 * The same computation as the exact forward, but every buffer is provided by the caller up front and there is NO host
 * synchronisation, so the call is CUDA-graph capturable and the CPU can run ahead.  Buffer sizes: gpsg_raster_geom_bytes
 * (P; P = 2*pixels_per_view for the maps), gpsg_raster_image_bytes(W, H) and gpsg_raster_binning_bytes(capacity_pairs),
 * where capacity_pairs bounds the number of (tile, Gaussian) pairs the binning buffer can hold.
 * Overflow: the kernels read the actual pair count from device memory; if it exceeds the capacity (or a tile list exceeds
 * the in-CTA sort limit) they set the overflow word and skip their work.  The caller must inspect the status words once
 * it next synchronises and, if the overflow word is set, retry with a larger capacity or the exact forward (out_color
 * and the aux outputs are then undefined).  Status words, [0] pairs N, [1] longest tile list, [2] overflow flag: kept in
 * the image buffer and copied to `status_host` (pinned host memory, >= 3 words) when it is not NULL.
 * gpsg_rasterize_forward_planned takes AoS Gaussians with colors_precomp (no SH); gpsg_rasterize_forward_maps_planned
 * renders many novel cameras from one pair's cached maps without gathering them.  For the backward of a planned forward
 * pass num_rendered = capacity_pairs. */
GPSG_API size_t gpsg_raster_geom_bytes(int P);
GPSG_API size_t gpsg_raster_binning_bytes(int64_t capacity_pairs);
GPSG_API size_t gpsg_raster_image_bytes(int W, int H);
GPSG_API int gpsg_rasterize_forward_planned(const GpsgRasterSettings* settings, int device, void* stream, int P,
                                            const float* means3D, const float* colors_precomp, const float* opacities,
                                            const float* scales, const float* rotations, const float* cov3D_precomp,
                                            float* out_color, float* out_depth, float* out_alpha, int32_t* radii,
                                            void* geom_buffer, void* binning_buffer, int64_t capacity_pairs,
                                            void* image_buffer, uint32_t* status_host, int flags);
GPSG_API int gpsg_rasterize_forward_maps_planned(const GpsgRasterSettings* settings, int device, void* stream,
                                                 int pixels_per_view, const uint8_t* const* valid,
                                                 const float* const* xyz, const float* const* img,
                                                 const float* const* rot, const float* const* scale,
                                                 const float* const* opacity, float* out_color, float* out_depth,
                                                 float* out_alpha, int32_t* radii, void* geom_buffer,
                                                 void* binning_buffer, int64_t capacity_pairs, void* image_buffer,
                                                 uint32_t* status_host, int flags);

/* ---- backward: replaces _C.rasterize_gaussians_backward -------------------------------------------------------------
 * gpsg_rasterize_backward differentiates gpsg_rasterize_forward or a planned AoS forward; gpsg_rasterize_backward_maps
 * differentiates the maps forwards and writes the gradients in map layout.  The geom / binning / image buffers, radii and
 * num_rendered are the forward's.  All dL_* outputs are written (zero for culled Gaussians).  AoS: dL_dmeans2D is [P,3]
 * (z unused); dL_dsh [P,sh_M,3] is given exactly when shs is; dL_dcolors may be NULL on the SH path and dL_dcov3D [P,6]
 * when not needed.
 * Aux gradients: dL_dout_depth[H,W] and dL_dout_alpha[H,W], both NULL or both set (either may hold zeros).  When set, the
 *   buffers (and num_rendered) must come from a forward of the same inputs that wrote the depth and alpha outputs those
 *   gradients belong to.  The depth gradient reaches dL_dmeans3D (maps: dL_dxyz) through the view matrix's third row; the
 *   alpha gradient reaches the opacities and the geometry through the compositing weights.
 * flags:
 *   0: per-Gaussian sums with atomics, as upstream.
 *   GPSG_BWD_DETERMINISTIC: bit-identical gradients for identical inputs on the same device and build, whatever the CTA
 *     schedule, concurrent work on other streams or the binning path (tile bucket or GPSG_BINNING=radix).  The
 *     compositing backward stores its per-(pair, warp) partial sums instead of adding them with atomics, and one thread
 *     per Gaussian adds them in a fixed order.  The gradients differ from flags = 0 only by fp32 re-association.  It
 *     reads the sorted keys and point list, so it needs the buffers of an EXACT forward (gpsg_rasterize_forward or maps
 *     _begin / _finish); the planned forwards do not write them and are not supported.
 *   Unknown flag bits return GPSG_E_INVALID before any other argument is checked.
 * No host synchronisation and no allocation in either mode: graph-capturable.
 * `workspace` must hold gpsg_rasterize_backward_workspace_bytes(P, num_rendered, flags, aux) bytes (maps:
 * gpsg_rasterize_backward_maps_workspace_bytes(pixels_per_view, ...)), aux = 1 when the aux gradients are set, else 0.
 * Without GPSG_BWD_DETERMINISTIC the size depends on neither num_rendered nor aux.  With it the partial sums add per pair
 * a 1-byte slot mask and 8 slots of 9 floats (aux = 0: 289 B) or 10 floats (aux = 1: 321 B), plus alignment.  The size
 * queries return 0 (message in gpsg_last_error) for unknown flag bits, an aux other than 0 or 1, or, with
 * GPSG_BWD_DETERMINISTIC, a num_rendered outside [0, 2^31). */
#define GPSG_BWD_DETERMINISTIC 1
GPSG_API size_t gpsg_rasterize_backward_workspace_bytes(int P, int64_t num_rendered, int flags, int aux);
GPSG_API int gpsg_rasterize_backward(const GpsgRasterSettings* settings, int device, void* stream, int P, int sh_M,
                                     int32_t num_rendered, const float* means3D, const float* colors_precomp,
                                     const float* shs, const float* opacities, const float* scales,
                                     const float* rotations, const float* cov3D_precomp, const int32_t* radii,
                                     const void* geom_buffer, const void* binning_buffer, const void* image_buffer,
                                     const float* dL_dout_color, const float* dL_dout_depth,
                                     const float* dL_dout_alpha, float* dL_dmeans2D, float* dL_dcolors,
                                     float* dL_dopacity, float* dL_dmeans3D, float* dL_dcov3D, float* dL_dsh,
                                     float* dL_dscales, float* dL_drotations, void* workspace, int flags);
GPSG_API size_t gpsg_rasterize_backward_maps_workspace_bytes(int pixels_per_view, int64_t num_rendered, int flags,
                                                             int aux);
GPSG_API int gpsg_rasterize_backward_maps(const GpsgRasterSettings* settings, int device, void* stream,
                                          int pixels_per_view, int32_t num_rendered, const uint8_t* const* valid,
                                          const float* const* xyz, const float* const* img, const float* const* rot,
                                          const float* const* scale, const float* const* opacity,
                                          const int32_t* radii, const void* geom_buffer, const void* binning_buffer,
                                          const void* image_buffer, const float* dL_dout_color,
                                          const float* dL_dout_depth, const float* dL_dout_alpha,
                                          float* const* dL_dxyz, float* const* dL_dimg, float* const* dL_drot,
                                          float* const* dL_dscale, float* const* dL_dopacity, void* workspace,
                                          int flags);

/* ---- replaces _C.mark_visible : present[P] (uint8) = view-space z > 0.2 ---------------------- */
GPSG_API int gpsg_mark_visible(int device, void* stream, int P, const float* means3D, const float* viewmatrix_host16,
                      uint8_t* present);

/* Introspection of the saved buffers (used by the parity tests: "tile indices bit-exact").
 * Each returns a device pointer INTO the given buffer. */
typedef struct GpsgGeomView {
    const float* depths;         /* [P] */
    const float* means2D;        /* [P,2] */
    const float* conic_opacity;  /* [P,4] */
    const uint32_t* tiles_touched; /* [P] */
    const uint32_t* point_offsets; /* [P] inclusive scan */
} GpsgGeomView;
typedef struct GpsgBinningView {
    const uint64_t* point_list_keys; /* [N] sorted */
    const uint32_t* point_list;      /* [N] sorted Gaussian ids */
    const float* slabA;              /* [N,4] (x, y, cull half-extent x, y), sorted */
    const uint32_t* block_lists;     /* [8N] per 8x4 block of a tile with range [s, s+n): its survivors' tile-local list
                                        positions at [8s + k*n, 8s + k*n + block_counts[8*tile + k]) */
} GpsgBinningView;
typedef struct GpsgImageView {
    const float* final_T;       /* [H*W] */
    const uint32_t* n_contrib;  /* [H*W] */
    const uint32_t* ranges;     /* [tiles,2] */
    const uint32_t* block_counts; /* [tiles,8] survivors per block (valid for non-empty tiles) */
} GpsgImageView;
GPSG_API int gpsg_geom_view(const void* geom_buffer, int P, GpsgGeomView* out);
GPSG_API int gpsg_binning_view(const void* binning_buffer, int64_t num_rendered, GpsgBinningView* out);
GPSG_API int gpsg_image_view(const void* image_buffer, int W, int H, GpsgImageView* out);

/* ---- replaces corr_sampler.forward (reference core/corr.py:22; SURVEY.md Appendix B) ---------
 * volume[B,H,W1,W2] with element strides (sb,sh,sw1; innermost contiguous), dtype 0=fp32 1=fp16;
 * coords: fp32, element (n,y,x) at coords[n*coords_sb + y*W1 + x] (channel 0 of [B,C,H,W1]);
 * out[B,2r+1,H,W1] contiguous, dtype of volume. */
GPSG_API int gpsg_corr_sampler_forward(int device, void* stream, int dtype, int B, int H, int W1, int W2, const void* volume,
                              int64_t sb, int64_t sh, int64_t sw1, const float* coords, int64_t coords_sb,
                              int radius, void* out);
/* ---- replaces corr_sampler.backward (reference core/corr.py:28) -------------------------------
 * grad_out[B,2r+1,H,W1] contiguous -> grad_volume[B,H,W1,W2] contiguous (fully written). */
GPSG_API int gpsg_corr_sampler_backward(int device, void* stream, int dtype, int B, int H, int W1, int W2,
                               const float* coords, int64_t coords_sb, const void* grad_out, int radius,
                               void* grad_volume);

/* ---- fused forms of the correlation block (reference core/corr.py:31-61), used by the mirrored CorrBlockFast1D ----
 * gpsg_corr_build_pyramid: fmap1[B,D,H,W1], fmap2[B,D,H,W2] (contiguous, dtype 0=fp32 1=fp16) ->
 *   vol[l][B,H,W1,W2>>l], l < levels<=4 : einsum/sqrt(D) then avg_pool2d([1,2]) per level, each level rounded to dtype.
 *   fp16 with D%16==0, D<=256, W1%8==0, W2%16==0, W2<=128 and 16-byte aligned pointers runs on the wgmma tensor-core kernel (csrc/corr_tc.cu),
 *   anything else on the FFMA kernel (csrc/corr.cu); same rounding chain, results agree to one fp16 ulp.  The environment
 *   variable GPSG_CORR_BUILD=ffma forces the FFMA kernels (tests compare the two).
 * gpsg_corr_lookup_pyramid_forward: all levels of CorrBlockFast1D.__call__ in one launch -> out[B, levels*(2r+1), H, W1]
 *   (coords: channel 0 of [B,C,H,W1] fp32, level l uses coords / 2^l).  _backward: grad_out -> grad_vol[l] (fully written). */
GPSG_API int gpsg_corr_build_pyramid(int device, void* stream, int dtype, int B, int D, int H, int W1, int W2,
                                     const void* fmap1, const void* fmap2, void* const* vols, int levels);
/* backward of the build w.r.t. the feature maps: grad_vol0[B,H,W1,W2] (pooled levels already folded in) -> d fmap1, d fmap2 */
GPSG_API int gpsg_corr_build_backward(int device, void* stream, int dtype, int B, int D, int H, int W1, int W2,
                                      const void* fmap1, const void* fmap2, const void* grad_vol0, void* dfmap1,
                                      void* dfmap2);
GPSG_API int gpsg_corr_lookup_pyramid_forward(int device, void* stream, int dtype, int B, int H, int W1,
                                              const void* const* vols, const int32_t* widths, int levels,
                                              const float* coords, int64_t coords_sb, int radius, void* out);
GPSG_API int gpsg_corr_lookup_pyramid_backward(int device, void* stream, int dtype, int B, int H, int W1,
                                               void* const* grad_vols, const int32_t* widths, int levels,
                                               const float* coords, int64_t coords_sb, int radius, const void* grad_out);

/* ---- fused unprojection, the producer of the rasterizer's means3D (reference lib/network.py:64-69 -> lib/utils.py:87-119:
 * flow2depth + depth2pc + `depth != 0`).  flow_pred[B,1,S,S], mask[B,C,S,S] (channel 0 used; batch stride in elements),
 * intr[B,3,3], extr[B,extr_rows>=3,4], ref_intr[B,3,3], Tf_x[B]  ->  depth[B,1,S,S], xyz[B,S*S,3], valid[B,S*S] (uint8).
 * Backward: dL_dxyz (and optionally an incoming dL_ddepth) -> dL_dflow[B,1,S,S]. */
GPSG_API int gpsg_unproject_forward(int device, void* stream, int B, int S, const float* flow_pred, const float* mask,
                                    int64_t mask_batch_stride, const float* intr, const float* extr, int extr_rows,
                                    const float* ref_intr, const float* Tf_x, float* depth, float* xyz, uint8_t* valid);
GPSG_API int gpsg_unproject_backward(int device, void* stream, int B, int S, const float* depth, const float* mask,
                                     int64_t mask_batch_stride, const float* intr, const float* extr, int extr_rows,
                                     const float* ref_intr, const float* Tf_x, const float* dL_dxyz,
                                     const float* dL_ddepth, float* dL_dflow);

/* ---- point splat: the stage-1 preview's 1-pixel z-buffer on inverse depth (reference lib/TaichiRender.py:13-24) ------
 * One call = one call of `render_respective_color` over the loop domain (B, N):
 *   pts[Bp, rows_per_batch, 6] = (x_pix, y_pix, inverse depth, r, g, b), mask[Bp, rows_per_batch] (point skipped when
 *   mask < 0.5), depth[Bp, 1, res, res] and color[Bp, 3, res, res] in/out, Bp >= B, rows_per_batch >= N.  Batches b >= B
 *   and rows i >= N are not read or written.
 * The result is the serial reading of the reference kernel (points in index order), race-free and bit-exact: per pixel,
 * with M the largest z landing there, colour <- rgb of the highest index with z == M when M >= old depth, and depth <-
 * M (the first such point's value) when M > old depth.  NaN z is skipped; x, y truncate towards zero with saturation
 * (NaN -> 0) and clamp to [0, res-1].
 * workspace: gpsg_point_splat_workspace_bytes(B, res) bytes, 8-byte aligned; the call zeroes it on the stream.
 * B == 0 or N == 0 is a no-op.  Refused (GPSG_E_INVALID): negative sizes, res < 1, N > rows_per_batch, res^2 >= 2^31,
 * NULL pointers when there is work. */
GPSG_API size_t gpsg_point_splat_workspace_bytes(int B, int res);
GPSG_API int gpsg_point_splat(int device, void* stream, int B, int N, int res, int64_t rows_per_batch, const float* pts,
                              const float* mask, float* depth, float* color, void* workspace);

/* ---- textured triangle mesh renderer of the dataset script (reference prepare_data/taichi_three) ---------------------
 * gpsg_mesh_render: one `Scene.render()` of the reference: every camera of `scene` is cleared and the mesh drawn into it,
 * in one launch chain on `stream`, without host synchronisation.  The result is the serial reading of the reference's
 * `render_triangle` (faces in index order): per pixel the face with the largest zindex = 1 / (screen-affine depth) wins,
 * the highest face index among equal zindex; the fp32 formulation is written down in csrc/mesh_render.cu.
 *   mesh (HOST struct of device pointers, by value):
 *     verts [num_verts,3] fp32; face_verts [num_faces,3] int32 (vertex indices);
 *     uvs [num_uvs,2] fp32 and face_uvs [num_faces,3] int32, or both NULL (every corner samples uv = (0, 0));
 *     tex [tex_w,tex_h,3] fp32 (the reference's texture field: tex[i,j] at uv*(tex_w, tex_h) = (i, j)), or NULL (the
 *     sample is 1).  A face with an index outside its array draws nothing.
 *   scene (HOST struct, by value): cameras[0..num_cameras), lights[0..num_lights).  Per camera: res = (width, height)
 *     (the reference's field shape (res[0], res[1])), fx, fy, cx, cy, pos, inv_rot = trans^-1 (row-major fp32; the caller
 *     inverts `trans` in fp64), and device outputs img [height,width,3], zbuf [height,width], mask [height,width,3] fp32
 *     (the reference's fields transposed to [y, x]; every pixel is written).  Per light: light_dir = the unit vector
 *     towards the light (-normalize(dir)), light_color.  A NaN img value is written as the canonical NaN 0x7fffffff.
 *   workspace: gpsg_mesh_render_workspace_bytes(num_faces, max over cameras of width*height) bytes, 256-byte aligned.
 * Refused (GPSG_E_INVALID): negative counts, num_cameras outside [1, GPSG_MESH_MAX_CAMERAS], num_lights outside
 * [0, GPSG_MESH_MAX_LIGHTS], a camera size < 1 or with >= 2^31 pixels, uvs without face_uvs (or the reverse), texture
 * sizes < 1, NULL pointers where there is data, a workspace smaller than the query or misaligned. */
#define GPSG_MESH_MAX_CAMERAS 8
#define GPSG_MESH_MAX_LIGHTS 16
typedef struct GpsgMesh {
    const float* verts;
    const int32_t* face_verts;
    const float* uvs;
    const int32_t* face_uvs;
    const float* tex;
    int32_t num_verts;
    int32_t num_faces;
    int32_t num_uvs;
    int32_t tex_w;
    int32_t tex_h;
} GpsgMesh;
typedef struct GpsgMeshCamera {
    int32_t width;
    int32_t height;
    float fx, fy, cx, cy;
    float pos[3];
    float inv_rot[9];
    float* img;
    float* zbuf;
    float* mask;
} GpsgMeshCamera;
typedef struct GpsgMeshScene {
    GpsgMeshCamera cameras[GPSG_MESH_MAX_CAMERAS];
    float light_dir[GPSG_MESH_MAX_LIGHTS][3];
    float light_color[GPSG_MESH_MAX_LIGHTS][3];
    int32_t num_cameras;
    int32_t num_lights;
} GpsgMeshScene;
GPSG_API size_t gpsg_mesh_render_workspace_bytes(int num_faces, int64_t max_pixels);
GPSG_API int gpsg_mesh_render(int device, void* stream, GpsgMesh mesh, GpsgMeshScene scene, void* workspace,
                              size_t workspace_bytes);

/* ---- stereo rectification of the real-data loader (reference lib/human_loader.py:245-366) ----------------------------
 * gpsg_rectify_remap: cv2.initUndistortRectifyMap(K, 0, R, P, (W, H), CV_32FC1) + cv2.remap(INTER_LINEAR,
 *   BORDER_CONSTANT 0) of both views of a pair in one launch, bit-identical to OpenCV 4.x (DESIGN.md §2).  cams[2] are
 *   HOST structs passed to the kernel by value: the source intrinsics K, the rectifying rotation R and P[:3,:3] of
 *   cv2.stereoRectify, all fp64 row-major.  Per view, planes[k] (HOST struct of device pointers):
 *     img [Hin,Win,C] uint8 (C in {1,3,4}); mask [Hin,Win,Cm] uint8 (Cm in {1,3,4}) or NULL; depth [Hin,Win] fp32 or NULL;
 *     numpy contract (what cv2.remap returns): img_out [H,W,C], mask_out [H,W,Cm] uint8, depth_out [H,W] fp32 (required
 *       with depth);
 *     tensor contract (stereo_to_dict_tensor, :319-331): img_tensor fp32 = (2*(v/255) - 1) * m_soft with m_soft =
 *       mask/255 (channel c of the mask, or channel 0 when Cm == 1; needs Cm == 1 or Cm == C), mask_tensor fp32 =
 *       (m_soft >= 0.5); both stored [H,W,C] / [H,W,Cm], i.e. the [C,H,W] tensors of that function with its strides
 *       (1, W*C, C), which it inherits from permuting the numpy image;
 *   any output may be NULL.  Refused: sizes < 1, unsupported C / Cm, NULL img, depth without depth_out, a tensor output
 *   that needs the mask without one.
 * gpsg_rectify_flow: the ground truth of stereo_pts2flow (:74-85) and the eroded valid mask (:298-315) of both views in
 *   one launch.  depth[k] [H,W] fp32 is the rectified depth (depth_out above), mask[k] [H,W,Cm] the rectified mask;
 *   flow[k] [H,W] fp64 = (cx_other - cx_self) - (-depth * Tf_x) (Tf_x -> -Tf_x for view 1), 0 where depth < 0.05, times
 *   valid; valid is the 3x3 erode (border +inf) of fp32(mask[...,0] / 255.0) thresholded at 0.66; valid[k] [H,W] uint8 =
 *   255 * valid.  cx0 / cx1 are P0[0,2] / P1[0,2].  Pointer arrays are host arrays of device pointers.
 * Both enqueue one kernel on `stream` and do not synchronise. */
typedef struct GpsgRectifyCamera {
    double K[9];
    double R[9];
    double P[9];
} GpsgRectifyCamera;
typedef struct GpsgRectifyPlanes {
    const uint8_t* img;
    const uint8_t* mask;
    const float* depth;
    uint8_t* img_out;
    uint8_t* mask_out;
    float* depth_out;
    float* img_tensor;
    float* mask_tensor;
} GpsgRectifyPlanes;
GPSG_API int gpsg_rectify_remap(int device, void* stream, const GpsgRectifyCamera* cams, int Hin, int Win, int C, int Cm,
                                int H, int W, const GpsgRectifyPlanes* planes);
GPSG_API int gpsg_rectify_flow(int device, void* stream, int H, int W, int Cm, double Tf_x, double cx0, double cx1,
                               const float* const* depth, const uint8_t* const* mask, double* const* flow,
                               uint8_t* const* valid);

/* ---- baseline JPEG decoding (the loader's source frames; rules in DESIGN.md §2 "JPEG decoding") ----------------------
 * gpsg_jpeg_parse: reads the markers of one JPEG file (host memory, `size` bytes) into `info`.  Returns 0 when the image
 *   is decoded natively, else a refusal code GPSG_JPEG_E_* (> 0; `info` is then partial), or GPSG_E_INVALID for NULL
 *   pointers.  Every length field is checked against `size`; nothing past it is read.  Decoded natively: SOF0 / SOF1,
 *   8-bit, one scan holding every component in frame order, Huffman coded; one component (Pillow mode L), or three
 *   YCbCr components with chroma 1x1 and luma 1x1, 2x1 or 2x2.
 * gpsg_jpeg_decode_workspace_bytes: the workspace of one gpsg_jpeg_decode over these infos (0 when they are refused).
 * gpsg_jpeg_decode: decodes n <= GPSG_JPEG_MAX_BATCH parsed images in one launch chain on `stream`.  data[i]: DEVICE
 *   pointer to the whole file of image i (the bytes gpsg_jpeg_parse read); out[i]: DEVICE [H,W] (one component) or
 *   [H,W,3] uint8, what Pillow's np.array(Image.open(f)) holds; status: DEVICE uint32[n], set to 0 and then to the
 *   GPSG_JPEG_ST_* bits of whatever made image i undecodable (its `out` is then unspecified).  The caller reads the
 *   status words after the stream reaches this call.  workspace: gpsg_jpeg_decode_workspace_bytes bytes, 256-byte
 *   aligned.  Refused: bad n, NULL pointers, infos that gpsg_jpeg_parse would refuse, a batch whose scans reach
 *   GPSG_JPEG_MAX_SCAN_BYTES (gpsg_jpeg_decode_workspace_bytes then returns 0), a short workspace. */
#define GPSG_JPEG_MAX_BATCH 64
#define GPSG_JPEG_MAX_SCAN_BYTES (1 << 28)   /* entropy-coded bytes of one gpsg_jpeg_decode, summed over its images */
#define GPSG_JPEG_E_TRUNCATED 1     /* a length field, the scan or the EOI marker lies past the end of the buffer */
#define GPSG_JPEG_E_MALFORMED 2     /* a marker or table that T.81 does not allow, or a table the scan needs is missing */
#define GPSG_JPEG_E_PROGRESSIVE 3   /* SOF2 */
#define GPSG_JPEG_E_ARITHMETIC 4    /* SOF9 / SOF10 / DAC */
#define GPSG_JPEG_E_LOSSLESS 5      /* SOF3 / SOF7 / SOF11 / SOF15 */
#define GPSG_JPEG_E_HIERARCHICAL 6  /* SOF5 / SOF6 / SOF13 / SOF14 */
#define GPSG_JPEG_E_PRECISION 7     /* sample precision other than 8 bits */
#define GPSG_JPEG_E_COLORSPACE 8    /* 2 or 4 components (CMYK), or RGB (Adobe transform 0, or R/G/B component ids) */
#define GPSG_JPEG_E_SAMPLING 9      /* sampling factors other than the three layouts above */
#define GPSG_JPEG_E_MULTISCAN 10    /* more than one scan, or a scan without every component in frame order */
#define GPSG_JPEG_E_DNL 11          /* height 0 / a DNL marker */
#define GPSG_JPEG_ST_BAD_CODE 1u    /* a Huffman code no table holds */
#define GPSG_JPEG_ST_OVERRUN 2u     /* a code or its bits run past the end of the restart segment */
#define GPSG_JPEG_ST_MCU_COUNT 4u   /* a restart segment (or the image) holds the wrong number of MCUs, or bad padding */
#define GPSG_JPEG_ST_RST 8u         /* an RSTn marker out of sequence */
#define GPSG_JPEG_ST_MARKER 16u     /* a marker other than RSTn or a stuffed 0xFF inside the scan */
#define GPSG_JPEG_ST_COEF 32u       /* a coefficient past index 63, or a magnitude category beyond 8-bit baseline */
typedef struct GpsgJpegInfo {
    int32_t width, height, num_components, restart_interval;
    int32_t h_samp[3], v_samp[3], quant_id[3], dc_id[3], ac_id[3];
    uint16_t quant[4][64];                      /* zigzag order */
    uint8_t dc_bits[4][16], ac_bits[4][16];     /* codes of length 1..16 */
    uint8_t dc_vals[4][256], ac_vals[4][256];
    int64_t ecs_offset, ecs_length;             /* the entropy-coded segment (RSTn markers included) in the file */
} GpsgJpegInfo;
GPSG_API int gpsg_jpeg_parse(const uint8_t* data, size_t size, GpsgJpegInfo* info);
GPSG_API size_t gpsg_jpeg_decode_workspace_bytes(int n, const GpsgJpegInfo* infos);
GPSG_API int gpsg_jpeg_decode(int device, void* stream, int n, const GpsgJpegInfo* infos, const uint8_t* const* data,
                              uint8_t* const* out, uint32_t* status, void* workspace, size_t workspace_bytes);

/* ---- baseline JPEG encoding (the output JPEGs; rules in DESIGN.md §2 "JPEG encoding") ---------------------------------
 * The file cv2.imencode('.jpg') and Pillow's save('JPEG') write with libjpeg-turbo's defaults at `quality`: Annex K
 * tables, islow FDCT, no Huffman optimisation, no restart markers, one interleaved scan, JFIF APP0.
 * GpsgJpegEncodeDesc: width, height in 1..65500; channels 1 (grayscale; `sampling` is then ignored but must be valid) or
 *   3 (interleaved, channel order GPSG_JPEG_ORDER_RGB or _BGR); pitch: bytes between rows, >= width * channels;
 *   quality 1..100; sampling 444, 422 or 420 (4:4:4, 4:2:2, 4:2:0 chroma).
 * gpsg_jpeg_encode_max_bytes: an upper bound on the file of one image (0 for a refused descriptor).
 * gpsg_jpeg_encode_workspace_bytes: the workspace of one gpsg_jpeg_encode over these descriptors (0 when refused, also
 *   for a batch too large for one call: 2^31 blocks or 2^30 32-bit words of 1664 bits per block).
 * gpsg_jpeg_encode: encodes n <= GPSG_JPEG_MAX_BATCH images in one launch chain on `stream`.  src[i]: DEVICE rows of
 *   image i; out[i]: DEVICE buffer of gpsg_jpeg_encode_max_bytes(descs + i) bytes, of which the first out_sizes[i]
 *   (DEVICE int64[n]) hold the complete file; nothing past them is written.  The caller reads out_sizes after the stream
 *   reaches this call.  workspace: gpsg_jpeg_encode_workspace_bytes bytes, 256-byte aligned.  Refused before any launch:
 *   bad n, NULL pointers, a refused descriptor, a short or misaligned workspace. */
#define GPSG_JPEG_ORDER_RGB 0
#define GPSG_JPEG_ORDER_BGR 1
typedef struct GpsgJpegEncodeDesc {
    int32_t width, height, channels, order, quality, sampling;
    int64_t pitch;
} GpsgJpegEncodeDesc;
GPSG_API size_t gpsg_jpeg_encode_max_bytes(const GpsgJpegEncodeDesc* desc);
GPSG_API size_t gpsg_jpeg_encode_workspace_bytes(int n, const GpsgJpegEncodeDesc* descs);
GPSG_API int gpsg_jpeg_encode(int device, void* stream, int n, const GpsgJpegEncodeDesc* descs, const uint8_t* const* src,
                              uint8_t* const* out, int64_t* out_sizes, void* workspace, size_t workspace_bytes);

/* ---- disparity head of both training stages (reference core/raft_stereo_human.py:69-81 and lib/loss.py:8-33) -----------
 * gpsg_convex_upsample_forward: FlowUpdateModule.upsample_flow.  flow [N,D,H,W] fp32, mask [N,9*f*f,H,W] of `mask_dtype`
 *   (0 = fp32, 1 = fp16), both contiguous; out [N,D,f*H,f*W] fp32.  With tap k = 3*ky + kx and mask channel
 *   k*f^2 + i*f + j: w = softmax over k of the 9 logits, computed in fp32 (max-subtracted exp over their sum) and rounded
 *   to the mask dtype; out[n,d,h*f+i,w*f+j] = sum_{k=0..8} w * f*flow[n,d,h+ky-1,w+kx-1] with fp32 products and sum,
 *   zero padding (padded taps keep their weight).  f in {2, 4, 8}, D in {1, 2}.
 * gpsg_convex_upsample_backward: grad_out [N,D,f*H,f*W] fp32 -> grad_mask (mask dtype; the weights are recomputed from
 *   the mask, dL/dweight is rounded to the mask dtype before the softmax backward) and grad_flow [N,D,H,W] fp32; either may
 *   be NULL, not both.  workspace: gpsg_convex_upsample_backward_workspace_bytes bytes, 4-byte aligned (the per-pixel tap
 *   sums, gathered into grad_flow without atomics, so the result is deterministic).
 * gpsg_sequence_loss_forward: args->pred[0..n_pred) and valid: `numel` fp32 elements each (the [N,1,H,W] tensors); gt:
 *   `numel` elements of `gt_dtype` (0 = fp32, 1 = fp16: the training cache's flow, widened exactly to fp32);
 *   stats (device float[6]) = { loss, EPE mean, fraction of EPE < 1, fraction of EPE < 3, 1 if gt is inf at a valid
 *   pixel else 0, 1 / valid count (in fp64, rounded once to fp32) }, with valid = (valid >= 0.5),
 *   loss = sum_i weight[i] * mean_valid |pred_i - gt| and EPE = sqrt((pred_last - gt)^2) in fp32.  Reductions run in a fixed order: bit-reproducible.  workspace:
 *   gpsg_sequence_loss_workspace_bytes() bytes, 8-byte aligned.
 * gpsg_sequence_loss_backward: args->grad[i] (numel fp32 each) = d(grad_loss * loss)/d(pred_i), reading 1 / count from
 *   the forward's stats; grad_loss is a DEVICE pointer to one float (NULL = 1).  No host synchronisation.
 * All enqueue on `stream` and do not synchronise. */
#define GPSG_SEQ_LOSS_MAX_PRED 32
typedef struct GpsgSeqLossArgs {
    const float* pred[GPSG_SEQ_LOSS_MAX_PRED];
    float* grad[GPSG_SEQ_LOSS_MAX_PRED];
    float weight[GPSG_SEQ_LOSS_MAX_PRED];
    const void* gt;
    const float* valid;
    int64_t numel;
    int n_pred;
    int gt_dtype;
} GpsgSeqLossArgs;
GPSG_API int gpsg_convex_upsample_forward(int device, void* stream, int mask_dtype, int factor, int N, int D, int H, int W,
                                          const float* flow, const void* mask, float* out);
GPSG_API size_t gpsg_convex_upsample_backward_workspace_bytes(int N, int D, int H, int W);
GPSG_API int gpsg_convex_upsample_backward(int device, void* stream, int mask_dtype, int factor, int N, int D, int H,
                                           int W, const float* flow, const void* mask, const float* grad_out,
                                           void* grad_mask, float* grad_flow, void* workspace);
GPSG_API size_t gpsg_sequence_loss_workspace_bytes(void);
GPSG_API int gpsg_sequence_loss_forward(int device, void* stream, GpsgSeqLossArgs args, float* stats, void* workspace);
GPSG_API int gpsg_sequence_loss_backward(int device, void* stream, GpsgSeqLossArgs args, const float* grad_loss,
                                         const float* stats);

/* ---- full-resolution tail of the Gaussian-parameter regressor (reference lib/gs_parm_network.py, GSRegresser) -------
 * gpsg_gs_head_forward: from the decoder1 output to the three parameter maps, forward only:
 *   up   = bilinear x2 upsampling of src [B,48,H/2,W/2] (align_corners=False: source (dst + 0.5) / 2 - 0.5, clamped at
 *          0 below, upper neighbour clamped to the last row / column);
 *   mid  = relu(conv3x3(cat[up, img [B,3,H,W], depth [B,1,H,W]], out_w, out_b)), zero padding of the concatenation;
 *   rot  [B,4,H,W] = normalize(conv1x1(relu(conv3x3(mid, rot_w1, rot_b1)), rot_w2, rot_b2)), x / max(||x||, 1e-12);
 *   scale [B,3,H,W] = min(softplus_100(conv1x1(relu(conv3x3(mid, scale_w1, ...)), ...)), 0.01), softplus_100(x) = x
 *          where 100 x > 20, else log1p(exp(100 x)) / 100;
 *   opacity [B,1,H,W] = sigmoid(conv1x1(relu(conv3x3(mid, opacity_w1, ...)), ...)).
 *   Weights in torch's layouts: out_w [32,52,3,3], *_w1 [32,32,3,3], rot_w2 [4,32,1,1], scale_w2 [3,32,1,1],
 *   opacity_w2 [1,32,1,1], biases [Cout]; every tensor fp32 and contiguous.  Every convolution operand (weights and
 *   activations) is rounded to TF32 (round to nearest, ties away), products and sums are fp32 in an unspecified order:
 *   the precision class of cuDNN with allow_tf32.  ReLU and the clamp keep NaN.  H and W even, B >= 0.
 *   workspace: gpsg_gs_head_workspace_bytes(B, H, W) bytes, 16-byte aligned (the 32-channel intermediate).
 *   Enqueues on `stream` and does not synchronise. */
typedef struct GpsgGsHeadWeights {
    const float* out_w; const float* out_b;
    const float* rot_w1; const float* rot_b1; const float* rot_w2; const float* rot_b2;
    const float* scale_w1; const float* scale_b1; const float* scale_w2; const float* scale_b2;
    const float* opacity_w1; const float* opacity_b1; const float* opacity_w2; const float* opacity_b2;
} GpsgGsHeadWeights;
GPSG_API size_t gpsg_gs_head_workspace_bytes(int B, int H, int W);
GPSG_API int gpsg_gs_head_forward(int device, void* stream, int B, int H, int W, const float* src, const float* img,
                                  const float* depth, float* rot, float* scale, float* opacity, GpsgGsHeadWeights weights,
                                  void* workspace);

/* gpsg_gs_head_backward: the gradients of gpsg_gs_head_forward's maps with respect to src, depth and the 14 weights, from
 * the upstream gradients g_rot [B,4,H,W], g_scale [B,3,H,W], g_opacity [B,1,H,W] (fp32, contiguous):
 *   d_src [B,48,H/2,W/2] (NULL: not computed), d_depth [B,1,H,W] (NULL: not computed), and `grads`, 14 device
 *   pointers in GpsgGsHeadWeights order and torch's layouts, all required.  The image's gradient is not computed.
 *   mid: the forward's workspace after gpsg_gs_head_forward on the same inputs and weights (the 32-channel intermediate),
 *   16-byte aligned; the pre-activations of the heads are recomputed from it.
 *   Masks and branches are those of torch's autograd on the forward's maths: ReLU passes the gradient where its result
 *   is not <= 0 (NaN passes), clamp_max(0.01) where the softplus is <= 0.01, softplus(beta 100, threshold 20) takes
 *   g where 100 x > 20 and g e / (e + 1), e = exp(100 x), elsewhere, normalize differentiates x / clamp_min(||x||,
 *   1e-12) with the norm's branch masked below 1e-12, sigmoid uses g (1 - y) y; the upsample's adjoint multiplies
 *   every interpolation weight in, zero weights included.  Non-finite upstream gradients reach the outputs as they do
 *   through torch's autograd.
 *   Precision as the forward: every convolution operand, forward recomputation and backward GEMMs (dh and dmid, the
 *   intermediates they read, the weights) is rounded to TF32 (round to nearest, ties away), products and sums are fp32.
 *   Bit-reproducible: no floating-point atomics; every sum has a fixed order given the shape and the device's SM count.
 *   workspace: gpsg_gs_head_backward_workspace_bytes(B, H, W) bytes, 16-byte aligned (128 channels per pixel of NHWC
 *   scratch and the per-CTA partial sums).  H and W even, B >= 0.  Enqueues on `stream` and does not synchronise. */
typedef struct GpsgGsHeadGrads {
    float* out_w; float* out_b;
    float* rot_w1; float* rot_b1; float* rot_w2; float* rot_b2;
    float* scale_w1; float* scale_b1; float* scale_w2; float* scale_b2;
    float* opacity_w1; float* opacity_b1; float* opacity_w2; float* opacity_b2;
} GpsgGsHeadGrads;
GPSG_API size_t gpsg_gs_head_backward_workspace_bytes(int B, int H, int W);
GPSG_API int gpsg_gs_head_backward(int device, void* stream, int B, int H, int W, const float* src, const float* img,
                                   const float* depth, const float* mid, const float* g_rot, const float* g_scale,
                                   const float* g_opacity, float* d_src, float* d_depth, GpsgGsHeadWeights weights,
                                   GpsgGsHeadGrads grads, void* workspace);

/* ---- half-resolution stem of the UnetExtractor (reference core/extractor.py: in_ds + res1), inference ------------------
 * gpsg_encoder_stem_forward: x1 [B,32,Ho,Wo] (NCHW fp32, Ho = ceil(H/2), Wo = ceil(W/2)), the output of res1, from the
 * input [B,Cin,H,W] (NCHW fp32, Cin 1 or 3, H, W >= 1):
 *   x0 = relu(GN8(conv5x5(input, in_conv_w, in_conv_b; stride 2, zero padding 2)))
 *   per residual block k = 1, 2 (input x, no downsample branch):
 *     h = relu(GN4(conv3x3(x, bk_conv1_w, bk_conv1_b)));  g = relu(GN4(conv3x3(h, bk_conv2_w, bk_conv2_b)));
 *     out = relu(x + g)
 *   GNg(y): GroupNorm with g groups over 32 channels per sample, biased variance, (y - mean) / sqrt(var + 1e-5) times
 *   the channel's weight plus its bias (evaluated as fmaf(y, A, C) with A = w rstd and C = b - mean A in fp32, the
 *   statistics in fp64).  A non-finite value in a (sample, group) makes that group NaN; ReLU keeps NaN.
 *   Weights in torch's layouts, every tensor fp32 and contiguous: in_conv_w [32,Cin,5,5], the 3x3 weights [32,32,3,3],
 *   biases and the GroupNorm weights / biases [32].
 *   precision GPSG_ENCODER_STEM_TF32 (cuDNN with allow_tf32): every convolution operand, weights and activations, rounded
 *     to TF32 (round to nearest, ties away); products and sums fp32 in an unspecified order; the bias added in fp32.
 *   precision GPSG_ENCODER_STEM_FP16 (CUDA autocast in fp16): the convolution operands (the input, each convolution's
 *     normalized input, the weights) and the biases rounded to fp16 (round to nearest even); products and sums fp32;
 *     each convolution's output, bias included, rounded to fp16 before GroupNorm reads it; GroupNorm, ReLU and the
 *     residual add in fp32.
 *   Bit-reproducible: no floating-point atomics; every sum has a fixed order given the shape and the device's SM count.
 *   workspace: gpsg_encoder_stem_workspace_bytes(B, Cin, H, W, precision) bytes, 256-byte aligned.  After the call it
 *   starts with the five raw convolution outputs y0 .. y4 (bias included, NHWC [B,Ho,Wo,32], fp32 in TF32 mode, fp16 in
 *   FP16 mode), y_i at byte i * S with S = B Ho Wo 32 sizeof(element) rounded up to a multiple of 256; then the
 *   per-channel A, C and the per-tile GroupNorm partials.  B >= 0.
 *   Enqueues on `stream` and does not synchronise. */
#define GPSG_ENCODER_STEM_TF32 0
#define GPSG_ENCODER_STEM_FP16 1
typedef struct GpsgEncoderStemWeights {
    const float* in_conv_w; const float* in_conv_b; const float* in_norm_w; const float* in_norm_b;
    const float* b1_conv1_w; const float* b1_conv1_b; const float* b1_norm1_w; const float* b1_norm1_b;
    const float* b1_conv2_w; const float* b1_conv2_b; const float* b1_norm2_w; const float* b1_norm2_b;
    const float* b2_conv1_w; const float* b2_conv1_b; const float* b2_norm1_w; const float* b2_norm1_b;
    const float* b2_conv2_w; const float* b2_conv2_b; const float* b2_norm2_w; const float* b2_norm2_b;
} GpsgEncoderStemWeights;
GPSG_API size_t gpsg_encoder_stem_workspace_bytes(int B, int Cin, int H, int W, int precision);
GPSG_API int gpsg_encoder_stem_forward(int device, void* stream, int B, int Cin, int H, int W, int precision,
                                       const float* input, GpsgEncoderStemWeights weights, float* x1_out,
                                       void* workspace);

/* ---- decoder1 of the Gaussian-parameter regressor (reference lib/gs_parm_network.py, two ResidualBlocks), inference ----
 * gpsg_decoder1_forward: out [B,48,H,W] (NCHW fp32, H = 2 Hs, W = 2 Ws), the output of `decoder1` on
 * cat(up2x(s), img_feat, depth_feat), from s [B,64,Hs,Ws] (the decoder2 output), img_feat and depth_feat [B,32,H,W]
 * (NCHW fp32, contiguous, Hs, Ws >= 1):
 *   up2x: bilinear x2, align_corners=False, as torch's upsample_bilinear2d: source (d + 0.5) / 2 - 0.5 clamped at 0,
 *     i0 = floor, i1 = min(i0 + 1, n - 1), evaluated in fp32 as l0y (l0x a + l1x b) + l1y (l0x c + l1x d);
 *   v = cat(up2x(s), img_feat, depth_feat) [B,128,H,W] (never stored);
 *   block 0: y1 = conv3x3(v, b0_conv1) ; yd = conv1x1(v, b0_down) ; y2 = conv3x3(relu(GN6(y1)), b0_conv2) ;
 *            xb = relu(GN6(yd) + relu(GN6(y2)))       (no ReLU on the downsample branch before the add)
 *   block 1: y3 = conv3x3(xb, b1_conv1) ; y4 = conv3x3(relu(GN6(y3)), b1_conv2) ; out = relu(xb + relu(GN6(y4)))
 *   every convolution with its bias and zero padding 1 (3x3) or 0 (1x1).
 *   GN6(y): GroupNorm(6, 48) per sample (8 channels per group), biased variance, eps 1e-5, the channel's weight and bias;
 *   evaluated as fmaf(y, A, C) with A = w rstd and C = b - mean A rounded to fp32, the statistics in fp64 from the stored
 *   fp32 y.  A non-finite value in a (sample, group) makes that group NaN; ReLU keeps NaN.
 *   Precision (cuDNN with allow_tf32): every convolution operand, weights and activations (the interpolated, normalized
 *   and residual-added values included), rounded to TF32 (round to nearest, ties away); products and sums fp32 in an
 *   unspecified order; the fp32 bias added after the sum.
 *   Weights in torch's layouts, fp32 and contiguous: b0_conv1_w [48,128,3,3], b0_down_w [48,128,1,1], the other 3x3
 *   weights [48,48,3,3], biases and GroupNorm weights / biases [48].
 *   Bit-reproducible: no floating-point atomics; every sum has a fixed order given the shape and the device's SM count.
 *   workspace: gpsg_decoder1_workspace_bytes(B, Hs, Ws) bytes, 256-byte aligned.  After the call it starts with the five
 *   raw convolution outputs y1, yd, y2, y3, y4 in that order (bias included, NHWC [B,H,W,48] fp32), the i-th at byte
 *   i * S with S = B H W 48 * 4 rounded up to a multiple of 256; then the per-channel A, C, the per-tile GroupNorm
 *   partials and the TF32-packed weights.  B >= 0 (B = 0 does nothing); Hs, Ws >= 1; NULL pointers are refused.
 *   Enqueues on `stream` and does not synchronise. */
typedef struct GpsgDecoder1Weights {
    const float* b0_conv1_w; const float* b0_conv1_b; const float* b0_norm1_w; const float* b0_norm1_b;
    const float* b0_conv2_w; const float* b0_conv2_b; const float* b0_norm2_w; const float* b0_norm2_b;
    const float* b0_down_w; const float* b0_down_b; const float* b0_norm3_w; const float* b0_norm3_b;
    const float* b1_conv1_w; const float* b1_conv1_b; const float* b1_norm1_w; const float* b1_norm1_b;
    const float* b1_conv2_w; const float* b1_conv2_b; const float* b1_norm2_w; const float* b1_norm2_b;
} GpsgDecoder1Weights;
GPSG_API size_t gpsg_decoder1_workspace_bytes(int B, int Hs, int Ws);
GPSG_API int gpsg_decoder1_forward(int device, void* stream, int B, int Hs, int Ws, const float* s, const float* img_feat,
                                   const float* depth_feat, GpsgDecoder1Weights weights, float* out, void* workspace);

/* ---- decoder3 and decoder2 of the Gaussian-parameter regressor (reference lib/gs_parm_network.py), inference ----------
 * gpsg_decoder3_forward: out [B,96,H,W] (NCHW fp32), the output of `decoder3` on cat(img_feat, depth_feat), from
 * img_feat and depth_feat [B,96,H,W] (img_feat3, depth_feat3; NCHW fp32, contiguous, H, W >= 1).  GN: GroupNorm(12, 96).
 * gpsg_decoder2_forward: out [B,64,H,W] (H = 2 Hs, W = 2 Ws), the output of `decoder2` on
 * cat(up2x(s), img_feat, depth_feat), from s [B,96,Hs,Ws] (the decoder3 output), img_feat and depth_feat [B,48,H,W]
 * (img_feat2, depth_feat2; Hs, Ws >= 1).  up2x is gpsg_decoder1_forward's.  GN: GroupNorm(8, 64).
 * In both, with v the concatenated input [B,192,H,W] (never stored) and C the output channels:
 *   block 0: ya = conv3x3(v, b0_conv1) ; yd = conv1x1(v, b0_down) ; yb = conv3x3(relu(GN(ya)), b0_conv2) ;
 *            xb = relu(GN(yd) + relu(GN(yb)))       (no ReLU on the downsample branch before the add)
 *   block 1: yc = conv3x3(xb, b1_conv1) ; ye = conv3x3(relu(GN(yc)), b1_conv2) ; out = relu(xb + relu(GN(ye)))
 *   every convolution with its bias and zero padding 1 (3x3) or 0 (1x1).
 *   GN(y): GroupNorm(C/8, C) per sample (8 channels per group) with its own weight and bias (norm1, norm2, norm3 in
 *   order of use), biased variance, eps 1e-5, evaluated as fmaf(y, A, C) with A = w rstd and C = b - mean A rounded to
 *   fp32, the statistics in fp64 from the stored fp32 y.  A non-finite value in a (sample, group) makes that group NaN;
 *   ReLU keeps NaN.
 *   Precision (cuDNN with allow_tf32): every convolution operand, weights and activations (the interpolated, normalized
 *   and residual-added values included), rounded to TF32 (round to nearest, ties away); products and sums fp32 in an
 *   unspecified order; the fp32 bias added after the sum.
 *   Weights in torch's layouts, fp32 and contiguous, in GpsgDecoder1Weights' field order: b0_conv1_w [C,192,3,3],
 *   b0_down_w [C,192,1,1], the other 3x3 weights [C,C,3,3], biases and GroupNorm weights / biases [C].
 *   Bit-reproducible: no floating-point atomics; every sum has a fixed order given the shape and the device's SM count.
 *   workspace: gpsg_decoder3_workspace_bytes(B, H, W) / gpsg_decoder2_workspace_bytes(B, Hs, Ws) bytes, 256-byte
 *   aligned.  After the call it starts with the five raw convolution outputs ya, yd, yb, yc, ye in that order (bias
 *   included, NHWC [B,H,W,C] fp32), the i-th at byte i * S with S = B H W C * 4 rounded up to a multiple of 256; then the
 *   per-channel A, C, the per-tile GroupNorm partials and the TF32-packed weights.  B >= 0 (B = 0 does nothing); sizes
 *   >= 1; NULL pointers are refused.  Enqueues on `stream` and does not synchronise. */
typedef struct GpsgDecoder23Weights {
    const float* b0_conv1_w; const float* b0_conv1_b; const float* b0_norm1_w; const float* b0_norm1_b;
    const float* b0_conv2_w; const float* b0_conv2_b; const float* b0_norm2_w; const float* b0_norm2_b;
    const float* b0_down_w; const float* b0_down_b; const float* b0_norm3_w; const float* b0_norm3_b;
    const float* b1_conv1_w; const float* b1_conv1_b; const float* b1_norm1_w; const float* b1_norm1_b;
    const float* b1_conv2_w; const float* b1_conv2_b; const float* b1_norm2_w; const float* b1_norm2_b;
} GpsgDecoder23Weights;
GPSG_API size_t gpsg_decoder3_workspace_bytes(int B, int H, int W);
GPSG_API int gpsg_decoder3_forward(int device, void* stream, int B, int H, int W, const float* img_feat,
                                   const float* depth_feat, GpsgDecoder23Weights weights, float* out, void* workspace);
GPSG_API size_t gpsg_decoder2_workspace_bytes(int B, int Hs, int Ws);
GPSG_API int gpsg_decoder2_forward(int device, void* stream, int B, int Hs, int Ws, const float* s, const float* img_feat,
                                   const float* depth_feat, GpsgDecoder23Weights weights, float* out, void* workspace);

/* ---- stride-2 residual stages of the UnetExtractor (reference core/extractor.py: res2, res3), inference -------------
 * gpsg_encoder_down_forward: out [B,C,Ho,Wo] (NCHW fp32, Ho = ceil(H/2), Wo = ceil(W/2)), the output of one stage of
 * two ResidualBlocks (the first with stride 2 and a 1x1 downsample) on input [B,Cin,H,W] (NCHW fp32, H, W >= 1);
 * (Cin, C) is (32, 48) (res2 of encoder_dims [32, 48, 96]) or (48, 96) (res3), any other pair is refused:
 *   block 0: ya = conv3x3(input, b0_conv1; stride 2, padding 1) ; yd = conv1x1(input, b0_down; stride 2, padding 0) ;
 *            yb = conv3x3(relu(GN(ya)), b0_conv2) ; xb = relu(GN(yd) + relu(GN(yb)))   (no ReLU on the downsample)
 *   block 1: yc = conv3x3(xb, b1_conv1) ; ye = conv3x3(relu(GN(yc)), b1_conv2) ; out = relu(xb + relu(GN(ye)))
 *   every convolution with its bias; the 3x3 ones of block 1 and conv2 with stride 1, padding 1.
 *   GN(y): GroupNorm(C/8, C) per sample with its own weight and bias (norm1, norm2, norm3 in order of use), biased
 *   variance, eps 1e-5, evaluated as fmaf(y, A, C) with A = w rstd and C = b - mean A rounded to fp32, the statistics in
 *   fp64.  A non-finite value in a (sample, group) makes that group NaN; ReLU keeps NaN.
 *   precision GPSG_ENCODER_STEM_TF32 / _FP16 with gpsg_encoder_stem_forward's semantics: TF32 operands (the input, each
 *   normalized input, the weights) and fp32 outputs, or fp16 operands and biases with each convolution's output, bias
 *   included, rounded to fp16; GroupNorm, ReLU and the residual adds in fp32 in both.
 *   Weights in torch's layouts, fp32 and contiguous: b0_conv1_w [C,Cin,3,3], b0_down_w [C,Cin,1,1], the other 3x3 weights
 *   [C,C,3,3], biases and GroupNorm weights / biases [C]; the field order is GpsgDecoder1Weights'.
 *   Bit-reproducible: no floating-point atomics; every sum has a fixed order given the shape and the device's SM count.
 *   workspace: gpsg_encoder_down_workspace_bytes(B, Cin, C, H, W, precision) bytes, 256-byte aligned.  After the call it
 *   starts with the five raw convolution outputs ya, yd, yb, yc, ye in that order (bias included, NHWC [B,Ho,Wo,C], fp32
 *   in TF32 mode, fp16 in FP16 mode), the i-th at byte i * S with S = B Ho Wo C sizeof(element) rounded up to a multiple
 *   of 256; then the per-channel A, C, the per-tile GroupNorm partials and the packed weights.  B >= 0 (B = 0 does
 *   nothing); NULL pointers are refused.  Enqueues on `stream` and does not synchronise. */
typedef struct GpsgEncoderDownWeights {
    const float* b0_conv1_w; const float* b0_conv1_b; const float* b0_norm1_w; const float* b0_norm1_b;
    const float* b0_conv2_w; const float* b0_conv2_b; const float* b0_norm2_w; const float* b0_norm2_b;
    const float* b0_down_w; const float* b0_down_b; const float* b0_norm3_w; const float* b0_norm3_b;
    const float* b1_conv1_w; const float* b1_conv1_b; const float* b1_norm1_w; const float* b1_norm1_b;
    const float* b1_conv2_w; const float* b1_conv2_b; const float* b1_norm2_w; const float* b1_norm2_b;
} GpsgEncoderDownWeights;
GPSG_API size_t gpsg_encoder_down_workspace_bytes(int B, int Cin, int C, int H, int W, int precision);
GPSG_API int gpsg_encoder_down_forward(int device, void* stream, int B, int Cin, int C, int H, int W, int precision,
                                       const float* input, GpsgEncoderDownWeights weights, float* out, void* workspace);

/* ---- disparity update block (reference core/update.py: BasicMultiUpdateBlock, n_gru_layers = 1), inference --------
 * One RAFT iteration of FlowUpdateModule.forward under CUDA autocast in fp16, at 1/8 resolution [H,W], hidden dims 96,
 * corr_levels 4, corr_radius 4, n_downsample 3.  With flow = fp16(coords1 - coords0) (coords0 the pixel grid, x then y):
 *   cor = relu(convc2(relu(convc1(corr))))  flo = relu(convf2(relu(convf1(flow))))   (1x1 36->64, 3x3, 7x7 2->64, 3x3)
 *   x = [relu(conv([cor, flo])), flow]  (3x3 128->126, then the two fp16 flow channels)
 *   z = sigmoid(convz([h, x]) + cz)   r = sigmoid(convr([h, x]) + cr)   q = tanh(convq([r*h, x]) + cq)
 *   h = (1 - z) h + z q
 *   delta = flow_head.conv2(relu(flow_head.conv1(h)))   coords1[:, 0] += delta[:, 0] (fp32; channel 1 is zeroed)
 *   mask = .25 * mask[2](relu(mask[0](h)))               (only when mask_out is not NULL)
 *   Every convolution takes fp16 operands and an fp16 bias and accumulates in fp32; its output is rounded to fp16, then
 *   the bias added and rounded again (cuDNN's convolution followed by the bias add).  Each elementwise op above rounds
 *   to fp16 as autocast's fp16 tensors do: the + cz / cr / cq adds, sigmoid, tanh, r*h, 1-z, (1-z) h, z q, their sum and
 *   the .25 scale.  ReLU keeps NaN.
 * gpsg_update_pack: the 24 fp32 weights (contiguous, torch's layouts) rounded to fp16 (to nearest even) into `packed`,
 *   gpsg_update_packed_bytes() bytes, 256-byte aligned.  Enqueues on `stream`.
 * gpsg_update_step: one iteration.  corr [B,36,H,W] NCHW contiguous, fp16 (corr_dtype 1) or fp32 (corr_dtype 0, rounded
 *   to fp16 at the convolution input); coords1 [B,2,H,W] fp32 contiguous, updated in place; czrq points at cz of the
 *   [B,288,H,W] fp16 context tensor (cz, cr, cq its channels 0-95, 96-191, 192-287, each plane H*W contiguous, sample i
 *   at czrq + i * czrq_batch_stride elements); mask_out NULL or [B,576,H,W] fp16 NCHW.  The hidden state h lives in the
 *   workspace as NHWC [B,H,W,96] fp16 and is updated in place; `net` non-NULL ([B,96,H,W] fp16 NCHW contiguous) loads it
 *   first (the first iteration), NULL continues from the workspace's h.  workspace: gpsg_update_workspace_bytes(B, H, W)
 *   bytes, 256-byte aligned; after the call it holds, each at a 256-byte-aligned offset in this order, NHWC fp16:
 *   h [96], x [128], cf1 = [relu(convc1), relu(convf1)] [128], cf2 = [cor, flo] [128], z [96], r*h [96],
 *   [relu(flow_head.conv1), relu(mask[0])] [512] (the mask half only when mask_out is set) and delta [2] (channel 1 not
 *   zeroed).  B >= 1, H, W >= 1.  Bit-reproducible; no floating-point atomics.  Enqueues on `stream` and does not
 *   synchronise. */
typedef struct GpsgUpdateWeights {
    const float* convc1_w; const float* convc1_b; const float* convc2_w; const float* convc2_b;
    const float* convf1_w; const float* convf1_b; const float* convf2_w; const float* convf2_b;
    const float* conv_w; const float* conv_b;
    const float* convz_w; const float* convz_b; const float* convr_w; const float* convr_b;
    const float* convq_w; const float* convq_b;
    const float* fh_conv1_w; const float* fh_conv1_b; const float* fh_conv2_w; const float* fh_conv2_b;
    const float* mask0_w; const float* mask0_b; const float* mask2_w; const float* mask2_b;
} GpsgUpdateWeights;
GPSG_API size_t gpsg_update_workspace_bytes(int B, int H, int W);
GPSG_API size_t gpsg_update_packed_bytes(void);
GPSG_API int gpsg_update_pack(int device, void* stream, GpsgUpdateWeights weights, void* packed);
GPSG_API int gpsg_update_step(int device, void* stream, int B, int H, int W, int corr_dtype, const void* corr,
                              float* coords1, const void* net, const void* czrq, int64_t czrq_batch_stride,
                              void* mask_out, const void* packed, void* workspace);

/* ---- fused photometric loss on the rendered image (SURVEY.md 8f-4)-----------------------------------------------
 * replaces  0.8 * l1_loss(img, gt) + 0.2 * (1 - ssim(img, gt))  (train_stage2.py:70-72; lib/loss.py:35-72: 11x11 Gaussian
 * window sigma 1.5, zero padding, C1 = 0.01^2, C2 = 0.03^2, means over all planes*H*W elements) and its autograd.
 * img, gt: [planes, H, W] fp32 (planes = B*C).  out3 (device float[3]) = { w_l1*L1 + w_ssim*(1-SSIM), L1, SSIM }.
 * dmaps (device float[3*planes*H*W], NULL when no gradient is needed) keeps the per-pixel SSIM partials for the backward,
 * which writes dimg = grad_loss * d(out3[0])/d(img); grad_loss is a DEVICE pointer to one float (NULL = 1). */
GPSG_API size_t gpsg_l1_ssim_workspace_bytes(int planes, int H, int W);
GPSG_API int gpsg_l1_ssim_forward(int device, void* stream, int planes, int H, int W, const float* img, const float* gt,
                                  float w_l1, float w_ssim, float* out3, float* dmaps, void* workspace);
GPSG_API int gpsg_l1_ssim_backward(int device, void* stream, int planes, int H, int W, const float* img, const float* gt,
                                   const float* dmaps, float w_l1, float w_ssim, const float* grad_loss, float* dimg);

/* ---- measurement hooks (used by bench.py; off by default) -----------------------------------
 * When enabled, every stage of the forward/backward is bracketed by CUDA events on the launching stream.
 * gpsg_profile_read() synchronises, then returns for stage i: total_ms[i] (summed over the calls since the last
 * reset), calls[i] and the number of kernel launches[i]; it returns the number of stages (names via
 * gpsg_profile_stage_name) and resets the accumulators.  Process-wide (autograd runs backward nodes on its own thread).  on = 2 counts launches only (no events: nothing is
 * inserted into the streams, for timed regions that should only be counted). */
/* fp16 correlation-volume build / backward: 0 = wgmma tensor-core kernels when the shape fits (default), 1 = FFMA kernels.
 * Process-wide switch for comparing the two formulations (tests, bench.py); GPSG_CORR_BUILD=ffma sets the initial value. */
GPSG_API int gpsg_set_corr_build(int mode);
GPSG_API int gpsg_profile_enable(int on);
GPSG_API int gpsg_profile_read(float* total_ms, int32_t* calls, int32_t* launches, int capacity);
GPSG_API const char* gpsg_profile_stage_name(int stage);

#ifdef __cplusplus
}
#endif
#endif /* GPSG_H */
