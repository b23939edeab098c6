/*
 * splatam_b200.h -- C-ABI of the H100-native (sm_90a) differentiable 3D-Gaussian rasterizer.
 *
 * This is the drop-in boundary for the ONE hot path SplaTAM has: the
 * `diff_gaussian_rasterization._C` extension.  Each entry point below names the
 * reference interface it replaces (paths relative to
 * /root/reference/diff-gaussian-rasterization-w-depth.git/, "X/").
 *
 *   reference                                                     this header
 *   ------------------------------------------------------------  -------------------------
 *   rasterize_gaussians          X/rasterize_points.h:18-37       sb_forward_geometry + sb_forward_render
 *     -> Rasterizer::forward     X/cuda_rasterizer/rasterizer.h:35-59
 *   rasterize_gaussians_backward X/rasterize_points.h:39-60       sb_backward
 *     -> Rasterizer::backward    X/cuda_rasterizer/rasterizer.h:61-89
 *   mark_visible                 X/rasterize_points.h:62-65       sb_mark_visible
 *     -> Rasterizer::markVisible X/cuda_rasterizer/rasterizer.h:27-33
 *   resize callbacks std::function<char*(size_t)>                 sb_*_workspace_bytes + caller-owned
 *                                X/rasterize_points.cu:27-33      device workspaces
 *   GaussianRasterizationSettings X/diff_gaussian_rasterization/__init__.py:134-145   sb_settings
 *
 * Conventions
 *   - plain C types only; every pointer marked "dev" is a DEVICE pointer owned by the caller.
 *   - NULL means "not provided" (the reference passes empty tensors whose data_ptr() is null,
 *     X/diff_gaussian_rasterization/__init__.py:173-183).
 *   - every call enqueues work on `stream` (a cudaStream_t passed as void*); only
 *     sb_forward_geometry synchronises that stream (it returns num_rendered to the host, like
 *     X/cuda_rasterizer/rasterizer_impl.cu:282).
 *   - return value: 0 = SB_OK, otherwise an sb_status code; sb_status_string() names it.
 *   - there is NO CPU fallback: without a CUDA device every compute entry returns SB_ERR_CUDA.
 */
#ifndef SPLATAM_B200_H_INCLUDED
#define SPLATAM_B200_H_INCLUDED

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#if defined(__GNUC__)
#define SB_API __attribute__((visibility("default")))
#else
#define SB_API
#endif

#define SB_ABI_VERSION 4
#define SB_TILE 16 /* BLOCK_X == BLOCK_Y == 16, X/cuda_rasterizer/config.h:16-17 (part of the key contract) */
#define SB_CHANNELS 3 /* NUM_CHANNELS, X/cuda_rasterizer/config.h:15 */

typedef enum sb_status {
    SB_OK = 0,
    SB_ERR_BAD_ARG = 1,      /* null/negative/inconsistent argument                     */
    SB_ERR_WORKSPACE = 2,    /* a caller-provided workspace is too small                */
    SB_ERR_CUDA = 3,         /* a CUDA runtime call or kernel launch failed             */
    SB_ERR_UNSUPPORTED = 4,  /* feature of the reference API not built (see DESIGN.md)  */
    SB_ERR_BINNING_TOO_SMALL = 5 /* sb_forward only: stage 1 is complete and *num_rendered is set, but the guessed
                                binning workspace cannot hold it -- finish with sb_forward_render */
} sb_status;

/* Mirror of GaussianRasterizationSettings (X/diff_gaussian_rasterization/__init__.py:134-145).
 * Matrices are the 16 floats of the reference's [1,4,4] tensors, read exactly as the reference
 * kernels read them (element k = flat index k; X/cuda_rasterizer/auxiliary.h:58-77). */
typedef struct sb_settings {
    int32_t image_height;
    int32_t image_width;
    float tanfovx;
    float tanfovy;
    const float* bg;          /* dev [3]  */
    float scale_modifier;
    const float* viewmatrix;  /* dev [16] */
    const float* projmatrix;  /* dev [16] */
    int32_t sh_degree;
    const float* campos;      /* dev [3]  */
    int32_t prefiltered;
} sb_settings;

SB_API int sb_abi_version(void);
SB_API const char* sb_status_string(int status);
/* Text of the last CUDA error seen by this thread's most recent failing call ("" if none). */
SB_API const char* sb_last_cuda_error(void);

/* ---- workspace sizing (replaces required<GeometryState/ImageState/BinningState>,
 *      X/cuda_rasterizer/rasterizer_impl.h:63-72) -------------------------------------- */
SB_API int sb_geometry_workspace_bytes(int P, size_t* bytes);
SB_API int sb_image_workspace_bytes(int width, int height, size_t* bytes);
/* color_sets = 1, or 2 for a render with a second colour set (see sb_forward_render). */
SB_API int sb_binning_workspace_bytes(int num_rendered, int width, int height, int color_sets, size_t* bytes);
SB_API int sb_backward_workspace_bytes(int P, int color_sets, size_t* bytes);

/* ---- forward, stage 1: per-Gaussian projection + depth ordering -----------------------
 * FORWARD::preprocess + InclusiveSum + num_rendered readback
 * (X/cuda_rasterizer/forward.cu:155-256, rasterizer_impl.cu:248-282).
 * means3D [P,3], opacities [P], scales [P,3], rotations [P,4] (or cov3D_precomp [P,6]).
 * Writes radii [P] (int32) and *num_rendered (host).  Synchronises `stream`. */
SB_API int sb_forward_geometry(const sb_settings* s, int P,
                        const float* means3D, const float* opacities,
                        const float* scales, const float* rotations,
                        const float* cov3D_precomp,
                        int32_t* radii,
                        void* geom_ws, size_t geom_ws_bytes,
                        int* num_rendered,
                        void* stream);

/* ---- forward, stage 2: tile duplication + sort + alpha-composite ------------------------
 * duplicateWithKeys + SortPairs + identifyTileRanges + FORWARD::render
 * (X/cuda_rasterizer/rasterizer_impl.cu:284-337, forward.cu:261-393).
 * colors [P,3] (colors_precomp).  out_color [3,H,W], out_depth [1,H,W].
 * Second colour set (SURVEY.md section 8(f) row N1): SplaTAM renders the SAME geometry twice per iteration with
 * different colours_precomp, RGB and [depth, 1, depth^2] (R/scripts/splatam.py:249,253).  colors2 [P,3] /
 * out_color2 [3,H,W] blend both sets in one pass over one projection and one sort; NULL for both is a plain
 * render.  Outputs of the first set are bit-identical to a plain render.  The binning workspace must then be
 * sized with color_sets = 2. */
SB_API int sb_forward_render(const sb_settings* s, int P, int num_rendered,
                      const float* colors, const float* colors2,
                      const void* geom_ws, size_t geom_ws_bytes,
                      void* binning_ws, size_t binning_ws_bytes,
                      void* image_ws, size_t image_ws_bytes,
                      float* out_color, float* out_color2, float* out_depth,
                      void* stream);

/* ---- backward ---------------------------------------------------------------------------
 * BACKWARD::render + BACKWARD::preprocess (X/cuda_rasterizer/backward.cu:399-657).
 * dL_dout_color [3,H,W].  Outputs are fully overwritten (no pre-zeroing needed):
 * dL_dmeans3D [P,3], dL_dmeans2D [P,3], dL_dcolors [P,3], dL_dopacity [P],
 * dL_dscales [P,3], dL_drotations [P,4]; dL_dcov3D [P,6] may be NULL.
 * Second colour set: dL_dout_color2 [3,H,W] and dL_dcolors2 [P,3], both NULL for a plain render.  dL_dmeans2D
 * then carries the FIRST set's share only (SplaTAM reads the means2D gradient of the RGB render,
 * splatam.py:250); every other gradient is the sum over both sets.  bwd_ws is sized with color_sets = 2. */
SB_API int sb_backward(const sb_settings* s, int P, int num_rendered,
                const float* means3D, const float* colors,
                const float* scales, const float* rotations,
                const float* cov3D_precomp,
                const int32_t* radii,
                const void* geom_ws, size_t geom_ws_bytes,
                const void* binning_ws, size_t binning_ws_bytes,
                const void* image_ws, size_t image_ws_bytes,
                void* bwd_ws, size_t bwd_ws_bytes,
                const float* dL_dout_color, const float* dL_dout_color2,
                float* dL_dmeans3D, float* dL_dmeans2D, float* dL_dcolors, float* dL_dcolors2,
                float* dL_dopacity, float* dL_dscales, float* dL_drotations,
                float* dL_dcov3D,
                void* stream);

/* ---- forward in one call ---------------------------------------------------------------------------------
 * sb_forward_geometry + sb_forward_render back to back WITHOUT returning to the caller between them, so
 * the GPU is idle only for the num_rendered read-back itself.  The caller passes a binning workspace sized
 * from a guess (e.g. the previous call's num_rendered plus slack); if it is too small the call returns
 * SB_ERR_BINNING_TOO_SMALL with *num_rendered set and stage 1 complete -- the caller then allocates
 * sb_binning_workspace_bytes(*num_rendered, ...) and finishes with sb_forward_render. */
SB_API int sb_forward(const sb_settings* s, int P, const float* means3D, const float* opacities, const float* scales,
               const float* rotations, const float* cov3D_precomp, const float* colors, const float* colors2,
               int32_t* radii, void* geom_ws, size_t geom_ws_bytes, void* binning_ws, size_t binning_ws_bytes,
               void* image_ws, size_t image_ws_bytes, float* out_color, float* out_color2, float* out_depth,
               int* num_rendered, void* stream);

/* ---- sync-free forward (CUDA-graph capturable) -------------------------------------------------------------
 * Same work as sb_forward but num_rendered never leaves the device: the caller fixes a CAPACITY (tile
 * instances) for the binning workspace (sb_binning_workspace_bytes(capacity, ...)); the instance count is read
 * on the device by the sort and the record gather, so only the live instances are processed.  No memcpy to the
 * host, no synchronisation, no allocation:
 * the call (and sb_backward with num_rendered := capacity) can be captured into a CUDA graph.
 * If the scene needs more than `capacity` instances the overflow flag (geometry workspace, int32 word 2) is set and
 * the images are written as NaN, so a truncated render cannot pass for a valid one;
 * sb_read_counts (which synchronises) returns the true count and the flag so the caller can grow and redo. */
SB_API int sb_forward_async(const sb_settings* s, int P, const float* means3D, const float* opacities,
                     const float* scales, const float* rotations, const float* cov3D_precomp, const float* colors,
                     const float* colors2, int32_t* radii, void* geom_ws, size_t geom_ws_bytes, void* binning_ws,
                     size_t binning_ws_bytes, int capacity, void* image_ws, size_t image_ws_bytes, float* out_color,
                     float* out_color2, float* out_depth, void* stream);
SB_API int sb_read_counts(const void* geom_ws, size_t geom_ws_bytes, int P, int* num_rendered, int* overflow,
                          void* stream);

/* ---- blend statistics of a finished render (splatam_b200/contrib.py) -------------------------------------------
 * Replays the per-pixel walk of the forward that filled the three workspaces (sb_forward / sb_forward_render, or
 * sb_forward_async with num_rendered := capacity and sync_free = 1), with the forward's own culling, thresholds,
 * early-outs and float operation order, and ADDS into the caller's per-Gaussian arrays [P] (kept across calls, so
 * one set gathers many views):
 *   blended[g]          pixels where g was composited: alpha >= 1/255 and test_T = T (1 - alpha) >= 1e-4
 *   ended[g]            pixels whose walk g stopped: alpha >= 1/255 and test_T < 1e-4 (g blends nothing there)
 *   max_weight_bits[g]  atomicMax of the float32 bits of alpha * T over the pixels g blended (weights are >= 0)
 * Writes no image and leaves the workspaces as they are.  A plain and a two-set render of the same geometry give
 * the same statistics (the binning workspace of either is accepted).  sync_free = 1: an overflowed render (flag word 2
 * of the geometry workspace set) adds nothing.  Integer and max atomics only: the result is deterministic.  The
 * caller keeps the counters from wrapping (at most 2^32 - 1 accumulated pixels).  No host synchronisation.
 * SB_ERR_BAD_ARG, before any launch, for bad settings, P < 0, num_rendered < 0, a null workspace or array the call
 * reads; SB_ERR_WORKSPACE for a workspace smaller than its size query gives. */
SB_API int sb_blend_stats(const sb_settings* s, int P, int num_rendered, int sync_free, const void* geom_ws,
                          size_t geom_ws_bytes, const void* binning_ws, size_t binning_ws_bytes, const void* image_ws,
                          size_t image_ws_bytes, uint32_t* blended, uint32_t* ended, uint32_t* max_weight_bits,
                          void* stream);

/* ---- spherical-harmonics colour branch (shs / sh_degree, X/cuda_rasterizer/forward.cu:20-71,
 *      backward.cu:20-139).  sb_sh_forward turns shs [P,max_coeffs,3] into the rgb [P,3] the render consumes
 *      (plus one clamp-flag byte per Gaussian); sb_sh_backward turns dL/drgb into dL/dshs and ADDS the
 *      view-direction term to dL_dmeans3D; Gaussians with radii[i] <= 0 (when `radii` is not NULL) get zero gradients,
 *      as the reference leaves them.  Unused by SplaTAM. */
SB_API int sb_sh_forward(int P, int sh_degree, int max_coeffs, const float* means3D, const float* campos,
                         const float* shs, float* rgb, uint8_t* clamped, void* stream);
SB_API int sb_sh_backward(int P, int sh_degree, int max_coeffs, const float* means3D, const float* campos,
                          const float* shs, const uint8_t* clamped, const float* dL_drgb, const int32_t* radii,
                          float* dL_dshs, float* dL_dmeans3D_accumulate, void* stream);

/* ---- markVisible (X/cuda_rasterizer/rasterizer_impl.cu:54-66,141-153) ------------------- */
SB_API int sb_mark_visible(int P, const float* means3D, const float* viewmatrix,
                    const float* projmatrix, uint8_t* present, void* stream);

/* ---- inspection (parity tests only): the intermediates the reference keeps in its
 *      geometry/binning/image byte buffers (X/cuda_rasterizer/rasterizer_impl.cu:155-194). ---
 * Any output pointer may be NULL.  All outputs are device pointers.
 *   depths [P] f32, means2D [P,2] f32, conic_opacity [P,4] f32, tiles_touched [P] u32 */
SB_API int sb_export_geometry(int P, const void* geom_ws, size_t geom_ws_bytes,
                       float* depths, float* means2D, float* conic_opacity,
                       uint32_t* tiles_touched, void* stream);
/*   keys [R] u64 = (tile<<32)|depth_bits, point_list [R] u32, both in sorted order;
 *   ranges [tiles,2] u32, final_T [H*W] f32, n_contrib [H*W] u32 */
SB_API int sb_export_binning(const sb_settings* s, int P, int num_rendered,
                      const void* geom_ws, size_t geom_ws_bytes,
                      const void* binning_ws, size_t binning_ws_bytes,
                      const void* image_ws, size_t image_ws_bytes,
                      uint64_t* keys, uint32_t* point_list, uint32_t* ranges,
                      float* final_T, uint32_t* n_contrib, void* stream);
/*   cover [R] u8: per sorted tile instance, bit w set iff the Gaussian can blend a pixel of the 8x4 rectangle
 *   (16 tx + 8 (w & 1), 16 ty + 4 (w >> 1)) of its tile (tx, ty) -- the only pairs the blend kernels evaluate */
SB_API int sb_export_cover(const sb_settings* s, int num_rendered, const void* binning_ws, size_t binning_ws_bytes,
                           uint8_t* cover, void* stream);
/* ---- the rasterizer's radix sort on its own (testing; csrc/radix_sort.cu: the depth sort, the tile sort and the
 *      mesh-evaluation grid all run it) ---------------------------------------------------------------------------
 * sb_radix_sort_pairs: stable ascending sort of the n pairs (keys_in[i], vals_in ? vals_in[i] : i) by the key bits
 *   [begin_bit, end_bit) (8-bit digits, one pass per digit), written to keys_out and vals_out [capacity] (device u32;
 *   the full keys, not just their sorted bits).  n = capacity, or clamp(*n_dev, 0, capacity) with n_dev (device int32)
 *   read on the device: the call never synchronises and can be captured in a CUDA graph.  keys_in and vals_in are not
 *   modified, and nothing is written at or past index n of the outputs.  temp: sb_radix_sort_temp_bytes(capacity,
 *   end_bit - begin_bit) device bytes, any content; that size never decreases as the capacity grows.
 * SB_ERR_BAD_ARG, before any launch, for capacity < 0 or >= 2^30, begin_bit < 0, end_bit > 32 and begin_bit >=
 * end_bit; then SB_OK with nothing launched for capacity 0; then SB_ERR_BAD_ARG for null pointers (NULL vals_in and
 * n_dev excepted) and an output that is an input or the other output (a pass may write an output while it reads the
 * inputs); SB_ERR_WORKSPACE for a short temp. */
SB_API int sb_radix_sort_temp_bytes(int capacity, int bits, size_t* bytes);
SB_API int sb_radix_sort_pairs(const uint32_t* keys_in, const uint32_t* vals_in, uint32_t* keys_out, uint32_t* vals_out,
                               int capacity, const int32_t* n_dev, int begin_bit, int end_bit, void* temp,
                               size_t temp_bytes, void* stream);

/* ---- per-iteration training ops around the rasterizer (SURVEY.md section 8(f) row N3) -----------------
 * sb_adam_step: torch.optim.Adam (no amsgrad / weight decay) over ONE flat parameter buffer whose segments
 * [seg_end[k-1], seg_end[k]) have learning rates seg_lr[k] (host arrays, <= 16 segments; hyper-parameters are doubles, rounded to float
 * once inside, as torch rounds its Python-float scalars); replaces the
 * multi-group optimizer.step() of R/scripts/splatam.py:160-166,869.  `step` counts from 1.
 * sb_image_loss_*: w_l1*mean|x-y| + w_ssim*(1-mean SSIM(x,y)) over [C,H,W] images with the reference's
 * 11x11 sigma-1.5 Gaussian window and zero padding (R/utils/slam_external.py:54-97, R/scripts/splatam.py:290).
 * forward writes sums[0] = sum of the SSIM map, sums[1] = sum|x-y| (device doubles) and 3*C*H*W floats of
 * partial derivatives into `work`; backward turns them into d loss / d x given the upstream scalar grad. */
SB_API int sb_adam_step(float* params, const float* grads, float* exp_avg, float* exp_avg_sq, size_t n,
                        const uint32_t* seg_end, const double* seg_lr, int num_segments, int step,
                        double beta1, double beta2, double eps, void* stream);
/* Guarded step for the sync-free (CUDA-graph) mapping loop: the step count and the bias-correction scalars live in a
 * device-side clock (`clock_dev`: sb_adam_clock_bytes() bytes, zero-initialised = step 0; first int = steps applied,
 * second int = steps skipped), and when `skip_if_nonzero` points at a non-zero device float the whole update is a
 * no-op -- used with the rasterizer's instance-capacity overflow flag, whose gradients are incomplete. */
SB_API size_t sb_adam_clock_bytes(void);
SB_API int sb_adam_step_guarded(float* params, const float* grads, float* exp_avg, float* exp_avg_sq, size_t n,
                                const uint32_t* seg_end, const double* seg_lr, int num_segments, void* clock_dev,
                                const float* skip_if_nonzero, double beta1, double beta2, double eps, void* stream);
SB_API size_t sb_image_loss_workspace_floats(int C, int H, int W);
SB_API int sb_image_loss_forward(const float* x, const float* y, int C, int H, int W, float* work,
                                 double* sums, void* stream);
SB_API int sb_image_loss_backward(const float* x, const float* y, int C, int H, int W, const float* work,
                                  const float* grad_out, float w_ssim, float w_l1, float* grad_x, void* stream);

/* ---- fused parameter glue (SURVEY.md section 8(f) row N2) ----------------------------------------------
 * sb_prepare_forward: raw SplaTAM parameters + frame pose -> the operator's inputs, in one kernel
 * (replaces transform_to_frame + transformed_params2rendervar + transformed_params2depthplussilhouette,
 * R/utils/slam_helpers.py:124-139,196-304).  scale_dim = 1 (isotropic log_scales [P,1]) or 3.
 * rel_w2c, w2c0: row-major 4x4; cam_rot: the normalised camera quaternion (w,x,y,z).
 * sb_prepare_backward: gradients of the six outputs (any may be NULL = zero) -> gradients of the raw
 * parameters; if want_pose, g_pose16 (16 device doubles, zeroed here) receives d/d rel_w2c[0:3,0:4] (12) then
 * d/d cam_rot (4), accumulated in double. */
SB_API int sb_prepare_forward(int P, int scale_dim, const float* means3D, const float* unnorm_rotations,
                              const float* logit_opacities, const float* log_scales, const float* rel_w2c,
                              const float* cam_rot, const float* w2c0, float* means_cam, float* rotations,
                              float* opacities, float* scales3, float* depth_sil_colors, void* stream);
SB_API int sb_prepare_backward(int P, int scale_dim, int want_pose, const float* means3D,
                               const float* unnorm_rotations, const float* rel_w2c, const float* cam_rot,
                               const float* w2c0, const float* means_cam, const float* opacities,
                               const float* scales3, const float* g_means_cam, const float* g_rotations,
                               const float* g_opacities, const float* g_scales3, const float* g_depth_sil_colors,
                               float* g_means3D, float* g_unnorm_rotations, float* g_logit_opacities,
                               float* g_log_scales, double* g_pose16, void* stream);

/* Masked L1 terms of SplaTAM's get_loss (R/scripts/splatam.py:254-288): mask = (gt_depth > 0) & !isnan(depth)
 * & !isnan(depth_sq - depth^2) [& silhouette > sil_thres when use_sil]; depth_sil is the [3,H,W] depth /
 * silhouette / depth^2 render.  forward: sums[0] = sum|gt_depth - depth|*mask, sums[1] = sum mask,
 * sums[2] = sum over channels |gt_im - im|*mask (im may be NULL).  backward: gradients w.r.t. depth_sil (only
 * channel 0 is non-zero) and im, for loss_depth = sums[0] (/ sums[1] if depth_mean) and loss_im = sums[2]. */
SB_API int sb_masked_l1_forward(const float* depth_sil, const float* gt_depth, const float* im, const float* gt_im,
                                int H, int W, float sil_thres, int use_sil, double* sums, void* stream);
SB_API int sb_masked_l1_backward(const float* depth_sil, const float* gt_depth, const float* im, const float* gt_im,
                                 int H, int W, float sil_thres, int use_sil, int depth_mean, const double* sums,
                                 const float* g_depth, const float* g_im, float* grad_depth_sil, float* grad_im,
                                 void* stream);
/* The same losses over the pixels whose `keep` byte (uint8 [H,W], device, non-NULL) is non-zero, through the same
 * device code: with every keep byte set they give the bits of the calls above.  sb_masked_l1_keep_*: mask &= keep.
 * sb_image_loss_keep_forward: sums[0] = sum over kept pixels and channels of the SSIM map, sums[1] = that of |x-y|,
 * sums[2] = the kept pixel count (3 device doubles, zeroed here); the loss is w_l1 sums[1] / (C sums[2]) +
 * w_ssim (1 - sums[0] / (C sums[2])).  sb_image_loss_keep_backward takes the forward's `sums`. */
SB_API int sb_masked_l1_keep_forward(const uint8_t* keep, const float* depth_sil, const float* gt_depth,
                                     const float* im, const float* gt_im, int H, int W, float sil_thres, int use_sil,
                                     double* sums, void* stream);
SB_API int sb_masked_l1_keep_backward(const uint8_t* keep, const float* depth_sil, const float* gt_depth,
                                      const float* im, const float* gt_im, int H, int W, float sil_thres, int use_sil,
                                      int depth_mean, const double* sums, const float* g_depth, const float* g_im,
                                      float* grad_depth_sil, float* grad_im, void* stream);
SB_API int sb_image_loss_keep_forward(const uint8_t* keep, const float* x, const float* y, int C, int H, int W,
                                      float* work, double* sums, void* stream);
SB_API int sb_image_loss_keep_backward(const uint8_t* keep, const float* x, const float* y, int C, int H, int W,
                                       const float* work, const double* sums, const float* grad_out, float w_ssim,
                                       float w_l1, float* grad_x, void* stream);

/* ---- map maintenance: stream compaction (SURVEY.md section 8(f) row N3) ---------------------------------
 * sb_prune_mask: keep[i] = !(sigmoid(logit_opacities[i]) < opacity_threshold || max_k exp(log_scales[i,k]) >
 * big_threshold); big_threshold <= 0 disables the size test (prune_gaussians, R/utils/slam_external.py:170-190).
 * sb_compact_plan: exclusive scan of a 0/1 byte mask -> dst_index[n] (destination row of every kept element) and
 * the number kept (*count_host; the call synchronises the stream).  temp: sb_compact_plan_bytes(n) device bytes.
 * sb_compact_flat: gathers the kept rows of a packed buffer [seg0: widths[0]*P | seg1: widths[1]*P | ...] into the
 * same packing with P_new rows (remove_points, R/utils/slam_external.py:144-167: parameters and both Adam moments).
 * sb_depth_error / sb_new_gaussian_mask: add_new_gaussians' non-presence test on the [3,H,W] depth/silhouette
 * render (R/scripts/splatam.py:385-405): err = |gt - depth| * (gt > 0); mask = ((sil < sil_thres) | ((depth > gt) &
 * (err > depth_err_thres))) & (gt > 0), depth_err_thres = 50 * median(err) supplied by the caller.
 * sb_backproject: pixels (all, or those with mask != 0 written to row dst_index[pixel]) -> new Gaussian rows:
 * means3D = c2w * ((x-cx)/fx*z, (y-cy)/fy*z, z, 1), rgb = colour of the pixel, log_scales = log(sqrt((z /
 * ((fx+fy)/2))^2)) repeated scale_dim times, optional mean_sq_dist (get_pointcloud, R/scripts/splatam.py:67-118;
 * initialize_new_params, :348-375).  c2w_host: 12+ floats, row-major 3x4 (or 4x4), HOST memory.
 * sb_densify_accumulate: the densification statistic (accumulate_mean2d_gradient, R/utils/slam_external.py:200-204):
 * for every i < P with seen[i] != 0, accum[i] += sqrt(g0^2 + g1^2) and denom[i] += 1, where g = means2D_grad + i *
 * grad_stride (>= 2 floats per row); one pass, no host synchronisation, bit-equal to the torch statement. */
SB_API int sb_prune_mask(int P, const float* logit_opacities, const float* log_scales, int scale_dim,
                         float opacity_threshold, float big_threshold, uint8_t* keep, void* stream);
SB_API int sb_compact_plan_bytes(int n, size_t* bytes);
SB_API int sb_compact_plan(int n, const uint8_t* keep, uint32_t* dst_index, void* temp, size_t temp_bytes,
                           int* count_host, void* stream);
SB_API int sb_compact_flat(int P, int P_new, const uint8_t* keep, const uint32_t* dst_index, int num_segments,
                           const int* widths, const float* src, float* dst, void* stream);
SB_API int sb_densify_accumulate(int P, const float* means2D_grad, int grad_stride, const uint8_t* seen, float* accum,
                                 float* denom, void* stream);
SB_API int sb_depth_error(int H, int W, const float* depth_sil, const float* gt_depth, float* err, void* stream);
SB_API int sb_new_gaussian_mask(int H, int W, const float* depth_sil, const float* gt_depth, float sil_thres,
                                float depth_err_thres, uint8_t* mask, void* stream);
SB_API int sb_backproject(int H, int W, const float* color, const float* depth, float fx, float fy, float cx, float cy,
                          const float* c2w_host, const uint8_t* mask, const uint32_t* dst_index, int scale_dim,
                          float* means3D, float* rgb, float* log_scales, float* mean_sq_dist, void* stream);

/* ---- final evaluation metrics (SURVEY.md section 8(f) row N4; R/utils/eval_helpers.py:408-623) -----------------
 * Forward only, deterministic (per-block partials reduced in a fixed order), no host synchronisation.
 * sb_frame_metrics: im, gt_im [3,H,W], depth_sil [3,H,W] (depth, silhouette, depth^2), gt_depth [1,H,W].
 * valid = gt_depth > 0, presence = silhouette > sil_thres, mask = presence*valid if use_presence else valid
 * (use_presence = mapping_iters == 0 && !add_new_gaussians in the reference).  Writes weighted_im = im*mask and
 * weighted_gt = gt_im*mask [3,H,W] and metrics[5] (device doubles) = {PSNR: mean over channels of the per-channel
 * PSNR, each MSE over all H*W pixels; "depth RMSE": sum(sqrt(e^2)*valid)/sum(valid), i.e. a masked mean absolute
 * error as the reference defines it; depth L1: sum(|e|*valid)/sum(valid); sum(valid); sum(mask)} with
 * e = (depth*valid - gt_depth) [* presence when use_presence].  Rendered values are not clamped.
 * sb_ms_ssim: pytorch_msssim.ms_ssim(x, y, data_range, 11-tap sigma-1.5 window, 5 levels) of [N,C,H,W] contiguous
 * float images, computed in double; per_channel [N*C] and/or mean (device doubles, either may be NULL).
 * min(H, W) must exceed 160.  Workspaces: the *_workspace_bytes queries (device memory, any content). */
SB_API int sb_frame_metrics_workspace_bytes(int H, int W, size_t* bytes);
SB_API int sb_frame_metrics(const float* im, const float* depth_sil, const float* gt_im, const float* gt_depth, int H,
                            int W, float sil_thres, int use_presence, float* weighted_im, float* weighted_gt,
                            void* workspace, size_t workspace_bytes, double* metrics, void* stream);
SB_API int sb_ms_ssim_workspace_bytes(int N, int C, int H, int W, size_t* bytes);
SB_API int sb_ms_ssim(const float* x, const float* y, int N, int C, int H, int W, double data_range, void* workspace,
                      size_t workspace_bytes, double* per_channel, double* mean, void* stream);

/* ---- LPIPS (AlexNet, v0.1) of the final evaluation (R/utils/eval_helpers.py:484-485, 730-731) ----------------------
 * torchmetrics' LearnedPerceptualImagePatchSimilarity(net_type='alex', normalize=True) applied to clamp(x, 0, 1) and
 * clamp(y, 0, 1), forward only, deterministic FP32 (no atomics, no split-K; per-block partials reduced in a fixed
 * order), no host synchronisation.  x, y: [N,3,H,W] contiguous float; per_image [N] and/or mean (device doubles, either
 * may be NULL, not both).  Per pair: inputs 2x - 1, then (x - shift) / scale with shift = (-0.030, -0.088, -0.188),
 * scale = (0.458, 0.448, 0.450); torchvision AlexNet features f1..f5 = relu(conv1..conv5) (3x3 stride-2 max-pools
 * after f1 and f2); per layer and pixel d = sum_c lin_c (fx / sqrt(1e-8 + |fx|^2) - fy / sqrt(1e-8 + |fy|^2))^2;
 * LPIPS = sum over the five layers of the mean of d over the layer's pixels.  H and W must be >= 31.
 * weights: sb_lpips_weights_floats() device floats, packed as
 *   for l = 0..4: conv_l weight as [K_l][Cout_l], k = (ci * ks + ky) * ks + kx (the transpose of torchvision's
 *                 features.{0,3,6,8,10}.weight viewed as [Cout_l, K_l]), then conv_l bias [Cout_l];
 *   then lin_0 .. lin_4 [Cout_l] (lpips' lin{l}.model.1.weight),
 * with (Cin, Cout, ks) = (3, 64, 11), (64, 192, 5), (192, 384, 3), (384, 256, 3), (256, 256, 3).
 * workspace: sb_lpips_workspace_bytes(N, H, W) device bytes (any content; ~39 MB per image at 1200x680, and
 * the 2N images of x and y all run). */
SB_API int sb_lpips_weights_floats(size_t* n);
SB_API int sb_lpips_workspace_bytes(int N, int H, int W, size_t* bytes);
SB_API int sb_lpips(const float* x, const float* y, int N, int H, int W, const float* weights, void* workspace,
                    size_t workspace_bytes, double* per_image, double* mean, void* stream);

/* ---- saved evaluation frames (R/utils/eval_helpers.py:509-528, 755-774, save_frames=True) ---------------------------
 * One launch per frame, no host synchronisation.  im, gt_im [3,H,W], depth_sil [3,H,W] (channel 0 is read),
 * gt_depth [1,H,W], contiguous float; lut: 256 x RGB uint8 (device), the colormap; out: uint8 [4,H,W,3] (device) =
 * {rendered RGB, rendered depth, ground-truth RGB, ground-truth depth}, HWC RGB.
 *   RGB:   u8 = round_half_even(clamp(x, 0, 1) * 255f), NaN -> 0 (cv2.imwrite of a float32 image)
 *   depth: lut[trunc(clip(d / 6f, 0, 1) * 255f)], an IEEE float32 division, NaN -> index 0
 * SB_ERR_BAD_ARG for null pointers and non-positive sizes. */
SB_API int sb_eval_frames_u8(const float* im, const float* depth_sil, const float* gt_im, const float* gt_depth, int H,
                             int W, const uint8_t* lut, uint8_t* out, void* stream);

/* ---- headless viewer (R/viz_scripts/final_recon.py, online_recon.py; splatam_b200/viewer.py) ----------------------
 * Frames are uint8 HWC RGB [H, W, 3] at H = h * s, W = w * s (s = view_scale >= 1), with a float32 depth buffer
 * zbuf [H, W] (camera z, +inf where nothing is drawn).  Background: white at infinite depth.  Colours:
 * round_half_even(clamp(x, 0, 1) * 255f), NaN -> 0.  No host synchronisation; every pass is enqueued on `stream`.
 * w2c: row-major float32 4x4 on the device (rows 0..2 are read).  fx, fy, cx, cy: the intrinsics at output size.
 *
 * sb_viewer_compose: color [3,h,w], depth [h,w], sil [h,w] (contiguous float) -> out, zbuf.  Output pixel (X, Y)
 *   shows render pixel (X / s, Y / s); a pixel with depth <= 0 or NaN is background.  mode 0: the colour; mode 1:
 *   lut[i] (256 x RGB uint8, matplotlib's jet), i = trunc(float32(d / vmax) * 256f) with 256 -> 255 and i = 0 when
 *   vmax == 0, vmax = max of d over pixels with 0 < d < 15 (device, `vmax_bits`: one scratch uint), d >= 15 white;
 *   mode 2: round_half_even(clamp(1 - sil, 0, 1) * 255f) in all three channels.  Only the inputs the mode reads
 *   need be non-NULL.
 * sb_viewer_points: P centres means [P,3] with colors [P,3]; with `timestep` [P] (may be NULL) only those with
 *   timestep <= t_max.  Camera z = ((r0 x + r1 y) + r2 z) + t per row, float32; points with !(near < z < far) or a
 *   non-finite u = fx x / z + cx, v = fy y / z + cy are skipped.  Each covers the s x s square whose top-left pixel is
 *   (floor(u + 0.5), floor(v + 0.5)); per pixel the key (float bits of z) << 32 | index is kept by atomicMin (nearest
 *   first, ties to the lower index).  keys: [H*W] uint64 scratch.  Writes every pixel of out and zbuf.
 * sb_viewer_lines: S segments [S,6] (two world points each) with colors [S,3] uint8, drawn over out.  Endpoints are
 *   clipped to z >= near (segments wholly at z <= near are dropped) and projected; a DDA along the major screen axis
 *   visits each pixel centre c + 0.5 within the span, a = (c + 0.5 - p0) / (p1 - p0), minor = floor(q0 + a dq), depth
 *   1 / ((1 - a) / z0 + a / z1).  A pixel is drawn when that depth is below zbuf; overlaps resolve by the (depth bits,
 *   segment index) atomicMin in keys ([H*W] uint64 scratch).  zbuf is read, not written.
 * SB_ERR_BAD_ARG for null pointers the call reads, non-positive sizes, view_scale < 1, near < 0 (points), near <= 0
 * (lines) or far <= near. */
SB_API int sb_viewer_compose(const float* color, const float* depth, const float* sil, int h, int w, int mode,
                             int view_scale, const uint8_t* lut, unsigned int* vmax_bits, uint8_t* out, float* zbuf,
                             void* stream);
SB_API int sb_viewer_points(int P, const float* means, const float* colors, const float* timestep, float t_max,
                            const float* w2c, float fx, float fy, float cx, float cy, int width, int height,
                            int view_scale, float near, float far, unsigned long long* keys, uint8_t* out, float* zbuf,
                            void* stream);
SB_API int sb_viewer_lines(int S, const float* segments, const uint8_t* colors, const float* w2c, float fx, float fy,
                           float cx, float cy, int width, int height, float near, const float* zbuf,
                           unsigned long long* keys, uint8_t* out, void* stream);

/* ---- frame ingest (the dataset readers, splatam_b200/datasets.py; R/datasets/gradslam_datasets/basedataset.py) ---
 * One launch: rgb uint8 [color_height, color_width, 3] (HWC) and depth uint16 [depth_height, depth_width] (device)
 * -> color_out float32 [3, height, width] = float32(bilinear_f64(rgb)) / 255 and depth_out float32 [1, height, width]
 * = float32(nearest(depth) / png_depth_scale), division in double: cv2.resize INTER_LINEAR / INTER_NEAREST on float64
 * as the reference's loader calls it, including cv2's exact-2x box average and the plain copy at equal size.  The two
 * source sizes may differ.  SB_ERR_BAD_ARG for a non-positive size or depth scale and for null pointers. */
SB_API int sb_ingest_rgbd(const uint8_t* rgb, int color_height, int color_width, const uint16_t* depth,
                          int depth_height, int depth_width, int height, int width, double png_depth_scale,
                          float* color_out, float* depth_out, void* stream);

/* ---- live capture packets (splatam_b200/capture.py; R/scripts/iphone_demo.py, nerfcapture2dataset.py) -----------
 * sb_ingest_capture: one packet's rgb uint8 [color_height, color_width, 3] and float32 depth in metres
 * [depth_height, depth_width] (device) -> color_out float32 [3, height, width] = cv2.resize(uint8, INTER_LINEAR) / 255
 * (cv2's fixed-point uint8 path; its 2x2 INTER_AREA at an exact 2x downscale; a copy at equal size) and depth_out
 * float32 [1, height, width] = cv2.resize(float32, INTER_NEAREST), every value passed through bit for bit.
 * sb_capture_depth_u16: out uint16 [height, width] = cv2.resize(uint16(depth * 65535 / depth_scale), INTER_NEAREST),
 * float32 arithmetic, the cast as numpy's on x86-64 (truncation to int32, low 16 bits; NaN, +-inf and values past
 * int32 give 0).  Both return SB_ERR_BAD_ARG, before any launch, for null pointers, non-positive sizes, sizes whose
 * element count passes INT_MAX, and (sb_capture_depth_u16) a depth scale that is not finite and positive. */
SB_API int sb_ingest_capture(const uint8_t* rgb, int color_height, int color_width, const float* depth,
                             int depth_height, int depth_width, int height, int width, float* color_out,
                             float* depth_out, void* stream);
SB_API int sb_capture_depth_u16(const float* depth, int depth_height, int depth_width, float depth_scale, int height,
                                int width, uint16_t* out, void* stream);

/* ---- mesh extraction: TSDF fusion and marching cubes (splatam_b200/mesh.py, csrc/mesh.cu) ------------------------
 * A volume of nz x ny x nx samples (x fastest) at p = origin + voxel * (i, j, k) holds tsdf, weight [nz,ny,nx] and
 * color [nz,ny,nx,3], float32 on the device; a fresh volume is T = 1, W = 0, C = 0.  Float32, each operation rounded
 * as written.  No host synchronisation except where the caller reads sb_mc_count's totals.
 * sb_tsdf_integrate: fuses B frames in order -- depth [B,H,W] (0 = no measurement), rgb [B,3,H,W], w2c [B,4,4]
 *   row-major (rows 0..2 read), one pinhole camera fx, fy, cx, cy -- into the volume; B frames give exactly what B
 *   single-frame calls give.  Per voxel and frame: (x, y, z) = ((r0 px + r1 py) + r2 pz) + t; z > 0; pixel
 *   (floor(((fx x) / z) + cx + 0.5), floor(((fy y) / z) + cy + 0.5)) inside the image; d = depth there, 0 < d <=
 *   depth_max (+inf: no limit); sdf = d - z >= -trunc; f = min(1, sdf / trunc); W' = W + 1, T' = (T W + f) / W',
 *   C' = (C W + rgb) / W'.
 * sb_mc_count / sb_mc_emit: the indexed mesh of the volume.  A cell is live iff its 8 samples have W >= min_weight,
 *   a sample is inside iff T < 0.  One vertex per crossed grid edge (id 3 * sample index + axis) that a live cell
 *   touches, at p_a + t * voxel along the axis, t = T_a / (T_a - T_b), colour C_a + t * (C_b - C_a), in ascending
 *   edge id; faces int32 [F,3] in ascending cell index, then the order of the generated table (csrc/mc_table.h),
 *   facing increasing T.  sb_mc_count writes totals (device int[2]) = {V, F}, -1 for a count past INT_MAX / 3;
 *   sb_mc_emit then fills vertices [V,3], colors [V,3] and faces [F,3] from the same workspace
 *   (sb_mc_workspace_bytes) and the same tsdf / color.
 * SB_ERR_BAD_ARG, before any launch, for null pointers the call reads, a non-positive size, a grid of 2^31 or more
 * samples (marching cubes: 2^32 / 5 or more, so the packed
 * per-sample counts cannot wrap in the scan), a non-finite origin, voxel, truncation, camera or min_weight, a
 * non-positive voxel, truncation or depth_max; SB_ERR_WORKSPACE for a short workspace. */
SB_API int sb_tsdf_integrate(int nx, int ny, int nz, float ox, float oy, float oz, float voxel, float trunc, int B,
                             int height, int width, const float* depth, const float* rgb, const float* w2c, float fx,
                             float fy, float cx, float cy, float depth_max, float* tsdf, float* weight, float* color,
                             void* stream);
SB_API int sb_mc_workspace_bytes(int nx, int ny, int nz, size_t* bytes);
SB_API int sb_mc_count(int nx, int ny, int nz, const float* tsdf, const float* weight, float min_weight,
                       void* workspace, size_t workspace_bytes, int* totals, void* stream);
SB_API int sb_mc_emit(int nx, int ny, int nz, float ox, float oy, float oz, float voxel, const float* tsdf,
                      const float* color, void* workspace, size_t workspace_bytes, float* vertices, float* colors,
                      int* faces, void* stream);

/* ---- navigation maps: occupancy labels, an exact Euclidean signed distance field and distance queries
 * (splatam_b200/navmap.py, csrc/navmap.cu; oracle/navmap_numpy.py restates every rule) ---------------------------
 * The grid is the TSDF volume's: nz x ny x nx samples (x fastest), sample (i, j, k) at origin + voxel * (i, j, k).
 * Every dimension is at most 8192 and the sample count below 2^31, so every finite squared distance fits in int32 and
 * every envelope comparison in int64.  Float32 operations are rounded as written.  No host synchronisation.
 * sb_nav_labels: labels uint8 [nz,ny,nx] from tsdf T and weight W: 0 (unknown) if W < min_weight, else 2 (occupied)
 *   if T * trunc <= occ_dist, else 1 (free).
 * sb_esdf: the obstacle set O is the occupied samples, and the unknown ones too when unknown_is_obstacle is 1.
 *   sd2 int32 [nz,ny,nx] in lattice units: a sample s outside O gets +min over o in O of |s - o|^2, a sample in O
 *   gets -min over f outside O of |s - f|^2; INT32_MAX everywhere if O is empty, -INT32_MAX everywhere if O is every
 *   sample.  esdf float32 [nz,ny,nx] in metres: sign(sd2) * (voxel * sqrt((float)|sd2|)), the sentinels +-inf.  The
 *   transform is exact (integer lower envelopes of parabolas along x, y, then z; workspace sb_esdf_workspace_bytes).
 * sb_esdf_query: dist [N] and grad [N,3] of the points [N,3] in the esdf.  Per axis u = (p - o) / voxel; a point is
 *   inside iff every u is finite and 0 <= u <= n - 1, and gets NaN distance and gradient otherwise.  i = min(floor(u),
 *   n - 2), t = u - i.  With c_zyx the corner esdf[k + z][j + y][i + x] and lerp(a, b, t) = a + t * (b - a):
 *     e_zy = lerp(c_zy0, c_zy1, tx);  f_z = lerp(e_z0, e_z1, ty);  dist = lerp(f_0, f_1, tz);
 *     grad_x = lerp(lerp(c_001 - c_000, c_011 - c_010, ty), lerp(c_101 - c_100, c_111 - c_110, ty), tz) / voxel;
 *     grad_y = lerp(e_01 - e_00, e_11 - e_10, tz) / voxel;  grad_z = (f_1 - f_0) / voxel
 *   the exact derivative of the interpolant.  If a corner is infinite, dist is the first infinite corner in the
 *   order c_000, c_001, c_010, ..., c_111 (x fastest) and grad is 0.
 * SB_ERR_BAD_ARG, before any launch, for null pointers the call reads, a dimension outside [1, 8192] (the query:
 * [2, 8192]), 2^31 or more samples, a non-finite origin, voxel, trunc, min_weight or occ_dist, a non-positive voxel or
 * trunc, unknown_is_obstacle outside {0, 1} and N < 0; SB_ERR_WORKSPACE for a short workspace. */
SB_API int sb_nav_labels(int nx, int ny, int nz, const float* tsdf, const float* weight, float trunc, float min_weight,
                         float occ_dist, uint8_t* labels, void* stream);
SB_API int sb_esdf_workspace_bytes(int nx, int ny, int nz, size_t* bytes);
SB_API int sb_esdf(int nx, int ny, int nz, const uint8_t* labels, float voxel, int unknown_is_obstacle,
                   void* workspace, size_t workspace_bytes, int* sd2, float* esdf, void* stream);
SB_API int sb_esdf_query(int nx, int ny, int nz, float ox, float oy, float oz, float voxel, const float* esdf, int N,
                         const float* points, float* dist, float* grad, void* stream);

/* ---- mesh evaluation: visibility culling and exact nearest neighbours (splatam_b200/mesh_eval.py,
 * csrc/mesh_eval.cu) ---------------------------------------------------------------------------------------------
 * Float32, each operation rounded as written.  No host synchronisation.
 * sb_points_visible: points [N,3]; depth [B,H,W] and w2c [B,4,4] row-major (rows 0..2 read); mask uint8 [N] is read
 *   once and set to 1 where some frame of the launch sees the point: sb_tsdf_integrate's projection -- (x, y, z) =
 *   ((r0 px + r1 py) + r2 pz) + t; z > 0; pixel (floor(((fx x) / z) + cx + 0.5), floor(((fy y) / z) + cy + 0.5))
 *   inside the image -- and the depth d there has d > 0 and z <= d + occlusion_eps.  A frame with a non-finite pose
 *   marks nothing.  B frames give exactly what B single-frame calls give.
 * sb_nn_grid_build: bins N >= 1 reference points [N,3] into the gx x gy x gz grid of cubic cells of edge `cell` from
 *   origin o (cell (floor((p - o) / cell)) per axis, clamped into the grid), at most 2^28 cells, and keeps in the
 *   workspace (sb_nn_grid_workspace_bytes) the points in cell order and the per-cell start offsets.
 * sb_nn_query: d2 [M] float32 = min over the N reference points of (dx dx + dy dy) + dz dz, dx = qx - px, ...: equal
 *   to the brute-force minimum bit for bit (NaN for a non-finite query).  The same grid arguments as the build.
 * SB_ERR_BAD_ARG, before any launch, for null pointers the call reads, negative counts, an empty reference set, a
 * non-positive image or grid size, more than 2^28 cells, a non-finite origin, cell, camera or occlusion_eps, a
 * non-positive cell or a negative occlusion_eps; SB_ERR_WORKSPACE for a short workspace. */
SB_API int sb_points_visible(int n, const float* points, int B, int height, int width, const float* depth,
                             const float* w2c, float fx, float fy, float cx, float cy, float occlusion_eps,
                             uint8_t* mask, void* stream);
SB_API int sb_nn_grid_workspace_bytes(int n, int gx, int gy, int gz, size_t* bytes);
SB_API int sb_nn_grid_build(int n, const float* points, float ox, float oy, float oz, float cell, int gx, int gy,
                            int gz, void* workspace, size_t workspace_bytes, void* stream);
SB_API int sb_nn_query(int m, const float* queries, int n, float ox, float oy, float oz, float cell, int gx, int gy,
                       int gz, const void* workspace, size_t workspace_bytes, float* d2, void* stream);

/* ---- mesh depth rendering: a z-buffer triangle rasterizer (splatam_b200/mesh_eval.py, csrc/mesh_render.cu) -------
 * sb_mesh_depth: depth [B,H,W] float32 and face_id [B,H,W] int32 of the mesh vertices [V,3], faces int32 [F,3] seen
 *   by B cameras w2c [B,4,4] row-major (rows 0..2 read) with one pinhole fx, fy, cx, cy.  Float32, each operation
 *   rounded as written.  Per view and face:
 *   1. (x, y, z) = ((r0 px + r1 py) + r2 pz) + t per vertex (sb_tsdf_integrate's transform).
 *   2. The face is dropped when an index lies outside [0, V) or any camera coordinate is non-finite.
 *   3. Near clipping, z >= near inside: all three inside, the face as it is; none, dropped; otherwise the polygon of
 *      3 or 4 vertices the edges (v0,v1), (v1,v2), (v2,v0) give in order (each inside vertex, then the crossing
 *      point of a crossing edge), fanned from its first vertex.  A crossing edge with P inside and Q outside crosses
 *      at s = (near - zP) / (zQ - zP), x = xP + s (xQ - xP), y likewise, z = near exactly.  Pieces keep the face index.
 *   4. u = ((fx x) / z) + cx, v = ((fy y) / z) + cy; pixel (c, r) has its centre at (u, v) = (c, r).
 *   5. The pixels tested are c in [ceil(min u), floor(max u)], r in [ceil(min v), floor(max v)], clamped to the image.
 *   6. Edge function of P -> Q: e = ((u1 - u0)(r - v0)) - ((v1 - v0)(c - u0)) with (u0, v0), (u1, v1) the endpoints
 *      in lexicographic (u, v) order, negated when that swapped them.  ea = e(b -> c), eb = e(c -> a), ec = e(a -> b).
 *      Covered: all three >= 0 or all three <= 0, and s = (ea + eb) + ec != 0.  No back-face culling.
 *   7. iz = (((ea / za) + (eb / zb)) + (ec / zc)) / s, z = 1 / iz, drawn when z is finite and > 0.
 *   8. Z-buffer: atomicMin of the key (uint64(bits(z)) << 32) | face, so the nearest wins and, at equal depth, the
 *      lower face index; the result does not depend on the order of the writes.  depth = z and face_id = face where
 *      some face drew, 0 and -1 elsewhere.
 *   B views give exactly what B single-view calls give.  No host synchronisation.
 * SB_ERR_BAD_ARG, before any launch, for null pointers, V or F < 1, B, H or W < 1, B H W >= 2^31, B F >= 2^31 - 1,
 * a non-finite camera, fx or fy <= 0 and near <= 0 or non-finite; SB_ERR_WORKSPACE for a workspace smaller than
 * sb_mesh_depth_workspace_bytes gives. */
SB_API int sb_mesh_depth_workspace_bytes(int f, int B, int height, int width, size_t* bytes);
SB_API int sb_mesh_depth(int v, const float* vertices, int f, const int* faces, int B, int height, int width,
                         const float* w2c, float fx, float fy, float cx, float cy, float near, void* workspace,
                         size_t workspace_bytes, float* depth, int* face_id, void* stream);

/* ---- pose initialisation: projective point-to-plane ICP (splatam_b200/icp.py, csrc/icp.cu) -----------------------
 * sb_icp_align: the pose of frame t from its sensor depth and the map's depth rendered at frame t-1's pose.
 *   model_depth_sil float32 [2,H,W] (depth_acc, silhouette of the depth/silhouette render at w2c_prev), data_depth
 *   float32 [H,W] (frame t), one pinhole fx, fy, cx, cy (a pixel's centre at its integer coordinates), w2c_prev and
 *   w2c_init float32 [4,4] row-major on the device (rows 0..2 read; w2c_init is the constant-velocity guess),
 *   iters: host int[SB_ICP_LEVELS], the iterations of levels 0 (full size), 1, 2.  Float32, each operation rounded as
 *   written; oracle/icp_numpy.py restates the rule.
 *   1. Level 0: model depth = depth_acc / sil where sil > 0.99 and the quotient is finite and positive, else 0
 *      (invalid); data depth = the sensor depth where finite and positive, else 0.
 *   2. Level l + 1 (H >> 1, W >> 1): pixel (x, y) averages, in the order (2x,2y), (2x+1,2y), (2x,2y+1), (2x+1,2y+1),
 *      the block's valid samples within 0.05 m of the block's smallest one (sum / count), 0 if none is valid.
 *      Intrinsics: fx/2, fy/2, (cx - 0.5)/2, (cy - 0.5)/2.
 *   3. Vertex (u, v) = ((u - cx)/fx z, (v - cy)/fy z, z), 0 where invalid.  Model normal = cross(V(u+1) - V(u-1),
 *      V(v+1) - V(v-1)) / its norm, 0 (invalid) on the border, where a neighbour is invalid or where
 *      |z_neighbour - z| fx > 5 z (fx of the level).
 *   4. T = w2c_prev inv(w2c_init) (double; camera t -> camera t-1).  Levels 2, 1, 0, iters[l] times each: every valid
 *      data vertex v goes to p = R v + t (T rounded to float32), is projected to (floor(fx px/pz + cx + 0.5),
 *      floor(fy py/pz + cy + 0.5)) and pairs with the model vertex q and normal n there if pz > 0, the pixel is in
 *      the image, q and n are valid and |p - q|^2 <= (0.1 2^l m)^2.  r = n.(p - q), J = [p x n, n]; JtJ, Jtr,
 *      sum r^2 and the counts are summed in double in a fixed order (the result does not depend on the run).  One
 *      thread solves JtJ xi = -Jtr by Cholesky and sets T <- exp(xi) T; with fewer than 32 pairs or a matrix that
 *      is not positive definite the update is skipped.
 *   5. Accepted iff the last iteration had inliers / valid data pixels >= 0.4, RMS r <= 0.03 m, smallest / largest
 *      Cholesky pivot >= 1e-5 and its update was applied.  w2c_out [4,4] = inv(T) w2c_prev (double, rounded) if
 *      accepted, else w2c_init.
 *   stats double[SB_ICP_STATS]: 0 accepted (1/0), 1 inlier fraction, 2 RMS residual [m], 3 inliers, 4 valid data
 *   pixels, 5 pivot ratio (0: not positive definite or too few pairs), 6 some update skipped, 7 the last update
 *   skipped -- all of the last iteration --, 8..28 its JtJ (upper triangle, row-major), 29..34 its Jtr, 35 its sum r^2.
 *   No host synchronisation: the call can be captured into a CUDA graph.
 * sb_icp_export: copies level `level`'s maps out of a workspace an sb_icp_align call has filled (stream-ordered):
 *   model_depth, data_depth [H_l, W_l], model_vertex, model_normal, data_vertex [3, H_l, W_l] (x, y, z planes) and
 *   assoc uint8 [H_l, W_l] (0 no valid data, 1 not paired, 2 paired) of the latest iteration at that level.
 * SB_ERR_BAD_ARG, before any launch, for null pointers, H or W < 4, H W >= 2^31, a non-finite camera, fx or fy <= 0,
 * iterations outside [0, 1000] and a level outside [0, SB_ICP_LEVELS); SB_ERR_WORKSPACE for a workspace smaller than
 * sb_icp_workspace_bytes gives. */
#define SB_ICP_LEVELS 3
#define SB_ICP_STATS 36
SB_API int sb_icp_workspace_bytes(int height, int width, size_t* bytes);
SB_API int sb_icp_align(int height, int width, const float* model_depth_sil, const float* data_depth, float fx,
                        float fy, float cx, float cy, const float* w2c_prev, const float* w2c_init, const int* iters,
                        void* workspace, size_t workspace_bytes, float* w2c_out, double* stats, void* stream);
SB_API int sb_icp_export(int height, int width, const void* workspace, size_t workspace_bytes, int level,
                         float* model_depth, float* data_depth, float* model_vertex, float* model_normal,
                         float* data_vertex, uint8_t* assoc, void* stream);

/* ---- RGB-D ICP: joint geometric and photometric alignment (splatam_b200/icp.py, csrc/icp.cu) ----------------------
 * sb_rgbd_icp_align: sb_icp_align's arguments plus model_rgb float32 [3,H,W] (the map's RGB render at w2c_prev),
 *   data_rgb float32 [3,H,W] (frame t) and weight (lambda, metres per unit of intensity, finite and >= 0).  Float32,
 *   each operation rounded as written, double sums in a fixed order; oracle/rgbd_icp_numpy.py restates the rule.
 *   Steps 1-3 and the pairs of step 4 are sb_icp_align's, computed by the same device code.  In addition:
 *   a. Level 0 grey = (0.299 r + 0.587 g) + 0.114 b; model grey where the model depth is valid, data grey where the
 *      data depth is valid, NaN elsewhere.  A grey value is valid iff finite.
 *   b. Level l + 1 grey = (sum of the grey of exactly the samples the depth pyramid averaged, in its order) / their
 *      count; NaN where the depth is 0.
 *   c. Model gradient (gu, gv) = ((I(u+1) - I(u-1)) / 2, (I(v+1) - I(v-1)) / 2) where the model normal is valid, NaN
 *      elsewhere (so no gradient crosses a depth edge).
 *   d. Every data pixel with a geometric pair at p = R v + t (step 4, whose distance gate is the occlusion test) is
 *      projected to (uc, vc) = (fx px/pz + cx, fy py/pz + cy); with u0 = floor(uc), v0 = floor(vc), a = uc - u0, b =
 *      vc - v0 the taps (u0, v0), (u0+1, v0), (u0, v0+1), (u0+1, v0+1) must lie in the image with finite grey and
 *      gradient.  Weights (1-a)(1-b), a(1-b), (1-a)b, ab; a sample is ((w00 x00 + w10 x10) + w01 x01) + w11 x11.
 *      r_I = I_model - I_data, paired iff |r_I| <= SB_RGBD_ICP_MAX_RESIDUAL; g = (dpi/dp)^T grad I =
 *      (gu fx / pz, gv fy / pz, -((gu fx / pz) px + (gv fy / pz) py) / pz); J_I = [p x g, g], paired only if all six
 *      entries are finite (so the photometric sums stay finite).
 *   e. JtJ_I, Jtr_I, sum r_I^2 and the pair count are summed in double in the geometric sums' fixed order; the system
 *      solved is JtJ + weight^2 JtJ_I, Jtr + weight^2 Jtr_I, with sb_icp_align's skip rule and Cholesky.
 *   f. Accepted iff sb_icp_align's test passes on the joint system and, when weight > 0, the last iteration had at
 *      least SB_RGBD_ICP_MIN_PAIRS photometric pairs and photometric RMS <= SB_RGBD_ICP_MAX_RMS.
 *   stats double[SB_RGBD_ICP_STATS]: 0..35 as sb_icp_align's (8..34: the joint system solved; 3, 4, 35 geometric),
 *   36 photometric pairs, 37 photometric RMS (inf if none), 38..58 JtJ_I, 59..64 Jtr_I, 65 sum r_I^2 -- all of the
 *   last iteration.  With weight 0 the pose and stats 0..35 equal sb_icp_align's bit for bit.  No host
 *   synchronisation: the call can be captured into a CUDA graph.
 * sb_rgbd_icp_workspace_bytes: its workspace, which begins with sb_icp_align's (sb_icp_export reads it).
 * sb_rgbd_icp_export: level `level`'s model_grey, data_grey [H_l, W_l], model_grad [2, H_l, W_l] and photometric codes
 *   uint8 [H_l, W_l] (0 no geometric pair, 1 no photometric pair, 2 paired) of the latest iteration at that level.
 * SB_ERR_BAD_ARG as sb_icp_align, and for a null rgb pointer and a negative or non-finite weight; SB_ERR_WORKSPACE for
 * a workspace smaller than sb_rgbd_icp_workspace_bytes gives. */
#define SB_RGBD_ICP_STATS 66
#define SB_RGBD_ICP_MAX_RESIDUAL 0.3f
#define SB_RGBD_ICP_MAX_RMS 0.1
#define SB_RGBD_ICP_MIN_PAIRS 32.0
SB_API int sb_rgbd_icp_workspace_bytes(int height, int width, size_t* bytes);
SB_API int sb_rgbd_icp_align(int height, int width, const float* model_depth_sil, const float* model_rgb,
                             const float* data_depth, const float* data_rgb, float fx, float fy, float cx, float cy,
                             const float* w2c_prev, const float* w2c_init, const int* iters, float weight,
                             void* workspace, size_t workspace_bytes, float* w2c_out, double* stats, void* stream);
SB_API int sb_rgbd_icp_export(int height, int width, const void* workspace, size_t workspace_bytes, int level,
                              float* model_grey, float* data_grey, float* model_grad, uint8_t* photo, void* stream);

/* ---- loop closure: map deformation and the keyframe pose graph (splatam_b200/loop.py, csrc/loop.cu) ---------------
 * A correction is a rigid map from the old world to the new one, float32 [12] row-major 3x4 [R | t]; the table holds
 * one per frame.  oracle/loop_numpy.py restates every rule below.
 * sb_deform_gaussians: in place, one thread per Gaussian i, nothing at all if *apply_flag (device int) is 0.  The
 *   Gaussian takes the correction c of frame timestep[i] (float32 [P], the creation frame); a timestep outside [0, T)
 *   and an exact identity correction leave it unchanged.  Float32, each operation rounded as written:
 *     mean:  x'_r = ((c_r0 x + c_r1 y) + c_r2 z) + c_r3 for r = 0, 1, 2;
 *     q_c:   f0 = ((1 + r00) + r11) + r22, f1 = ((1 + r00) - r11) - r22, f2 = ((1 - r00) + r11) - r22,
 *            f3 = ((1 - r00) - r11) + r22; k = the first largest; row k of
 *            [[f0, r21 - r12, r02 - r20, r10 - r01], [r21 - r12, f1, r10 + r01, r02 + r20],
 *             [r02 - r20, r10 + r01, f2, r12 + r21], [r10 - r01, r02 + r20, r12 + r21, f3]]
 *            divided by 2 sqrt(max(f_k, 0));
 *     quaternion (unnormalised, w x y z): q' = q_c q, the Hamilton product with the terms in the order
 *            w = ((aw bw - ax bx) - ay by) - az bz, x = ((aw bx + ax bw) + ay bz) - az by,
 *            y = ((aw by - ax bz) + ay bw) + az bx, z = ((aw bz + ax by) - ay bx) + az bw.
 *   Scales, colours and opacities are not touched.  means3D [P,3] and unnorm_rotations [P,4] need 4-byte alignment.
 * sb_pose_graph_normal_equations: N nodes (w2c poses, double [N,12]), E edges (device int [E,2]: i, j), measurements
 *   Z double [E,12] and weights double [E,2] (w_rot, w_trans).  Edge e has the residual r = log(Z T_i T_j^-1) in se(3)
 *   (tangent order: rotation, translation; the log takes the angle atan2(|vee(R - R^T)| / 2, (tr R - 1) / 2) and
 *   assumes it is below pi), weighted by
 *   diag(w_rot I3, w_trans I3), with the left perturbation T <- exp(xi) T:
 *     d r / d xi_i = Jl^-1(r) Ad(Z), d r / d xi_j = -Jl^-1(r) Ad(Z T_i T_j^-1), Ad(T) = [[R, 0], [t^ R, R]],
 *     Jl^-1(r) = I - ad(r)/2 + ad(r)^2/12 (the series to the second order), ad(r) = [[phi^, 0], [rho^, phi^]].
 *   Writes residuals double [E,6], jacobians double [E,72] (the two row-major 6x6 blocks) and the dense normal equations
 *   of the free nodes 1..N-1 (node 0 is fixed): H double [6(N-1)]^2 = sum_e A^T W A and b double [6(N-1)] = sum_e
 *   A^T W r, accumulated edge by edge in order, so every call gives the same bits.  An edge with a node outside
 *   [0, N) or i == j adds nothing and gets NaN residuals.
 * sb_pose_graph_update: T_n <- exp(xi_n) T_n for n = 1..N-1 (xi double [6(N-1)], node n at 6(n-1)); then every edge's
 *   E = Z T_i T_j^-1 gives edge_err double [E,2] = (|t_E| in m, its rotation angle in rad, as above) and
 *   *apply_flag = 1 iff every
 *   edge has |t_E| <= max_residual_m and angle <= max_residual_rad (NaN fails); then corrections float32 [T,12]:
 *   frame s takes C = T_n^-1 T_n_old (double, rounded) of node n = frame_node[s] (device int [T]), the exact identity
 *   where node n did not move or frame_node[s] is outside [0, N).  One block, no host synchronisation.
 * SB_ERR_BAD_ARG, before any launch, for null pointers, P < 0, T < 1, N outside [2, 20000], E < 1 and negative or NaN
 * bounds. */
SB_API int sb_deform_gaussians(int P, float* means3D, float* unnorm_rotations, const float* timestep, int T,
                               const float* corrections, const int* apply_flag, void* stream);
SB_API int sb_pose_graph_normal_equations(int N, int E, const double* poses, const int* edges, const double* Z,
                                          const double* weights, double* residuals, double* jacobians, double* H,
                                          double* b, void* stream);
SB_API int sb_pose_graph_update(int N, int E, int T, double* poses, const double* poses_old, const double* xi,
                                const int* edges, const double* Z, const int* frame_node, double max_residual_m,
                                double max_residual_rad, float* corrections, int* apply_flag, double* edge_err,
                                void* stream);

/* ---- relocalisation: thumbnail retrieval and the tracking health check (splatam_b200/reloc.py, csrc/reloc.cu) -----
 * oracle/reloc_numpy.py restates every rule below.
 * sb_reloc_thumbnail_size: the descriptor size h x w of an H x W image: s = max(1, H / SB_RELOC_THUMB_ROWS) (integer
 *   division), h = H / s, w = W / s (the right and bottom remainder is cropped: 1200x680 -> 85x48, 640x480 -> 64x48).
 * sb_reloc_thumbnails: B images -> out float32 [B,2,h,w] (channel 0 grey, 1 depth); scratch float32 [B,2,h,w].
 *   rgb float32 [B,3,H,W], depth [B,H,W], sil [B,H,W] or NULL (a map render passes its silhouette and its depth_acc
 *   as `depth`; a sensor frame passes NULL and its depth).  Float32, each operation rounded as written:
 *   1. Sample (u, v): grey = (0.299 r + 0.587 g) + 0.114 b; depth = d, or d / sil with a silhouette.  With a silhouette,
 *      a sample with sil <= 0.99 (or NaN) is invalid in both channels.  A grey sample is valid if finite, a depth
 *      sample if finite and > 0.
 *   2. Block (x, y) = samples u in [x s, x s + s), v in [y s, y s + s): sum of the valid samples in row-major order
 *      (v outer, u inner) starting at 0, divided by their count; NaN (invalid) unless 2 count >= s^2.  Per channel.
 *   3. Blur: a valid value becomes sum w v / sum w over its valid 3x3 neighbours inside the descriptor (itself
 *      included), neighbours in row-major order (dy outer), w = (dy == 0 ? 2 : 1) (dx == 0 ? 2 : 1), each sum starting
 *      at 0; an invalid value stays NaN.
 * sb_reloc_score: query float32 [2,h,w] against database float32 [N,2,h,w] (pixels = h w) -> scores double [N].  Per
 *   channel: the pixels valid (not NaN) in both; n their count, m_q, m_d the means of their values (double);
 *   ncc = sum (q - m_q)(d - m_d) / sqrt(sum (q - m_q)^2 sum (d - m_d)^2), 0 where either sum of squares is 0.  Score =
 *   (ncc_grey + ncc_depth) / 2, or -2 when, in either channel, the query has no valid pixel, n < 2 or 2 n < the
 *   query's valid pixel count.  Sums in double in a fixed order (the same bits on every call).
 * sb_reloc_topk: the k <= SB_RELOC_MAX_K best of scores double [N] (k <= N): indices int [k] and their scores double
 *   [k], highest first, the lower index on ties (numpy's stable argsort of -score); NaN ranks below every number.
 * sb_track_health: depth_sil float32 [2,H,W] (depth_acc, silhouette of the map's depth/silhouette render at the tracked
 *   pose), frame_depth float32 [H,W].  Valid: frame depth finite and > 0; covered: valid and sil > 0.99; r =
 *   depth_acc / sil - frame depth (float32, rounded as written); inlier: covered and |r| < max(tau_abs, tau_rel *
 *   frame depth).  stats double [SB_RELOC_HEALTH_STATS]: 0 valid, 1 covered, 2 inliers, 3 RMS of r over the covered
 *   pixels (inf if none), 4 healthy (1/0): valid > 0, covered > 0, covered / valid >= min_coverage and inliers /
 *   covered >= min_inliers.  Counts are exact; the sum of r^2 is in double over SB_RELOC_HEALTH_BLOCKS fixed partials
 *   (scratch double [4 SB_RELOC_HEALTH_BLOCKS]), summed in block order.  No host synchronisation.
 * sb_track_health_rgb: sb_track_health's inputs plus map_rgb float32 [3,H,W] (the map's RGB render at the tracked pose)
 *   and frame_rgb float32 [3,H,W].  Entries 0..3 equal sb_track_health's bit for bit.  Over the inliers whose six
 *   colour values (map and frame r, g, b) are all finite: 5 their count, 6 the colour NCC of the map against the
 *   frame: each channel centred on its own mean, ncc = sum_c sum (m_c - mm_c)(f_c - mf_c) / sqrt(sum_c sum (m_c -
 *   mm_c)^2 sum_c sum (f_c - mf_c)^2), 0 where either sum of squares is 0.  In double, in two passes (the means, then
 *   the centred sums) over SB_RELOC_HEALTH_BLOCKS fixed partials summed in block order (scratch double
 *   [22 SB_RELOC_HEALTH_BLOCKS]).  4 healthy: sb_track_health's test, ncc >= min_ncc and count >=
 *   SB_RELOC_MIN_NCC_PAIRS.  No host synchronisation.
 * SB_ERR_BAD_ARG, before any launch, for null pointers (sil may be NULL), sizes < 1, pixels > SB_RELOC_MAX_PIXELS,
 * k outside [1, min(N, SB_RELOC_MAX_K)], negative or non-finite tolerances, thresholds outside [0, 1] and min_ncc
 * outside [-1, 1]. */
#define SB_RELOC_THUMB_ROWS 48
#define SB_RELOC_MAX_K 8
#define SB_RELOC_MAX_PIXELS 28000
#define SB_RELOC_HEALTH_BLOCKS 128
#define SB_RELOC_HEALTH_STATS 5
#define SB_RELOC_HEALTH_RGB_STATS 7
#define SB_RELOC_MIN_NCC_PAIRS 64.0
SB_API int sb_reloc_thumbnail_size(int height, int width, int* h, int* w);
SB_API int sb_reloc_thumbnails(int B, int height, int width, const float* rgb, const float* depth, const float* sil,
                               float* scratch, float* out, void* stream);
SB_API int sb_reloc_score(int N, int pixels, const float* query, const float* database, double* scores, void* stream);
SB_API int sb_reloc_topk(int N, int k, const double* scores, int* indices, double* top_scores, void* stream);
SB_API int sb_track_health(int height, int width, const float* depth_sil, const float* frame_depth, float tau_abs,
                           float tau_rel, double min_coverage, double min_inliers, double* scratch, double* stats,
                           void* stream);
SB_API int sb_track_health_rgb(int height, int width, const float* depth_sil, const float* frame_depth,
                               const float* map_rgb, const float* frame_rgb, float tau_abs, float tau_rel,
                               double min_coverage, double min_inliers, double min_ncc, double* scratch, double* stats,
                               void* stream);

/* ---- per-frame exposure and white balance (splatam_b200/train_ops.py `exposure`, csrc/exposure.cu) --------------
 * A frame's colour correction is ab float32 [6] (device) = (a_r, a_g, a_b, b_r, b_g, b_b): log-gains and biases.
 * Images are float32 [3,H,W] (device), channel c the values c*H*W .. (c+1)*H*W - 1; no alignment is assumed.
 * Every call reads ab from device memory (a graph replay picks up new values) and never synchronises the host.
 * sb_exposure_apply: g_c = float(exp(double(a_c))), or float(exp(-double(a_c))) when `inverse`;
 *   y = __fadd_rn(__fmul_rn(g_c, x), b_c), or when `inverse` y = __fmul_rn(__fsub_rn(x, b_c), g_c).  y may be x.
 * sb_exposure_backward: the gradient of the forward transform for an upstream gy [3,H,W]: gx = __fmul_rn(g_c, gy)
 *   (float32 [3,H,W], may be gy) and g_ab double [6] = (exp(double(a_c)) S_c, G_c) with S_c = sum over channel c of
 *   double(gy) double(x) and G_c = sum of double(gy): each sum over SB_EXPOSURE_BLOCKS fixed partials added in block
 *   order, no atomics, so a call gives the same bits every time.  workspace: sb_exposure_workspace_bytes.
 * SB_ERR_BAD_ARG, before any launch, for sizes < 1, null pointers and `inverse` outside {0, 1}; SB_ERR_WORKSPACE for
 * a short workspace. */
#define SB_EXPOSURE_BLOCKS 264
SB_API int sb_exposure_workspace_bytes(int height, int width, size_t* bytes);
SB_API int sb_exposure_apply(int height, int width, const float* x, const float* ab, int inverse, float* y,
                             void* stream);
SB_API int sb_exposure_backward(int height, int width, const float* x, const float* ab, const float* gy, float* gx,
                                double* g_ab, void* workspace, size_t workspace_bytes, void* stream);

/* ---- motion masks from the map's depth residual (splatam_b200/dynamic.py, csrc/dynamic.cu) ------------------------
 * Inputs: depth_sil float32 [3,H,W] (device; d = channel 0, s = channel 1), the frame's depth g float32 [H,W].
 * valid = g > 0 & isfinite(d) & s > sil_thres;  r = __fdiv_rn(__fsub_rn(d, g), g).
 * sb_dynamic_residual: writes r [H*W] (every pixel), zeroes then fills hist uint32 [SB_DYNAMIC_BINS] with the counts
 *   of bits(|r|) >> 16 over valid pixels, zeroes stats float32 [SB_DYNAMIC_STATS] and sets stats[0] = valid count.
 * sb_dynamic_scale: one CTA; stats[1] = scale = the float with bits b << 16, b the bin holding element (n - 1) / 2 of
 *   the valid |r| sorted ascending (n = stats[0]; 0 when n = 0).
 * sb_dynamic_seeds: thr(k, f) = k*scale if k*scale > f else f (float32).  occ = valid & r > thr(k_high, r_min),
 *   dis = valid & -r > thr(k_high, r_min); a seed is kept when >= 4 of its 8 neighbours are seeds of its kind.
 *   cand = g > 0 & ((valid & r > thr(k_low, r_min * 0.5f)) | s <= sil_thres).  flags uint8 [H*W] = kept occ (1) |
 *   kept dis (2) | cand (4); dyn uint8 [H*W] = kept occ (0/1); stats[2], stats[3] += kept occ, dis counts.
 * sb_dynamic_grow: `radius` Jacobi steps of  dyn'(q) = dyn(q) | (cand(q) & some 4-neighbour p has dyn(p) and
 *   |g_p - g_q| <= tau * min(g_p, g_q))  (float32, rounded as written), SB_DYNAMIC_GROW_STEPS steps per launch; the
 *   result is in `dyn`; tmp uint8 [H*W] is scratch.
 * sb_dynamic_dilate: dynamic = Chebyshev dilation by `dilate` of grown, inconsistent = that of the kept dis seeds
 *   (uint8 0/1 [H*W]); stats[4], stats[5] += their counts.
 * stats = (valid, scale, occ seeds, dis seeds, dynamic, inconsistent): counts are float32 sums of integers, exact
 * because H*W < 2^24.  No call synchronises the host; all can be captured in a CUDA graph.
 * SB_ERR_BAD_ARG, before any launch, for H or W < 1, H*W >= 2^24, null pointers, NaN k_high / k_low, r_min or tau
 * not finite and >= 0, radius < 0, dilate outside [0, 64] and dyn == tmp. */
#define SB_DYNAMIC_BINS 32768
#define SB_DYNAMIC_STATS 6
#define SB_DYNAMIC_GROW_STEPS 8
SB_API int sb_dynamic_residual(int height, int width, const float* depth_sil, const float* gt_depth, float sil_thres,
                               float* residual, uint32_t* hist, float* stats, void* stream);
SB_API int sb_dynamic_scale(const uint32_t* hist, float* stats, void* stream);
SB_API int sb_dynamic_seeds(int height, int width, const float* depth_sil, const float* gt_depth,
                            const float* residual, float sil_thres, float k_high, float k_low, float r_min,
                            uint8_t* flags, uint8_t* dyn, float* stats, void* stream);
SB_API int sb_dynamic_grow(int height, int width, const float* gt_depth, const uint8_t* flags, float tau, int radius,
                           uint8_t* dyn, uint8_t* tmp, void* stream);
SB_API int sb_dynamic_dilate(int height, int width, const uint8_t* grown, const uint8_t* flags, int dilate,
                             uint8_t* dynamic, uint8_t* inconsistent, float* stats, void* stream);

/* ---- per-stage device timing (measurement only; bench.py's roofline pass) -------------------
 * Between sb_profile_begin() and sb_profile_end() every stage launch of this process is bracketed
 * by CUDA events on its stream.  sb_profile_end synchronises, writes the summed milliseconds and call
 * counts per stage (arrays of SB_NUM_STAGES) and disables the bracketing.  Not thread-safe. */
#define SB_NUM_STAGES 10
SB_API int sb_profile_begin(void);
SB_API int sb_profile_end(float* stage_ms, int* stage_calls);
SB_API const char* sb_stage_name(int stage);

#ifdef __cplusplus
}
#endif
#endif /* SPLATAM_B200_H_INCLUDED */
