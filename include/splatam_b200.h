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
 * parameters; if want_pose, g_pose16 receives d/d rel_w2c[0:3,0:4] (12) then d/d cam_rot (4). */
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
                               float* g_log_scales, float* g_pose16, void* stream);

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

/* ---- frame ingest (the dataset readers, splatam_b200/datasets.py; R/datasets/gradslam_datasets/basedataset.py) ---
 * One launch: rgb uint8 [color_height, color_width, 3] (HWC) and depth uint16 [depth_height, depth_width] (device)
 * -> color_out float32 [3, height, width] = float32(bilinear_f64(rgb)) / 255 and depth_out float32 [1, height, width]
 * = float32(nearest(depth) / png_depth_scale), division in double: cv2.resize INTER_LINEAR / INTER_NEAREST on float64
 * as the reference's loader calls it, including cv2's exact-2x box average and the plain copy at equal size.  The two
 * source sizes may differ.  SB_ERR_BAD_ARG for a non-positive size or depth scale and for null pointers. */
SB_API int sb_ingest_rgbd(const uint8_t* rgb, int color_height, int color_width, const uint16_t* depth,
                          int depth_height, int depth_width, int height, int width, double png_depth_scale,
                          float* color_out, float* depth_out, void* stream);

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
