// map_ops.cu -- map maintenance of the SLAM loop as stream-compaction kernels (SURVEY.md section 8(f) row N3,
// "prune/densify compaction"):
//   * prune:  keep mask from opacity / size thresholds (prune_gaussians, R/utils/slam_external.py:170-190) and
//             compaction of the packed parameter buffer and both Adam moments (remove_points, :144-167), which the
//             reference does as 15 boolean-mask gathers plus 4 more for its bookkeeping vectors;
//   * grow:   non-presence mask of a frame (add_new_gaussians, R/scripts/splatam.py:378-420) and back-projection of
//             the selected pixels into new Gaussian rows (get_pointcloud, :67-118; initialize_new_params, :348-375).
// Both are "mask -> exclusive scan -> scatter": the scan (CUB) is shared (sb_compact_plan).
#include "common.cuh"
#include <cub/device/device_scan.cuh>
#include <cub/iterator/transform_input_iterator.cuh>

namespace sb {

namespace {

constexpr int kMaxSeg = 16;
struct FlatSegs { uint32_t end[kMaxSeg]; uint32_t width[kMaxSeg]; int n; };

struct MaskToCount {
    __host__ __device__ uint32_t operator()(uint8_t m) const { return m ? 1u : 0u; }
};

__global__ void __launch_bounds__(256)
prune_mask_kernel(int P, const float* __restrict__ logit_opacities, const float* __restrict__ log_scales,
                  int scale_dim, float opacity_threshold, float big_threshold, uint8_t* __restrict__ keep) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P) return;
    // torch.sigmoid(x) < threshold, in the same float arithmetic (1 / (1 + exp(-x)))
    const float op = 1.0f / (1.0f + expf(-logit_opacities[i]));
    bool remove = op < opacity_threshold;
    if (big_threshold > 0.f) {        // exp(log_scales).max(dim=1) > 0.1 * scene_radius
        float s = expf(log_scales[(size_t)i * scale_dim]);
        for (int k = 1; k < scale_dim; ++k) s = fmaxf(s, expf(log_scales[(size_t)i * scale_dim + k]));
        remove = remove || (s > big_threshold);
    }
    keep[i] = remove ? 0 : 1;
}

__global__ void count_kernel(int n, const uint8_t* __restrict__ keep, const uint32_t* __restrict__ dst_index,
                             int32_t* __restrict__ count) {
    if (threadIdx.x == 0 && blockIdx.x == 0) *count = (int32_t)(dst_index[n - 1] + (keep[n - 1] ? 1u : 0u));
}

// One thread per element of the packed source buffer [seg0: w0*P | seg1: w1*P | ...] (coalesced reads); kept
// rows land in the packed destination of P_new rows.
__global__ void __launch_bounds__(256)
compact_flat_kernel(uint32_t n, uint32_t P, uint32_t P_new, const uint8_t* __restrict__ keep,
                    const uint32_t* __restrict__ dst_index, FlatSegs segs, const float* __restrict__ src,
                    float* __restrict__ dst) {
    const uint32_t e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= n) return;
    uint32_t start = 0, start_new = 0, width = 1;
    for (int k = 0; k < segs.n; ++k) {
        width = segs.width[k];
        if (e < segs.end[k]) break;
        start = segs.end[k];
        start_new += width * P_new;
    }
    const uint32_t local = e - start, row = local / width, col = local - row * width;
    if (keep[row]) dst[start_new + dst_index[row] * width + col] = src[e];
}

__global__ void __launch_bounds__(256)
depth_error_kernel(int HW, const float* __restrict__ depth_sil, const float* __restrict__ gt_depth,
                   float* __restrict__ err) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= HW) return;
    const float gt = gt_depth[i];
    err[i] = fabsf(gt - depth_sil[i]) * (gt > 0.f ? 1.f : 0.f);        // splatam.py:391
}

__global__ void __launch_bounds__(256)
new_gaussian_mask_kernel(int HW, const float* __restrict__ depth_sil, const float* __restrict__ gt_depth,
                         float sil_thres, float depth_err_thres, uint8_t* __restrict__ mask) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= HW) return;
    const float gt = gt_depth[i], rd = depth_sil[i], sil = depth_sil[HW + i];
    const float err = fabsf(gt - rd) * (gt > 0.f ? 1.f : 0.f);
    const bool no_sil = sil < sil_thres;                                 // splatam.py:386
    const bool in_front = (rd > gt) && (err > depth_err_thres);          // :392, threshold = 50 * median(err)
    mask[i] = ((no_sil || in_front) && gt > 0.f) ? 1 : 0;                // :394, :404-405
}

// accumulate_mean2d_gradient of densify (R/utils/slam_external.py:200-204) without the boolean-mask gathers and the
// nonzero they synchronise on: each seen row gets accum += |g[:2]| and denom += 1, each element one addition, so the
// result is the torch statement's bit for bit.  The norm is sqrt(round(gx^2) + round(gy^2)), the rounding of torch's
// two-element NormTwoOps reduction: explicit _rn intrinsics keep nvcc from contracting it into an FMA.
__global__ void __launch_bounds__(256)
densify_accumulate_kernel(int P, const float* __restrict__ means2D_grad, int grad_stride,
                          const uint8_t* __restrict__ seen, float* __restrict__ accum, float* __restrict__ denom) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P || !seen[i]) return;
    const float gx = means2D_grad[(size_t)i * grad_stride], gy = means2D_grad[(size_t)i * grad_stride + 1];
    accum[i] = __fadd_rn(accum[i], sqrtf(__fadd_rn(__fmul_rn(gx, gx), __fmul_rn(gy, gy))));
    denom[i] = __fadd_rn(denom[i], 1.0f);
}

struct Mat34 { float m[12]; };

__global__ void __launch_bounds__(256)
backproject_kernel(int H, int W, const float* __restrict__ color, const float* __restrict__ depth, float fx, float fy,
                   float cx, float cy, Mat34 c2w, const uint8_t* __restrict__ mask,
                   const uint32_t* __restrict__ dst_index, int scale_dim, float* __restrict__ means3D,
                   float* __restrict__ rgb, float* __restrict__ log_scales, float* __restrict__ mean_sq_dist) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const int HW = H * W;
    if (i >= HW) return;
    if (mask != nullptr && !mask[i]) return;
    const uint32_t j = mask != nullptr ? dst_index[i] : (uint32_t)i;
    const int px = i % W, py = i / W;
    const float z = depth[i];
    const float xx = ((float)px - cx) / fx, yy = ((float)py - cy) / fy;  // splatam.py:79-80
    const float x = xx * z, y = yy * z;
    for (int r = 0; r < 3; ++r)                                          // (c2w @ [x y z 1]^T)[:3]
        means3D[3 * (size_t)j + r] = fmaf(c2w.m[4 * r + 2], z, fmaf(c2w.m[4 * r + 1], y, c2w.m[4 * r] * x)) + c2w.m[4 * r + 3];
    for (int c = 0; c < 3; ++c) rgb[3 * (size_t)j + c] = color[(size_t)c * HW + i];
    const float s = z / ((fx + fy) / 2.0f);                              // "projective" mean distance, :99-101
    const float sq = s * s;
    if (mean_sq_dist != nullptr) mean_sq_dist[j] = sq;
    const float ls = logf(sqrtf(sq));                                    // initialize_new_params, :353-357
    for (int k = 0; k < scale_dim; ++k) log_scales[(size_t)j * scale_dim + k] = ls;
}

}  // namespace
}  // namespace sb

using namespace sb;

extern "C" {

SB_API int sb_prune_mask(int P, const float* logit_opacities, const float* log_scales, int scale_dim,
                         float opacity_threshold, float big_threshold, uint8_t* keep, void* stream) {
    if (P < 0 || (scale_dim != 1 && scale_dim != 3)) return SB_ERR_BAD_ARG;
    if (P == 0) return SB_OK;
    if (!logit_opacities || !log_scales || !keep) return SB_ERR_BAD_ARG;
    prune_mask_kernel<<<(P + 255) / 256, 256, 0, (cudaStream_t)stream>>>(P, logit_opacities, log_scales, scale_dim,
                                                                         opacity_threshold, big_threshold, keep);
    SB_LAUNCH_CHECK("prune_mask_kernel");
    return SB_OK;
}

SB_API int sb_compact_plan_bytes(int n, size_t* bytes) {
    if (n < 0 || !bytes) return SB_ERR_BAD_ARG;
    size_t temp = 0;
    cub::TransformInputIterator<uint32_t, MaskToCount, const uint8_t*> it(nullptr, MaskToCount());
    cub::DeviceScan::ExclusiveSum(nullptr, temp, it, (uint32_t*)nullptr, n > 0 ? n : 1);
    *bytes = ((temp + 255) / 256) * 256 + 256;      // scan temp + one 256-B slot for the device-side count
    return SB_OK;
}

SB_API int sb_compact_plan(int n, const uint8_t* keep, uint32_t* dst_index, void* temp, size_t temp_bytes,
                           int* count_host, void* stream) {
    if (n < 0 || !count_host) return SB_ERR_BAD_ARG;
    *count_host = 0;
    if (n == 0) return SB_OK;
    size_t need = 0;
    sb_compact_plan_bytes(n, &need);
    if (!keep || !dst_index || !temp) return SB_ERR_BAD_ARG;
    if (temp_bytes < need) return SB_ERR_WORKSPACE;
    cudaStream_t st = (cudaStream_t)stream;
    int32_t* count_dev = reinterpret_cast<int32_t*>(temp);
    void* scan_temp = reinterpret_cast<char*>(temp) + 256;
    size_t scan_bytes = temp_bytes - 256;
    cub::TransformInputIterator<uint32_t, MaskToCount, const uint8_t*> it(keep, MaskToCount());
    SB_CUDA_CHECK(cub::DeviceScan::ExclusiveSum(scan_temp, scan_bytes, it, dst_index, n, st));
    count_kernel<<<1, 32, 0, st>>>(n, keep, dst_index, count_dev);
    SB_LAUNCH_CHECK("count_kernel");
    int32_t c = 0;
    SB_CUDA_CHECK(cudaMemcpyAsync(&c, count_dev, sizeof(int32_t), cudaMemcpyDeviceToHost, st));
    SB_CUDA_CHECK(cudaStreamSynchronize(st));
    *count_host = (int)c;
    return SB_OK;
}

SB_API int sb_compact_flat(int P, int P_new, const uint8_t* keep, const uint32_t* dst_index, int num_segments,
                           const int* widths, const float* src, float* dst, void* stream) {
    if (P < 0 || P_new < 0 || P_new > P || num_segments < 1 || num_segments > kMaxSeg || !widths) return SB_ERR_BAD_ARG;
    FlatSegs segs;
    segs.n = num_segments;
    uint64_t acc = 0;
    for (int k = 0; k < num_segments; ++k) {
        if (widths[k] < 1) return SB_ERR_BAD_ARG;
        acc += (uint64_t)widths[k] * (uint64_t)P;
        if (acc > 0xFFFFFFFFull) return SB_ERR_BAD_ARG;
        segs.end[k] = (uint32_t)acc;
        segs.width[k] = (uint32_t)widths[k];
    }
    if (P == 0 || P_new == 0) return SB_OK;
    if (!keep || !dst_index || !src || !dst) return SB_ERR_BAD_ARG;
    const uint32_t n = (uint32_t)acc;
    compact_flat_kernel<<<(n + 255) / 256, 256, 0, (cudaStream_t)stream>>>(n, (uint32_t)P, (uint32_t)P_new, keep,
                                                                           dst_index, segs, src, dst);
    SB_LAUNCH_CHECK("compact_flat_kernel");
    return SB_OK;
}

SB_API int sb_densify_accumulate(int P, const float* means2D_grad, int grad_stride, const uint8_t* seen, float* accum,
                                 float* denom, void* stream) {
    if (P < 0 || grad_stride < 2) return SB_ERR_BAD_ARG;
    if (P == 0) return SB_OK;
    if (!means2D_grad || !seen || !accum || !denom) return SB_ERR_BAD_ARG;
    densify_accumulate_kernel<<<(P + 255) / 256, 256, 0, (cudaStream_t)stream>>>(P, means2D_grad, grad_stride, seen,
                                                                                 accum, denom);
    SB_LAUNCH_CHECK("densify_accumulate_kernel");
    return SB_OK;
}

SB_API int sb_depth_error(int H, int W, const float* depth_sil, const float* gt_depth, float* err, void* stream) {
    if (H <= 0 || W <= 0 || !depth_sil || !gt_depth || !err) return SB_ERR_BAD_ARG;
    const int HW = H * W;
    depth_error_kernel<<<(HW + 255) / 256, 256, 0, (cudaStream_t)stream>>>(HW, depth_sil, gt_depth, err);
    SB_LAUNCH_CHECK("depth_error_kernel");
    return SB_OK;
}

SB_API int sb_new_gaussian_mask(int H, int W, const float* depth_sil, const float* gt_depth, float sil_thres,
                                float depth_err_thres, uint8_t* mask, void* stream) {
    if (H <= 0 || W <= 0 || !depth_sil || !gt_depth || !mask) return SB_ERR_BAD_ARG;
    const int HW = H * W;
    new_gaussian_mask_kernel<<<(HW + 255) / 256, 256, 0, (cudaStream_t)stream>>>(HW, depth_sil, gt_depth, sil_thres,
                                                                                depth_err_thres, mask);
    SB_LAUNCH_CHECK("new_gaussian_mask_kernel");
    return SB_OK;
}

SB_API int sb_backproject(int H, int W, const float* color, const float* depth, float fx, float fy, float cx, float cy,
                          const float* c2w_host, const uint8_t* mask, const uint32_t* dst_index, int scale_dim,
                          float* means3D, float* rgb, float* log_scales, float* mean_sq_dist, void* stream) {
    if (H <= 0 || W <= 0 || !color || !depth || !c2w_host || !means3D || !rgb || !log_scales) return SB_ERR_BAD_ARG;
    if ((scale_dim != 1 && scale_dim != 3) || (mask != nullptr && dst_index == nullptr)) return SB_ERR_BAD_ARG;
    Mat34 m;
    for (int k = 0; k < 12; ++k) m.m[k] = c2w_host[k];
    const int HW = H * W;
    backproject_kernel<<<(HW + 255) / 256, 256, 0, (cudaStream_t)stream>>>(H, W, color, depth, fx, fy, cx, cy, m, mask,
                                                                          dst_index, scale_dim, means3D, rgb,
                                                                          log_scales, mean_sq_dist);
    SB_LAUNCH_CHECK("backproject_kernel");
    return SB_OK;
}

}  // extern "C"
