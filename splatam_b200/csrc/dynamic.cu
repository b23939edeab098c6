// dynamic.cu -- per-frame motion masks from the map's depth residual (splatam_b200/dynamic.py; the rule is stated in
// include/splatam_b200.h and restated in oracle/dynamic_numpy.py, which gives the same bits).
//
//   sb_dynamic_residual  r = (d - g) / g per pixel, and a 32768-bin histogram of the top 16 bits of |r| over the
//                        valid pixels (integer atomics: the counts do not depend on the order)
//   sb_dynamic_scale     one CTA: the bin of the lower-middle valid |r|, scale = the float whose bits are bin << 16
//   sb_dynamic_seeds     16x16 tiles with a one-pixel halo of raw seeds in shared memory: occluding / disoccluding
//                        seeds with >= 4 of 8 seed neighbours, and the growth candidates
//   sb_dynamic_grow      `radius` Jacobi steps of 4-connected, depth-continuous dilation through the candidates,
//                        kGrowHalo steps per launch on a 32x32 tile with a kGrowHalo halo held in shared memory
//   sb_dynamic_dilate    Chebyshev dilation of the grown mask and of the disoccluding seeds, and their counts
// Stats are float32 sums of integers (exact below 2^24 pixels, which the entry points require), so they too do not
// depend on the order of the atomics.  Nothing here synchronises the host; every call can be captured in a graph.
#include <cmath>

#include "common.cuh"

namespace sb {

namespace {

constexpr int kBins = SB_DYNAMIC_BINS;
constexpr int kScaleThreads = 1024;
constexpr int kSeedTile = 16;
constexpr int kGrowTile = 32;
constexpr int kGrowHalo = SB_DYNAMIC_GROW_STEPS;
constexpr int kGrowExt = kGrowTile + 2 * kGrowHalo;
constexpr uint8_t kOcc = 1, kDis = 2, kCand = 4;

__device__ __forceinline__ bool valid_px(float g, float d, float s, float sil_thres) {
    return g > 0.f && isfinite(d) && s > sil_thres;
}

// max(k * scale, floor) with a NaN product (inf * 0) taking the floor, as the numpy and torch statements do
__device__ __forceinline__ float threshold(float k, float scale, float floor_) {
    const float t = __fmul_rn(k, scale);
    return t > floor_ ? t : floor_;
}

__device__ __forceinline__ bool continuous(float gp, float gq, float tau) {
    return fabsf(__fsub_rn(gp, gq)) <= __fmul_rn(tau, fminf(gp, gq));
}

// one float32 atomic per CTA of an integer count: exact below 2^24, so the sum does not depend on the order
__device__ __forceinline__ void block_count(int v, float* dst) {
    const int n = __syncthreads_count(v);
    if (threadIdx.x == 0 && threadIdx.y == 0 && n) atomicAdd(dst, (float)n);
}

__global__ void __launch_bounds__(256) residual_kernel(int HW, const float* __restrict__ depth_sil,
                                                       const float* __restrict__ gt, float sil_thres,
                                                       float* __restrict__ residual, uint32_t* __restrict__ hist,
                                                       float* __restrict__ stats) {
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    bool v = false;
    if (p < HW) {
        const float d = depth_sil[p], s = depth_sil[HW + p], g = gt[p];
        const float r = __fdiv_rn(__fsub_rn(d, g), g);
        residual[p] = r;
        v = valid_px(g, d, s, sil_thres);
        if (v) atomicAdd(&hist[__float_as_uint(fabsf(r)) >> 16], 1u);
    }
    block_count(v, &stats[0]);
}

// the lower-middle element (0-based index (n - 1) / 2 of the sorted valid |r|) lies in the first bin whose inclusive
// prefix count exceeds that index; n = 0 gives scale 0
__global__ void __launch_bounds__(kScaleThreads) scale_kernel(const uint32_t* __restrict__ hist,
                                                              float* __restrict__ stats) {
    constexpr int kPer = kBins / kScaleThreads;
    __shared__ uint32_t part[kScaleThreads];
    const int t = threadIdx.x;
    uint32_t local = 0;
    for (int i = 0; i < kPer; ++i) local += hist[t * kPer + i];
    part[t] = local;
    __syncthreads();
    for (int off = 1; off < kScaleThreads; off <<= 1) {       // inclusive Hillis-Steele scan of the thread sums
        const uint32_t add = t >= off ? part[t - off] : 0u;
        __syncthreads();
        part[t] += add;
        __syncthreads();
    }
    const uint32_t n = (uint32_t)stats[0];
    if (n == 0) {
        if (t == 0) stats[1] = 0.f;
        return;
    }
    const uint32_t k = (n - 1) / 2;
    uint32_t acc = part[t] - local;
    if (acc <= k && k < part[t]) {                            // exactly one thread holds the element
        int b = t * kPer;
        for (;; ++b) {
            acc += hist[b];
            if (acc > k) break;
        }
        stats[1] = __uint_as_float((uint32_t)b << 16);
    }
}

__device__ __forceinline__ uint8_t raw_flags(int x, int y, int W, int H, const float* depth_sil, const float* gt,
                                             const float* residual, float sil_thres, float thr_hi, float thr_lo) {
    if (x < 0 || y < 0 || x >= W || y >= H) return 0;
    const int HW = W * H, p = y * W + x;
    const float d = depth_sil[p], s = depth_sil[HW + p], g = gt[p], r = residual[p];
    if (!(g > 0.f)) return 0;
    const bool v = valid_px(g, d, s, sil_thres);
    uint8_t f = 0;
    if (v && r > thr_hi) f |= kOcc;
    if (v && -r > thr_hi) f |= kDis;
    if ((v && r > thr_lo) || s <= sil_thres) f |= kCand;
    return f;
}

__global__ void __launch_bounds__(kSeedTile * kSeedTile) seeds_kernel(
    int H, int W, const float* __restrict__ depth_sil, const float* __restrict__ gt,
    const float* __restrict__ residual, float sil_thres, float k_high, float k_low, float r_min,
    uint8_t* __restrict__ flags, uint8_t* __restrict__ dyn, float* __restrict__ stats) {
    __shared__ uint8_t raw[kSeedTile + 2][kSeedTile + 2];
    const float scale = stats[1];
    const float thr_hi = threshold(k_high, scale, r_min), thr_lo = threshold(k_low, scale, __fmul_rn(r_min, 0.5f));
    const int x0 = blockIdx.x * kSeedTile - 1, y0 = blockIdx.y * kSeedTile - 1;
    const int tid = threadIdx.y * kSeedTile + threadIdx.x;
    for (int i = tid; i < (kSeedTile + 2) * (kSeedTile + 2); i += kSeedTile * kSeedTile) {
        const int ry = i / (kSeedTile + 2), rx = i % (kSeedTile + 2);
        raw[ry][rx] = raw_flags(x0 + rx, y0 + ry, W, H, depth_sil, gt, residual, sil_thres, thr_hi, thr_lo);
    }
    __syncthreads();
    const int x = blockIdx.x * kSeedTile + threadIdx.x, y = blockIdx.y * kSeedTile + threadIdx.y;
    const uint8_t me = raw[threadIdx.y + 1][threadIdx.x + 1];
    int n_occ = 0, n_dis = 0;
#pragma unroll
    for (int dy = 0; dy < 3; ++dy)
#pragma unroll
        for (int dx = 0; dx < 3; ++dx) {
            if (dy == 1 && dx == 1) continue;
            const uint8_t f = raw[threadIdx.y + dy][threadIdx.x + dx];
            n_occ += f & kOcc;
            n_dis += (f & kDis) >> 1;
        }
    uint8_t out = me & kCand;
    if ((me & kOcc) && n_occ >= 4) out |= kOcc;
    if ((me & kDis) && n_dis >= 4) out |= kDis;
    const bool inside = x < W && y < H;
    if (inside) {
        flags[y * W + x] = out;
        dyn[y * W + x] = out & kOcc;
    }
    block_count(inside && (out & kOcc), &stats[2]);
    block_count(inside && (out & kDis), &stats[3]);
}

// `steps` (<= kGrowHalo) Jacobi steps on a tile: after step j the values at distance >= j from the edge of the
// loaded (tile + halo) region are exact, so after kGrowHalo steps the tile itself is
__global__ void __launch_bounds__(256) grow_kernel(int H, int W, const float* __restrict__ gt,
                                                   const uint8_t* __restrict__ flags, float tau, int steps,
                                                   const uint8_t* __restrict__ src, uint8_t* __restrict__ dst) {
    __shared__ float sg[kGrowExt][kGrowExt];
    __shared__ uint8_t sf[kGrowExt][kGrowExt];           // candidate bit
    __shared__ uint8_t sd[2][kGrowExt][kGrowExt];
    const int x0 = blockIdx.x * kGrowTile - kGrowHalo, y0 = blockIdx.y * kGrowTile - kGrowHalo;
    const int tid = threadIdx.x, nt = blockDim.x;
    for (int i = tid; i < kGrowExt * kGrowExt; i += nt) {
        const int ry = i / kGrowExt, rx = i % kGrowExt, x = x0 + rx, y = y0 + ry;
        const bool in = x >= 0 && y >= 0 && x < W && y < H;
        sg[ry][rx] = in ? gt[y * W + x] : 0.f;
        sf[ry][rx] = in ? (flags[y * W + x] & kCand) : 0;
        sd[0][ry][rx] = in ? src[y * W + x] : 0;
    }
    __syncthreads();
    int cur = 0;
    for (int s = 0; s < steps; ++s) {
        for (int i = tid; i < kGrowExt * kGrowExt; i += nt) {
            const int ry = i / kGrowExt, rx = i % kGrowExt;
            uint8_t v = sd[cur][ry][rx];
            if (!v && sf[ry][rx]) {
                const float gq = sg[ry][rx];
                v = (ry > 0 && sd[cur][ry - 1][rx] && continuous(sg[ry - 1][rx], gq, tau)) ||
                    (ry + 1 < kGrowExt && sd[cur][ry + 1][rx] && continuous(sg[ry + 1][rx], gq, tau)) ||
                    (rx > 0 && sd[cur][ry][rx - 1] && continuous(sg[ry][rx - 1], gq, tau)) ||
                    (rx + 1 < kGrowExt && sd[cur][ry][rx + 1] && continuous(sg[ry][rx + 1], gq, tau));
            }
            sd[cur ^ 1][ry][rx] = v;
        }
        __syncthreads();
        cur ^= 1;
    }
    for (int i = tid; i < kGrowTile * kGrowTile; i += nt) {
        const int ry = i / kGrowTile, rx = i % kGrowTile;
        const int x = blockIdx.x * kGrowTile + rx, y = blockIdx.y * kGrowTile + ry;
        if (x < W && y < H) dst[y * W + x] = sd[cur][ry + kGrowHalo][rx + kGrowHalo];
    }
}

__global__ void __launch_bounds__(256) dilate_kernel(int H, int W, const uint8_t* __restrict__ grown,
                                                     const uint8_t* __restrict__ flags, int dilate,
                                                     uint8_t* __restrict__ dynamic, uint8_t* __restrict__ inconsistent,
                                                     float* __restrict__ stats) {
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    bool a = false, b = false;
    if (p < H * W) {
        const int x = p % W, y = p / W;
        const int ya = max(y - dilate, 0), yb = min(y + dilate, H - 1);
        const int xa = max(x - dilate, 0), xb = min(x + dilate, W - 1);
        for (int yy = ya; yy <= yb && !(a && b); ++yy)
            for (int xx = xa; xx <= xb; ++xx) {
                a = a || grown[yy * W + xx];
                b = b || (flags[yy * W + xx] & kDis);
            }
        dynamic[p] = a;
        inconsistent[p] = b;
    }
    block_count(a, &stats[4]);
    block_count(b, &stats[5]);
}

inline bool bad_size(int H, int W) { return H < 1 || W < 1 || (long long)H * W >= (1LL << 24); }

}  // namespace

}  // namespace sb

using namespace sb;

extern "C" {

SB_API int sb_dynamic_residual(int height, int width, const float* depth_sil, const float* gt_depth, float sil_thres,
                               float* residual, uint32_t* hist, float* stats, void* stream) {
    if (bad_size(height, width) || !depth_sil || !gt_depth || !residual || !hist || !stats) return SB_ERR_BAD_ARG;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    SB_CUDA_CHECK(cudaMemsetAsync(hist, 0, kBins * sizeof(uint32_t), st));
    SB_CUDA_CHECK(cudaMemsetAsync(stats, 0, SB_DYNAMIC_STATS * sizeof(float), st));
    const int HW = height * width;
    residual_kernel<<<(HW + 255) / 256, 256, 0, st>>>(HW, depth_sil, gt_depth, sil_thres, residual, hist, stats);
    SB_LAUNCH_CHECK("dynamic_residual_kernel");
    return SB_OK;
}

SB_API int sb_dynamic_scale(const uint32_t* hist, float* stats, void* stream) {
    if (!hist || !stats) return SB_ERR_BAD_ARG;
    scale_kernel<<<1, kScaleThreads, 0, static_cast<cudaStream_t>(stream)>>>(hist, stats);
    SB_LAUNCH_CHECK("dynamic_scale_kernel");
    return SB_OK;
}

SB_API int sb_dynamic_seeds(int height, int width, const float* depth_sil, const float* gt_depth,
                            const float* residual, float sil_thres, float k_high, float k_low, float r_min,
                            uint8_t* flags, uint8_t* dyn, float* stats, void* stream) {
    if (bad_size(height, width) || !depth_sil || !gt_depth || !residual || !flags || !dyn || !stats ||
        std::isnan(k_high) || std::isnan(k_low) || !(r_min >= 0.f) || std::isinf(r_min))
        return SB_ERR_BAD_ARG;
    dim3 grid((width + kSeedTile - 1) / kSeedTile, (height + kSeedTile - 1) / kSeedTile), block(kSeedTile, kSeedTile);
    seeds_kernel<<<grid, block, 0, static_cast<cudaStream_t>(stream)>>>(height, width, depth_sil, gt_depth, residual,
                                                                        sil_thres, k_high, k_low, r_min, flags, dyn,
                                                                        stats);
    SB_LAUNCH_CHECK("dynamic_seeds_kernel");
    return SB_OK;
}

SB_API int sb_dynamic_grow(int height, int width, const float* gt_depth, const uint8_t* flags, float tau, int radius,
                           uint8_t* dyn, uint8_t* tmp, void* stream) {
    if (bad_size(height, width) || !gt_depth || !flags || !dyn || !tmp || radius < 0 || !(tau >= 0.f) ||
        std::isinf(tau) || dyn == tmp)
        return SB_ERR_BAD_ARG;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int launches = (radius + kGrowHalo - 1) / kGrowHalo;
    uint8_t* bufs[2] = {dyn, tmp};
    int cur = 0;
    if (launches & 1) {                       // an odd number of ping-pong launches then ends in `dyn`
        SB_CUDA_CHECK(cudaMemcpyAsync(tmp, dyn, (size_t)height * width, cudaMemcpyDeviceToDevice, st));
        cur = 1;
    }
    dim3 grid((width + kGrowTile - 1) / kGrowTile, (height + kGrowTile - 1) / kGrowTile);
    for (int l = 0; l < launches; ++l) {
        const int steps = radius - l * kGrowHalo < kGrowHalo ? radius - l * kGrowHalo : kGrowHalo;
        grow_kernel<<<grid, 256, 0, st>>>(height, width, gt_depth, flags, tau, steps, bufs[cur], bufs[cur ^ 1]);
        SB_LAUNCH_CHECK("dynamic_grow_kernel");
        cur ^= 1;
    }
    return SB_OK;
}

SB_API int sb_dynamic_dilate(int height, int width, const uint8_t* grown, const uint8_t* flags, int dilate,
                             uint8_t* dynamic, uint8_t* inconsistent, float* stats, void* stream) {
    if (bad_size(height, width) || !grown || !flags || !dynamic || !inconsistent || !stats || dilate < 0 ||
        dilate > 64)
        return SB_ERR_BAD_ARG;
    const int HW = height * width;
    dilate_kernel<<<(HW + 255) / 256, 256, 0, static_cast<cudaStream_t>(stream)>>>(height, width, grown, flags, dilate,
                                                                                   dynamic, inconsistent, stats);
    SB_LAUNCH_CHECK("dynamic_dilate_kernel");
    return SB_OK;
}

}  // extern "C"
