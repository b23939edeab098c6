// reloc.cu -- relocalisation: RGB-D thumbnail descriptors, their retrieval scores and top-k, and the tracking health
// check (splatam_b200/reloc.py; the rules are stated in include/splatam_b200.h and restated in oracle/reloc_numpy.py).
//
//   sb_reloc_thumbnails   block means (one thread per descriptor pixel, samples in row-major order), then the 3x3
//                         binomial blur over valid pixels (one thread per descriptor value); float32, each operation
//                         rounded as written, so the result equals the numpy restatement bit for bit
//   sb_reloc_score        one CTA per database entry with the query in shared memory: two passes (means, then
//                         centred sums) in double, each thread over a strided share of the pixels, then warp shuffles,
//                         then warps in order
//   sb_reloc_topk         one CTA: k rounds of a block arg-max (higher score first, the lower index on ties)
//   sb_track_health       kHealthBlocks fixed blocks of grid-stride partial counts in double, summed in block order by
//                         one thread
#include <cmath>

#include "common.cuh"

namespace sb {

namespace {

constexpr int kThreads = 256;
constexpr int kTopkThreads = 1024;
constexpr int kHealthBlocks = SB_RELOC_HEALTH_BLOCKS;   // fixed, so the summation order does not depend on the device
constexpr float kSilThres = 0.99f;                      // a pixel is observed where the silhouette exceeds this
constexpr int kHealthRgbTerms = 11;                    // sb_track_health_rgb's partials: four counts, seven NCC sums
constexpr int kScoreTerms = 5;                          // per channel: n, n_query, then pass 1 sums q, d / pass 2 cross

inline unsigned int blocks_for(long long n) { return (unsigned int)((n + kThreads - 1) / kThreads); }

__device__ __forceinline__ bool depth_ok(float d) { return isfinite(d) && d > 0.f; }

// block means: out [B,2,h,w] (grey, depth), NaN where fewer than half of the block's s*s samples are valid
__global__ void __launch_bounds__(kThreads)
thumb_means_kernel(int B, int H, int W, int s, int h, int w, const float* __restrict__ rgb,
                   const float* __restrict__ depth, const float* __restrict__ sil, float* __restrict__ out) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long long)B * h * w) return;
    const int x = (int)(i % w), y = (int)((i / w) % h), b = (int)(i / ((long long)w * h));
    const size_t plane = (size_t)H * W;
    const float* R = rgb + (size_t)b * 3 * plane;
    const float* D = depth + (size_t)b * plane;
    const float* S = sil ? sil + (size_t)b * plane : nullptr;
    float gs = 0.f, ds = 0.f;
    int gn = 0, dn = 0;
    for (int yy = 0; yy < s; ++yy) {
        const size_t row = (size_t)(y * s + yy) * W + (size_t)x * s;
        for (int xx = 0; xx < s; ++xx) {
            const size_t p = row + xx;
            bool seen = true;
            float d = D[p];
            if (S) {
                const float sv = S[p];
                seen = sv > kSilThres;
                d = __fdiv_rn(d, sv);
            }
            const float g = grey_of(R, plane, p);
            if (seen && isfinite(g)) { gs = __fadd_rn(gs, g); ++gn; }
            if (seen && depth_ok(d)) { ds = __fadd_rn(ds, d); ++dn; }
        }
    }
    const int need = s * s;
    const size_t o = (size_t)b * 2 * h * w + (size_t)y * w + x;
    out[o] = 2 * gn >= need ? __fdiv_rn(gs, (float)gn) : NAN;
    out[o + (size_t)h * w] = 2 * dn >= need ? __fdiv_rn(ds, (float)dn) : NAN;
}

// 3x3 binomial blur over the valid (non-NaN) neighbours of each valid value: sum_k w_k v_k / sum_k w_k, neighbours in
// row-major order, weights (1 2 1) x (1 2 1)
__global__ void __launch_bounds__(kThreads)
thumb_blur_kernel(int BC, int h, int w, const float* __restrict__ src, float* __restrict__ dst) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long long)BC * h * w) return;
    const int x = (int)(i % w), y = (int)((i / w) % h);
    const float* P = src + (i / ((long long)w * h)) * (long long)h * w;
    if (isnan(P[(size_t)y * w + x])) { dst[i] = NAN; return; }
    float acc = 0.f, wsum = 0.f;
    for (int dy = -1; dy <= 1; ++dy) {
        const int yy = y + dy;
        if (yy < 0 || yy >= h) continue;
        for (int dx = -1; dx <= 1; ++dx) {
            const int xx = x + dx;
            if (xx < 0 || xx >= w) continue;
            const float v = P[(size_t)yy * w + xx];
            if (isnan(v)) continue;
            const float wt = (float)((dy == 0 ? 2 : 1) * (dx == 0 ? 2 : 1));
            acc = __fadd_rn(acc, __fmul_rn(wt, v));
            wsum = __fadd_rn(wsum, wt);
        }
    }
    dst[i] = __fdiv_rn(acc, wsum);
}

// fixed-order block sum of `n` doubles per thread into red[0..n): warp shuffles, then warps in order (thread 0)
template <int N>
__device__ __forceinline__ void block_sum(double (&v)[N], double (*red)[N]) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int k = 0; k < N; ++k) {
        double s = v[k];
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) s += __shfl_xor_sync(0xffffffffu, s, off);
        if (lane == 0) red[warp][k] = s;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int k = 0; k < N; ++k) {
            double s = 0.0;
            for (int q = 0; q < kThreads / 32; ++q) s += red[q][k];
            red[0][k] = s;
        }
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < N; ++k) v[k] = red[0][k];
    __syncthreads();
}

// zero-mean NCC of one database entry against the query (grey and depth), combined as their mean; -2 where, in some
// channel, fewer than half of the query's valid pixels (or fewer than 2) are valid in both
__global__ void __launch_bounds__(kThreads)
reloc_score_kernel(int P, const float* __restrict__ query, const float* __restrict__ db, double* __restrict__ scores) {
    extern __shared__ float sq[];                        // [2P] the query
    __shared__ double red[kThreads / 32][2 * kScoreTerms];
    for (int i = threadIdx.x; i < 2 * P; i += kThreads) sq[i] = query[i];
    __syncthreads();
    const float* d = db + (size_t)blockIdx.x * 2 * P;
    double a[2 * kScoreTerms];
#pragma unroll
    for (int k = 0; k < 2 * kScoreTerms; ++k) a[k] = 0.0;
    // pass 1: [c*5 + 0] pixels valid in both, [1] query-valid pixels, [2] sum q, [3] sum d
#pragma unroll
    for (int c = 0; c < 2; ++c) {
        for (int i = threadIdx.x; i < P; i += kThreads) {
            const float q = sq[c * P + i], v = d[(size_t)c * P + i];
            if (isnan(q)) continue;
            a[c * kScoreTerms + 1] += 1.0;
            if (isnan(v)) continue;
            a[c * kScoreTerms + 0] += 1.0;
            a[c * kScoreTerms + 2] += (double)q;
            a[c * kScoreTerms + 3] += (double)v;
        }
    }
    block_sum<2 * kScoreTerms>(a, red);
    double n[2], mq[2], md[2];
    bool ok = true;
#pragma unroll
    for (int c = 0; c < 2; ++c) {
        n[c] = a[c * kScoreTerms];
        ok = ok && a[c * kScoreTerms + 1] > 0.0 && n[c] >= 2.0 && 2.0 * n[c] >= a[c * kScoreTerms + 1];
        mq[c] = a[c * kScoreTerms + 2] / n[c];
        md[c] = a[c * kScoreTerms + 3] / n[c];
    }
    if (!ok) {                                           // uniform across the block
        if (threadIdx.x == 0) scores[blockIdx.x] = -2.0;
        return;
    }
    // pass 2: [c*5 + 2] sum (q - mq)(d - md), [3] sum (q - mq)^2, [4] sum (d - md)^2
#pragma unroll
    for (int k = 0; k < 2 * kScoreTerms; ++k) a[k] = 0.0;
#pragma unroll
    for (int c = 0; c < 2; ++c) {
        for (int i = threadIdx.x; i < P; i += kThreads) {
            const float q = sq[c * P + i], v = d[(size_t)c * P + i];
            if (isnan(q) || isnan(v)) continue;
            const double eq = (double)q - mq[c], ed = (double)v - md[c];
            a[c * kScoreTerms + 2] += eq * ed;
            a[c * kScoreTerms + 3] += eq * eq;
            a[c * kScoreTerms + 4] += ed * ed;
        }
    }
    block_sum<2 * kScoreTerms>(a, red);
    if (threadIdx.x != 0) return;
    double sc = 0.0;
#pragma unroll
    for (int c = 0; c < 2; ++c) {
        const double vq = a[c * kScoreTerms + 3], vd = a[c * kScoreTerms + 4];
        sc += (vq > 0.0 && vd > 0.0) ? a[c * kScoreTerms + 2] / sqrt(vq * vd) : 0.0;
    }
    scores[blockIdx.x] = 0.5 * sc;
}

__device__ __forceinline__ bool better(double sa, int ia, double sb, int ib) {
    return sa > sb || (sa == sb && ia < ib);
}

__global__ void __launch_bounds__(kTopkThreads)
reloc_topk_kernel(int N, int k, const double* __restrict__ scores, int* __restrict__ idx, double* __restrict__ top) {
    __shared__ double bs[kTopkThreads];
    __shared__ int bi[kTopkThreads];
    __shared__ int chosen[SB_RELOC_MAX_K];
    for (int r = 0; r < k; ++r) {
        double best = -INFINITY;
        int arg = N;                                     // N: none yet
        for (int i = threadIdx.x; i < N; i += kTopkThreads) {
            bool taken = false;
            for (int q = 0; q < r; ++q) taken = taken || chosen[q] == i;
            if (taken) continue;
            double v = scores[i];
            if (isnan(v)) v = -INFINITY;
            if (arg == N || better(v, i, best, arg)) { best = v; arg = i; }
        }
        bs[threadIdx.x] = best;
        bi[threadIdx.x] = arg;
        __syncthreads();
        for (int half = kTopkThreads / 2; half > 0; half >>= 1) {
            if (threadIdx.x < half) {
                const int o = threadIdx.x + half;
                if (bi[o] < N && (bi[threadIdx.x] >= N || better(bs[o], bi[o], bs[threadIdx.x], bi[threadIdx.x]))) {
                    bs[threadIdx.x] = bs[o];
                    bi[threadIdx.x] = bi[o];
                }
            }
            __syncthreads();
        }
        if (threadIdx.x == 0) {
            chosen[r] = bi[0];
            idx[r] = bi[0];
            top[r] = bs[0];
        }
        __syncthreads();
    }
}

// per-block partial counts: valid frame depth, covered (valid and observed by the map), inliers, sum of squared
// residuals over the covered pixels.  kMode 0: sb_track_health.  kMode 1 and 2, the two passes of
// sb_track_health_rgb's colour NCC over the inliers whose six colour values are all finite: [4] pairs, [5..8) sums of
// the map's r, g, b, [8..11) of the frame's; then, with the per-channel means from pass 1's partials (summed in block
// order), [4] sum over channels of (m - mm)(f - mf), [5] of (m - mm)^2, [6] of (f - mf)^2
template <int kMode>
__global__ void __launch_bounds__(kThreads)
health_partials_kernel(int n, const float* __restrict__ depth_sil, const float* __restrict__ frame_depth, float tau_abs,
                       float tau_rel, double* __restrict__ partials, const float* __restrict__ map_rgb,
                       const float* __restrict__ frame_rgb, const double* __restrict__ pass1) {
    constexpr int N = kMode == 0 ? 4 : kHealthRgbTerms;
    __shared__ double red[kThreads / 32][N];
    double a[N] = {0.0, 0.0, 0.0, 0.0};
    double mm[3] = {0.0, 0.0, 0.0}, mf[3] = {0.0, 0.0, 0.0};
    if constexpr (kMode == 2) {
        double s[7] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
        for (int b = 0; b < kHealthBlocks; ++b)
            for (int k = 0; k < 7; ++k) s[k] += pass1[(size_t)b * N + 4 + k];
        for (int c = 0; c < 3; ++c) {
            mm[c] = s[1 + c] / s[0];
            mf[c] = s[4 + c] / s[0];
        }
    }
    for (int i = blockIdx.x * kThreads + threadIdx.x; i < n; i += kHealthBlocks * kThreads) {
        const float df = frame_depth[i];
        if (!depth_ok(df)) continue;
        a[0] += 1.0;
        const float sil = depth_sil[n + i];
        if (!(sil > kSilThres)) continue;
        a[1] += 1.0;
        const float r = __fsub_rn(__fdiv_rn(depth_sil[i], sil), df);
        a[2] += fabsf(r) < fmaxf(tau_abs, __fmul_rn(tau_rel, df)) ? 1.0 : 0.0;
        a[3] += (double)r * (double)r;
        if constexpr (kMode != 0) {
            if (!(fabsf(r) < fmaxf(tau_abs, __fmul_rn(tau_rel, df)))) continue;
            float cm[3], cf[3];
            bool ok = true;
#pragma unroll
            for (int c = 0; c < 3; ++c) {
                cm[c] = map_rgb[(size_t)c * n + i];
                cf[c] = frame_rgb[(size_t)c * n + i];
                ok = ok && isfinite(cm[c]) && isfinite(cf[c]);
            }
            if (!ok) continue;
            if constexpr (kMode == 1) {
                a[4] += 1.0;
#pragma unroll
                for (int c = 0; c < 3; ++c) {
                    a[5 + c] += (double)cm[c];
                    a[8 + c] += (double)cf[c];
                }
            } else {
#pragma unroll
                for (int c = 0; c < 3; ++c) {
                    const double em = (double)cm[c] - mm[c], ef = (double)cf[c] - mf[c];
                    a[4] += em * ef;
                    a[5] += em * em;
                    a[6] += ef * ef;
                }
            }
        }
    }
    block_sum<N>(a, red);
    if (threadIdx.x == 0)
        for (int k = 0; k < N; ++k) partials[(size_t)blockIdx.x * N + k] = a[k];
}

__global__ void health_finish_kernel(const double* __restrict__ partials, double min_coverage, double min_inliers,
                                     double* __restrict__ stats) {
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    double s[4] = {0.0, 0.0, 0.0, 0.0};
    for (int b = 0; b < kHealthBlocks; ++b)
        for (int k = 0; k < 4; ++k) s[k] += partials[(size_t)b * 4 + k];
    stats[0] = s[0];
    stats[1] = s[1];
    stats[2] = s[2];
    stats[3] = s[1] > 0.0 ? sqrt(s[3] / s[1]) : INFINITY;
    stats[4] = (s[0] > 0.0 && s[1] > 0.0 && s[1] / s[0] >= min_coverage && s[2] / s[1] >= min_inliers) ? 1.0 : 0.0;
}

// sb_track_health_rgb's record: sb_track_health's five entries (the same sums), the NCC pairs and the colour NCC
__global__ void health_rgb_finish_kernel(const double* __restrict__ pass1, const double* __restrict__ pass2,
                                         double min_coverage, double min_inliers, double min_ncc,
                                         double* __restrict__ stats) {
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    double s[5] = {0.0, 0.0, 0.0, 0.0, 0.0}, c[3] = {0.0, 0.0, 0.0};
    for (int b = 0; b < kHealthBlocks; ++b) {
        for (int k = 0; k < 5; ++k) s[k] += pass1[(size_t)b * kHealthRgbTerms + k];
        for (int k = 0; k < 3; ++k) c[k] += pass2[(size_t)b * kHealthRgbTerms + 4 + k];
    }
    stats[0] = s[0];
    stats[1] = s[1];
    stats[2] = s[2];
    stats[3] = s[1] > 0.0 ? sqrt(s[3] / s[1]) : INFINITY;
    const bool geo = s[0] > 0.0 && s[1] > 0.0 && s[1] / s[0] >= min_coverage && s[2] / s[1] >= min_inliers;
    const double ncc = (c[1] > 0.0 && c[2] > 0.0) ? c[0] / sqrt(c[1] * c[2]) : 0.0;
    stats[5] = s[4];
    stats[6] = ncc;
    stats[4] = (geo && s[4] >= SB_RELOC_MIN_NCC_PAIRS && ncc >= min_ncc) ? 1.0 : 0.0;
}

}  // namespace

}  // namespace sb

using namespace sb;

extern "C" {

SB_API int sb_reloc_thumbnail_size(int height, int width, int* h, int* w) {
    if (height < 1 || width < 1 || !h || !w) return SB_ERR_BAD_ARG;
    const int s = height / SB_RELOC_THUMB_ROWS > 1 ? height / SB_RELOC_THUMB_ROWS : 1;
    *h = height / s;
    *w = width / s;
    return SB_OK;
}

SB_API int sb_reloc_thumbnails(int B, int height, int width, const float* rgb, const float* depth, const float* sil,
                               float* scratch, float* out, void* stream) {
    if (B < 1 || height < 1 || width < 1 || (long long)B * 3 * height * width >= (1LL << 40) || !rgb || !depth ||
        !scratch || !out)
        return SB_ERR_BAD_ARG;
    const int s = height / SB_RELOC_THUMB_ROWS > 1 ? height / SB_RELOC_THUMB_ROWS : 1;
    const int h = height / s, w = width / s;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const long long n = (long long)B * h * w;
    thumb_means_kernel<<<blocks_for(n), kThreads, 0, st>>>(B, height, width, s, h, w, rgb, depth, sil, scratch);
    SB_LAUNCH_CHECK("thumb_means_kernel");
    thumb_blur_kernel<<<blocks_for(2 * n), kThreads, 0, st>>>(2 * B, h, w, scratch, out);
    SB_LAUNCH_CHECK("thumb_blur_kernel");
    return SB_OK;
}

SB_API int sb_reloc_score(int N, int pixels, const float* query, const float* database, double* scores,
                          void* stream) {
    if (N < 1 || pixels < 1 || pixels > SB_RELOC_MAX_PIXELS || !query || !database || !scores) return SB_ERR_BAD_ARG;
    const size_t smem = (size_t)2 * pixels * sizeof(float);
    if (smem > 48 * 1024)
        SB_CUDA_CHECK(cudaFuncSetAttribute(reloc_score_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    reloc_score_kernel<<<N, kThreads, smem, static_cast<cudaStream_t>(stream)>>>(pixels, query, database, scores);
    SB_LAUNCH_CHECK("reloc_score_kernel");
    return SB_OK;
}

SB_API int sb_reloc_topk(int N, int k, const double* scores, int* indices, double* top_scores, void* stream) {
    if (N < 1 || k < 1 || k > SB_RELOC_MAX_K || k > N || !scores || !indices || !top_scores) return SB_ERR_BAD_ARG;
    reloc_topk_kernel<<<1, kTopkThreads, 0, static_cast<cudaStream_t>(stream)>>>(N, k, scores, indices, top_scores);
    SB_LAUNCH_CHECK("reloc_topk_kernel");
    return SB_OK;
}

SB_API int sb_track_health(int height, int width, const float* depth_sil, const float* frame_depth, float tau_abs,
                           float tau_rel, double min_coverage, double min_inliers, double* scratch, double* stats,
                           void* stream) {
    if (height < 1 || width < 1 || (long long)height * width >= (1LL << 31) || !depth_sil || !frame_depth ||
        !scratch || !stats || !(std::isfinite(tau_abs) && tau_abs >= 0.f) || !(std::isfinite(tau_rel) && tau_rel >= 0.f)
        || !(min_coverage >= 0.0 && min_coverage <= 1.0) || !(min_inliers >= 0.0 && min_inliers <= 1.0))
        return SB_ERR_BAD_ARG;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    health_partials_kernel<0><<<kHealthBlocks, kThreads, 0, st>>>(height * width, depth_sil, frame_depth, tau_abs,
                                                                  tau_rel, scratch, nullptr, nullptr, nullptr);
    SB_LAUNCH_CHECK("health_partials_kernel");
    health_finish_kernel<<<1, 1, 0, st>>>(scratch, min_coverage, min_inliers, stats);
    SB_LAUNCH_CHECK("health_finish_kernel");
    return SB_OK;
}

SB_API int sb_track_health_rgb(int height, int width, const float* depth_sil, const float* frame_depth,
                               const float* map_rgb, const float* frame_rgb, float tau_abs, float tau_rel,
                               double min_coverage, double min_inliers, double min_ncc, double* scratch, double* stats,
                               void* stream) {
    if (height < 1 || width < 1 || (long long)height * width >= (1LL << 31) || !depth_sil || !frame_depth ||
        !map_rgb || !frame_rgb || !scratch || !stats || !(std::isfinite(tau_abs) && tau_abs >= 0.f) ||
        !(std::isfinite(tau_rel) && tau_rel >= 0.f) || !(min_coverage >= 0.0 && min_coverage <= 1.0) ||
        !(min_inliers >= 0.0 && min_inliers <= 1.0) || !(min_ncc >= -1.0 && min_ncc <= 1.0))
        return SB_ERR_BAD_ARG;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    double* pass1 = scratch;
    double* pass2 = scratch + (size_t)kHealthRgbTerms * kHealthBlocks;
    const int n = height * width;
    health_partials_kernel<1><<<kHealthBlocks, kThreads, 0, st>>>(n, depth_sil, frame_depth, tau_abs, tau_rel, pass1,
                                                                  map_rgb, frame_rgb, nullptr);
    SB_LAUNCH_CHECK("health_partials_kernel");
    health_partials_kernel<2><<<kHealthBlocks, kThreads, 0, st>>>(n, depth_sil, frame_depth, tau_abs, tau_rel, pass2,
                                                                  map_rgb, frame_rgb, pass1);
    SB_LAUNCH_CHECK("health_partials_kernel");
    health_rgb_finish_kernel<<<1, 1, 0, st>>>(pass1, pass2, min_coverage, min_inliers, min_ncc, stats);
    SB_LAUNCH_CHECK("health_rgb_finish_kernel");
    return SB_OK;
}

}  // extern "C"
