// eval_metrics.cu -- SplaTAM's final evaluation metrics (R/utils/eval_helpers.py:408-623, SURVEY.md section 8(f)
// row N4) as forward-only kernels:
//   * per-frame masked PSNR and depth errors in one pass over the pixels, which also writes the two weighted images
//     that MS-SSIM compares (eval_helpers.py:463-505, calc_psnr R/utils/slam_external.py:49-51);
//   * MS-SSIM as pytorch_msssim.ms_ssim defines it (eval_helpers.py:482): 5 levels of an 11-tap sigma-1.5 Gaussian
//     filtered SSIM with a VALID window, a 2x2 average pool (zero padding counted) between levels.
// Both are deterministic: every block writes its own partial sums and one block reduces them in a fixed order; no
// float atomics.  The MS-SSIM moments, maps and pyramid are double, so the result follows the float64 definition
// (oracle/metrics_torch.py) instead of inheriting float32 cancellation in E[x^2] - mu^2.
#include "common.cuh"

namespace sb {

namespace {

// ---- frame metrics ---------------------------------------------------------------------------------------------
// partial row per block: squared error of the three weighted channels, sum sqrt(e^2)*valid, sum |e|*valid,
// sum valid, sum mask (the weighting mask: presence*valid or valid)
constexpr int kFrameCols = 7;
constexpr int kFrameStride = 8;
constexpr int kFrameThreads = 256;
constexpr int kFrameMaxBlocks = 528;    // 132 SMs x 4

int frame_blocks(int HW) { return (HW + kFrameThreads - 1) / kFrameThreads < kFrameMaxBlocks
                                      ? (HW + kFrameThreads - 1) / kFrameThreads : kFrameMaxBlocks; }

__global__ void __launch_bounds__(kFrameThreads)
frame_metrics_kernel(const float* __restrict__ im, const float* __restrict__ depth_sil, const float* __restrict__ gt_im,
                     const float* __restrict__ gt_depth, int HW, float sil_thres, int use_presence,
                     float* __restrict__ w_im, float* __restrict__ w_gt, double* __restrict__ partials) {
    __shared__ double red[kFrameThreads / 32];
    double acc[kFrameCols] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
    for (int p = blockIdx.x * blockDim.x + threadIdx.x; p < HW; p += gridDim.x * blockDim.x) {
        const float gd = gt_depth[p];
        const float valid = gd > 0.f ? 1.f : 0.f;
        const float pres = depth_sil[HW + p] > sil_thres ? 1.f : 0.f;
        const float m = use_presence ? pres * valid : valid;
        // the reference multiplies by the masks (0 * inf = NaN propagates as it does there)
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            const float a = im[c * HW + p] * m, b = gt_im[c * HW + p] * m;
            w_im[c * HW + p] = a;
            w_gt[c * HW + p] = b;
            const float d = a - b;
            acc[c] += (double)(d * d);
        }
        // rastered_depth = depth * valid; e = (rastered_depth - gt) [* presence]
        const float e = use_presence ? (depth_sil[p] * valid - gd) * pres : depth_sil[p] * valid - gd;
        acc[3] += (double)(sqrtf(e * e) * valid);
        acc[4] += (double)(fabsf(e) * valid);
        acc[5] += (double)valid;
        acc[6] += (double)m;
    }
#pragma unroll
    for (int k = 0; k < kFrameCols; ++k) {
        const double s = block_sum<kFrameThreads>(acc[k], red, threadIdx.x);
        if (threadIdx.x == 0) partials[(size_t)blockIdx.x * kFrameStride + k] = s;
    }
}

// one block: metrics = {psnr, depth_rmse, depth_l1, n_valid, n_mask}
__global__ void __launch_bounds__(kFrameThreads)
frame_metrics_finalize_kernel(const double* __restrict__ partials, int nblocks, int HW, double* __restrict__ metrics) {
    __shared__ double red[kFrameThreads / 32];
    __shared__ double tot[kFrameCols];
    for (int k = 0; k < kFrameCols; ++k) {
        double v = 0.0;
        for (int b = threadIdx.x; b < nblocks; b += blockDim.x) v += partials[(size_t)b * kFrameStride + k];
        const double s = block_sum<kFrameThreads>(v, red, threadIdx.x);
        if (threadIdx.x == 0) tot[k] = s;
    }
    if (threadIdx.x == 0) {
        double psnr = 0.0;
        for (int c = 0; c < 3; ++c) psnr += 20.0 * log10(1.0 / sqrt(tot[c] / (double)HW));
        metrics[0] = psnr / 3.0;
        metrics[1] = tot[3] / tot[5];
        metrics[2] = tot[4] / tot[5];
        metrics[3] = tot[5];
        metrics[4] = tot[6];
    }
}

// ---- MS-SSIM -----------------------------------------------------------------------------------------------------
constexpr int kLevels = 5;
constexpr int kMinSide = 161;                       // pytorch_msssim: smaller side > (11 - 1) * 2^4
constexpr int kTW = 32, kTH = 8, kWin = 11;         // output tile 32x8, valid 11-tap separable Gaussian
constexpr int kPW = kTW + kWin - 1, kPH = kTH + kWin - 1;
constexpr int kLevelThreads = kTW * kTH;
struct MsWin { double w[kWin]; };
struct MsWeights { double w[kLevels]; };

int level_blocks_x(int W) { return (W - kWin + 1 + kTW - 1) / kTW; }
int level_blocks_y(int H) { return (H - kWin + 1 + kTH - 1) / kTH; }

// One level: the five filtered moments of an output tile in double, cs and ssim maps, their tile sums into
// partials[(plane * nblk + block) * 2 + {0: cs, 1: ssim}].
template <typename T>
__global__ void __launch_bounds__(kLevelThreads)
ms_ssim_level_kernel(const T* __restrict__ x, const T* __restrict__ y, int H, int W, const MsWin win, double C1,
                     double C2, double* __restrict__ partials) {
    __shared__ double sx[kPH][kPW], sy[kPH][kPW];
    __shared__ double h[5][kPH][kTW];
    __shared__ double red[kLevelThreads / 32];
    const int plane = blockIdx.z, x0 = blockIdx.x * kTW, y0 = blockIdx.y * kTH;
    const int Ho = H - kWin + 1, Wo = W - kWin + 1;
    const T* xc = x + (size_t)plane * H * W;
    const T* yc = y + (size_t)plane * H * W;
    const int tid = threadIdx.y * kTW + threadIdx.x;
    for (int i = tid; i < kPH * kPW; i += kLevelThreads) {
        const int r = i / kPW, q = i % kPW, gy = y0 + r, gx = x0 + q;
        const bool in = gy < H && gx < W;            // only feeds outputs that are discarded when false
        sx[r][q] = in ? (double)xc[(size_t)gy * W + gx] : 0.0;
        sy[r][q] = in ? (double)yc[(size_t)gy * W + gx] : 0.0;
    }
    __syncthreads();
    for (int i = tid; i < kPH * kTW; i += kLevelThreads) {
        const int r = i / kTW, q = i % kTW;
        double a = 0.0, b = 0.0, aa = 0.0, bb = 0.0, ab = 0.0;
#pragma unroll
        for (int k = 0; k < kWin; ++k) {
            const double w = win.w[k], xv = sx[r][q + k], yv = sy[r][q + k];
            a = fma(w, xv, a); b = fma(w, yv, b);
            aa = fma(w, xv * xv, aa); bb = fma(w, yv * yv, bb); ab = fma(w, xv * yv, ab);
        }
        h[0][r][q] = a; h[1][r][q] = b; h[2][r][q] = aa; h[3][r][q] = bb; h[4][r][q] = ab;
    }
    __syncthreads();
    const int px = x0 + threadIdx.x, py = y0 + threadIdx.y;
    double cs = 0.0, ss = 0.0;
    if (px < Wo && py < Ho) {
        double mu1 = 0.0, mu2 = 0.0, e11 = 0.0, e22 = 0.0, e12 = 0.0;
#pragma unroll
        for (int k = 0; k < kWin; ++k) {
            const double w = win.w[k];
            mu1 = fma(w, h[0][threadIdx.y + k][threadIdx.x], mu1);
            mu2 = fma(w, h[1][threadIdx.y + k][threadIdx.x], mu2);
            e11 = fma(w, h[2][threadIdx.y + k][threadIdx.x], e11);
            e22 = fma(w, h[3][threadIdx.y + k][threadIdx.x], e22);
            e12 = fma(w, h[4][threadIdx.y + k][threadIdx.x], e12);
        }
        const double m11 = mu1 * mu1, m22 = mu2 * mu2, m12 = mu1 * mu2;
        const double s1 = e11 - m11, s2 = e22 - m22, s12 = e12 - m12;
        cs = (2.0 * s12 + C2) / (s1 + s2 + C2);
        ss = (2.0 * m12 + C1) / (m11 + m22 + C1) * cs;
    }
    const double tcs = block_sum<kLevelThreads>(cs, red, tid);
    const double tss = block_sum<kLevelThreads>(ss, red, tid);
    if (tid == 0) {
        const size_t blk = (size_t)blockIdx.y * gridDim.x + blockIdx.x;
        const size_t o = ((size_t)plane * gridDim.x * gridDim.y + blk) * 2;
        partials[o] = tcs;
        partials[o + 1] = tss;
    }
}

// F.avg_pool2d(kernel 2, stride 2, padding (H % 2, W % 2)), zero padding counted: every output divides by 4.
template <typename T>
__global__ void __launch_bounds__(256)
ms_ssim_pool_kernel(const T* __restrict__ x, const T* __restrict__ y, int NC, int H, int W, int Hn, int Wn,
                    double* __restrict__ xo, double* __restrict__ yo) {
    const int pH = H & 1, pW = W & 1;
    const size_t n = (size_t)NC * Hn * Wn;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const int j = (int)(i % Wn), r = (int)((i / Wn) % Hn);
        const size_t plane = i / ((size_t)Hn * Wn);
        const T* xc = x + plane * H * W;
        const T* yc = y + plane * H * W;
        double a = 0.0, b = 0.0;
#pragma unroll
        for (int dy = 0; dy < 2; ++dy)
#pragma unroll
            for (int dx = 0; dx < 2; ++dx) {
                const int gy = 2 * r - pH + dy, gx = 2 * j - pW + dx;
                if (gy >= 0 && gy < H && gx >= 0 && gx < W) {
                    a += (double)xc[(size_t)gy * W + gx];
                    b += (double)yc[(size_t)gy * W + gx];
                }
            }
        xo[i] = a * 0.25;
        yo[i] = b * 0.25;
    }
}

struct MsLevels {
    int H[kLevels], W[kLevels], nblk[kLevels];
    size_t part_off[kLevels];   // offset (doubles) of each level's partials
};

MsLevels ms_levels(int NC, int H, int W) {
    MsLevels L;
    size_t off = 0;
    for (int l = 0; l < kLevels; ++l) {
        L.H[l] = H; L.W[l] = W;
        L.nblk[l] = level_blocks_x(W) * level_blocks_y(H);
        L.part_off[l] = off;
        off += (size_t)NC * L.nblk[l] * 2;
        H = H / 2 + (H & 1);      // (H + 2 * (H % 2) - 2) / 2 + 1
        W = W / 2 + (W & 1);
    }
    return L;
}

// one block: per-plane prod(relu(cs_l)^w_l, l < 4) * relu(ssim_4)^w_4, and their mean
__global__ void __launch_bounds__(kLevelThreads)
ms_ssim_finalize_kernel(const double* __restrict__ partials, int NC, const MsLevels L, const MsWeights wt,
                        double* __restrict__ per_plane, double* __restrict__ mean) {
    __shared__ double red[kLevelThreads / 32];
    const int tid = threadIdx.x;
    double total = 0.0;
    for (int p = 0; p < NC; ++p) {
        double val = 1.0;
        for (int l = 0; l < kLevels; ++l) {
            const int nb = L.nblk[l];
            const double* part = partials + L.part_off[l] + (size_t)p * nb * 2 + (l < kLevels - 1 ? 0 : 1);
            double v = 0.0;
            for (int b = tid; b < nb; b += blockDim.x) v += part[(size_t)b * 2];
            const double s = block_sum<kLevelThreads>(v, red, tid);
            if (tid == 0) {
                const double m = s / ((double)(L.H[l] - kWin + 1) * (double)(L.W[l] - kWin + 1));
                val *= pow(m > 0.0 ? m : 0.0, wt.w[l]);
            }
        }
        if (tid == 0) {
            if (per_plane) per_plane[p] = val;
            total += val;
        }
    }
    if (tid == 0 && mean) *mean = total / (double)NC;
}

size_t ms_ssim_bytes(int NC, int H, int W, MsLevels* out, double** xs, double** ys, double** partials, void* ws) {
    const MsLevels L = ms_levels(NC, H, W);
    Carver c(ws);
    for (int l = 1; l < kLevels; ++l) {
        const size_t n = (size_t)NC * L.H[l] * L.W[l];
        double* a = c.take<double>(n);
        double* b = c.take<double>(n);
        if (xs) { xs[l] = a; ys[l] = b; }
    }
    double* part = c.take<double>(L.part_off[kLevels - 1] + (size_t)NC * L.nblk[kLevels - 1] * 2);
    if (partials) *partials = part;
    if (out) *out = L;
    return c.used();
}

bool ms_ssim_args_ok(int N, int C, int H, int W) {
    return N >= 1 && C >= 1 && H >= kMinSide && W >= kMinSide && (long long)N * C * H * W < (1LL << 40);
}

}  // namespace

}  // namespace sb

using namespace sb;

extern "C" {

SB_API int sb_frame_metrics_workspace_bytes(int H, int W, size_t* bytes) {
    if (!bytes || H < 1 || W < 1) return SB_ERR_BAD_ARG;
    *bytes = (size_t)frame_blocks(H * W) * kFrameStride * sizeof(double);
    return SB_OK;
}

SB_API int sb_frame_metrics(const float* im, const float* depth_sil, const float* gt_im, const float* gt_depth, int H,
                            int W, float sil_thres, int use_presence, float* weighted_im, float* weighted_gt,
                            void* workspace, size_t workspace_bytes, double* metrics, void* stream) {
    if (!im || !depth_sil || !gt_im || !gt_depth || !weighted_im || !weighted_gt || !workspace || !metrics || H < 1 ||
        W < 1 || (long long)H * W >= (1LL << 31) / 3)
        return SB_ERR_BAD_ARG;
    const int HW = H * W, G = frame_blocks(HW);
    if (workspace_bytes < (size_t)G * kFrameStride * sizeof(double)) return SB_ERR_WORKSPACE;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    double* partials = static_cast<double*>(workspace);
    frame_metrics_kernel<<<G, kFrameThreads, 0, st>>>(im, depth_sil, gt_im, gt_depth, HW, sil_thres, use_presence,
                                                      weighted_im, weighted_gt, partials);
    SB_LAUNCH_CHECK("frame_metrics_kernel");
    frame_metrics_finalize_kernel<<<1, kFrameThreads, 0, st>>>(partials, G, HW, metrics);
    SB_LAUNCH_CHECK("frame_metrics_finalize_kernel");
    return SB_OK;
}

SB_API int sb_ms_ssim_workspace_bytes(int N, int C, int H, int W, size_t* bytes) {
    if (!bytes || !ms_ssim_args_ok(N, C, H, W)) return SB_ERR_BAD_ARG;
    *bytes = ms_ssim_bytes(N * C, H, W, nullptr, nullptr, nullptr, nullptr, nullptr);
    return SB_OK;
}

SB_API int sb_ms_ssim(const float* x, const float* y, int N, int C, int H, int W, double data_range, void* workspace,
                      size_t workspace_bytes, double* per_channel, double* mean, void* stream) {
    if (!x || !y || !workspace || (!per_channel && !mean) || !ms_ssim_args_ok(N, C, H, W)) return SB_ERR_BAD_ARG;
    const int NC = N * C;
    MsLevels L;
    double* xs[kLevels] = {nullptr};
    double* ys[kLevels] = {nullptr};
    double* partials = nullptr;
    if (workspace_bytes < ms_ssim_bytes(NC, H, W, &L, xs, ys, &partials, workspace)) return SB_ERR_WORKSPACE;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    // the window of pytorch_msssim._fspecial_gauss_1d(11, 1.5), normalised, in double
    MsWin win;
    double wsum = 0.0;
    for (int k = 0; k < kWin; ++k) { win.w[k] = exp(-(double)((k - 5) * (k - 5)) / (2.0 * 1.5 * 1.5)); wsum += win.w[k]; }
    for (int k = 0; k < kWin; ++k) win.w[k] /= wsum;
    const MsWeights wt = {{0.0448, 0.2856, 0.3001, 0.2363, 0.1333}};
    const double C1 = (0.01 * data_range) * (0.01 * data_range), C2 = (0.03 * data_range) * (0.03 * data_range);
    for (int l = 0; l < kLevels; ++l) {
        dim3 grid(level_blocks_x(L.W[l]), level_blocks_y(L.H[l]), NC), block(kTW, kTH);
        double* part = partials + L.part_off[l];
        if (l == 0)
            ms_ssim_level_kernel<float><<<grid, block, 0, st>>>(x, y, L.H[l], L.W[l], win, C1, C2, part);
        else
            ms_ssim_level_kernel<double><<<grid, block, 0, st>>>(xs[l], ys[l], L.H[l], L.W[l], win, C1, C2, part);
        SB_LAUNCH_CHECK("ms_ssim_level_kernel");
        if (l == kLevels - 1) break;
        const size_t n = (size_t)NC * L.H[l + 1] * L.W[l + 1];
        const unsigned blocks = (unsigned)((n + 255) / 256 < 1056 ? (n + 255) / 256 : 1056);
        if (l == 0)
            ms_ssim_pool_kernel<float><<<blocks, 256, 0, st>>>(x, y, NC, L.H[l], L.W[l], L.H[l + 1], L.W[l + 1],
                                                               xs[l + 1], ys[l + 1]);
        else
            ms_ssim_pool_kernel<double><<<blocks, 256, 0, st>>>(xs[l], ys[l], NC, L.H[l], L.W[l], L.H[l + 1],
                                                                L.W[l + 1], xs[l + 1], ys[l + 1]);
        SB_LAUNCH_CHECK("ms_ssim_pool_kernel");
    }
    ms_ssim_finalize_kernel<<<1, kLevelThreads, 0, st>>>(partials, NC, L, wt, per_channel, mean);
    SB_LAUNCH_CHECK("ms_ssim_finalize_kernel");
    return SB_OK;
}

}  // extern "C"
