// lpips.cu -- LPIPS v0.1 with the AlexNet backbone, as SplaTAM's evaluation calls it through torchmetrics
// (LearnedPerceptualImagePatchSimilarity(net_type='alex', normalize=True) on the clamped weighted images,
// R/utils/eval_helpers.py:484-485, 730-731), forward only:
//   * the five ReLU convolutions of torchvision's AlexNet as implicit GEMMs (M = images x output pixels, N = Cout,
//     K = Cin*kh*kw) in FP32 FFMA with FP32 accumulation, bias and ReLU in the epilogue; conv1's gather fuses
//     clamp(x, 0, 1), 2x - 1 and the per-channel scaling layer;
//   * the 3x3 stride-2 max-pools after conv1 and conv2 as a small kernel of their own (f1 and f2 are kept unpooled,
//     the heads read them);
//   * one head kernel per layer: both feature vectors unit-normalised over channels, the linear head's weighted
//     squared difference, per-block double partials; one block reduces them in a fixed order.
// x and y run as one batch of 2N images.  No atomics and no split-K: every output has one fixed summation order, so
// repeated calls are bit-identical, and identical images give exactly 0.
#include "common.cuh"

namespace sb {

namespace {

constexpr int kLayers = 5;
constexpr int kMinSide = 31;                 // the smallest side whose second max-pool has an output
// torchmetrics' feature normalisation: f / sqrt(kNormEps + sum_c f^2)
constexpr double kNormEps = 1e-8;

struct ConvSpec { int cin, cout, ks, stride, pad; };
// torchvision alexnet features.{0,3,6,8,10}
constexpr ConvSpec kConv[kLayers] = {{3, 64, 11, 4, 2}, {64, 192, 5, 1, 2}, {192, 384, 3, 1, 1},
                                     {384, 256, 3, 1, 1}, {256, 256, 3, 1, 1}};

// the scaling layer of lpips / torchmetrics (ScalingLayer): (x - shift) / scale per channel
__constant__ float c_shift[3] = {-0.030f, -0.088f, -0.188f};
__constant__ float c_scale[3] = {0.458f, 0.448f, 0.450f};

// ---- convolution: implicit GEMM ------------------------------------------------------------------------------------
// Block tile 128 (output pixels) x 64 (output channels) x 8 (K), 256 threads, each 8 x 4 outputs; shared tiles are
// double-buffered and the next K slice is fetched into registers while the current one is multiplied.
constexpr int kBM = 128, kBN = 64, kBK = 8, kConvThreads = 256;

// in: [B, Cin, H, W]; images n < n_split are read from in0 (+ n), the rest from in1 (+ n - n_split).
// wk: [K][Cout] (k = (ci * KS + ky) * KS + kx), bias [Cout]; out: [B, Cout, OH, OW] = relu(conv + bias).
template <int KS, int STRIDE, int PAD, bool INPUT>
__global__ void __launch_bounds__(kConvThreads, 2)
conv_relu_kernel(const float* __restrict__ in0, const float* __restrict__ in1, int n_split, int Cin, int H, int W,
                 int OH, int OW, int M, int Cout, const float* __restrict__ wk, const float* __restrict__ bias,
                 float* __restrict__ out) {
    __shared__ __align__(16) float As[2][kBK][kBM];
    __shared__ __align__(16) float Bs[2][kBK][kBN];
    constexpr int KK = KS * KS;
    const int K = Cin * KK;
    const int tid = threadIdx.x;
    const int m0 = blockIdx.x * kBM, n0 = blockIdx.y * kBN;
    const int OHW = OH * OW;

    // the output pixel whose input patch this thread gathers (A rows ak, ak + 2, ak + 4, ak + 6 of every K slice)
    const int am = m0 + (tid & (kBM - 1)), ak = tid >> 7;
    const bool a_ok = am < M;
    int iy0 = 0, ix0 = 0;
    const float* src = in0;
    if (a_ok) {
        const int n = am / OHW, pix = am - n * OHW, oy = pix / OW, ox = pix - oy * OW;
        iy0 = oy * STRIDE - PAD;
        ix0 = ox * STRIDE - PAD;
        src = n < n_split ? in0 + (size_t)n * Cin * H * W : in1 + (size_t)(n - n_split) * Cin * H * W;
    }
    const int bk = tid / kBN, bn = tid % kBN;    // B rows bk, bk + 4 of every K slice, column bn

    float ra[4], rb[2];
    auto fetch = [&](int k0) {
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int k = k0 + ak + 2 * j;
            float v = 0.f;                       // zero padding and the K tail
            if (a_ok && k < K) {
                const int ci = k / KK, r = k - ci * KK, ky = r / KS, kx = r - ky * KS;
                const int iy = iy0 + ky, ix = ix0 + kx;
                if ((unsigned)iy < (unsigned)H && (unsigned)ix < (unsigned)W) {
                    v = __ldg(src + ((size_t)ci * H + iy) * W + ix);
                    if (INPUT) {
                        v = v < 0.f ? 0.f : (v > 1.f ? 1.f : v);            // clamp (a NaN stays NaN)
                        v = (2.f * v - 1.f - c_shift[ci]) / c_scale[ci];
                    }
                }
            }
            ra[j] = v;
        }
#pragma unroll
        for (int j = 0; j < 2; ++j) {
            const int k = k0 + bk + 4 * j;
            rb[j] = k < K ? __ldg(wk + (size_t)k * Cout + n0 + bn) : 0.f;
        }
    };
    auto stash = [&](int buf) {
#pragma unroll
        for (int j = 0; j < 4; ++j) As[buf][ak + 2 * j][tid & (kBM - 1)] = ra[j];
#pragma unroll
        for (int j = 0; j < 2; ++j) Bs[buf][bk + 4 * j][bn] = rb[j];
    };

    // thread (tx, ty) owns output pixels m0 + tx*4 + {0..3} and m0 + 64 + tx*4 + {0..3}, channels n0 + ty*4 + {0..3}
    const int tx = tid & 15, ty = tid >> 4;
    float acc[8][4];
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

    const int nt = (K + kBK - 1) / kBK;
    fetch(0);
    stash(0);
    __syncthreads();
    for (int t = 0; t < nt; ++t) {
        const int buf = t & 1;
        if (t + 1 < nt) fetch((t + 1) * kBK);
#pragma unroll
        for (int kk = 0; kk < kBK; ++kk) {
            const float4 a0 = *reinterpret_cast<const float4*>(&As[buf][kk][tx * 4]);
            const float4 a1 = *reinterpret_cast<const float4*>(&As[buf][kk][64 + tx * 4]);
            const float4 b = *reinterpret_cast<const float4*>(&Bs[buf][kk][ty * 4]);
            const float a[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
            const float bb[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
            for (int i = 0; i < 8; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], bb[j], acc[i][j]);
        }
        if (t + 1 < nt) stash(buf ^ 1);
        __syncthreads();
    }

#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const int m = m0 + (i < 4 ? tx * 4 + i : 64 + tx * 4 + i - 4);
        if (m >= M) continue;
        const int n = m / OHW, pix = m - n * OHW;
        float* o = out + (size_t)n * Cout * OHW + pix;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int co = n0 + ty * 4 + j;
            const float v = acc[i][j] + __ldg(bias + co);
            o[(size_t)co * OHW] = v < 0.f ? 0.f : v;                        // relu (a NaN stays NaN)
        }
    }
}

// F.max_pool2d(kernel 3, stride 2), no padding, floor mode: every window lies inside the input.
__global__ void __launch_bounds__(256)
maxpool_kernel(const float* __restrict__ in, int planes, int H, int W, int OH, int OW, float* __restrict__ out) {
    const size_t n = (size_t)planes * OH * OW;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const int ox = (int)(i % OW), oy = (int)((i / OW) % OH);
        const float* p = in + (i / ((size_t)OH * OW)) * H * W + (size_t)(2 * oy) * W + 2 * ox;
        float m = p[0];
#pragma unroll
        for (int dy = 0; dy < 3; ++dy)
#pragma unroll
            for (int dx = 0; dx < 3; ++dx) {
                const float v = p[dy * W + dx];
                if (!(v <= m)) m = v;                                       // a NaN wins, as in torch
            }
        out[i] = m;
    }
}

// ---- heads ---------------------------------------------------------------------------------------------------------
// A block covers 32 pixels (one per lane) and splits the channels over its 8 warps (c = warp, warp + 8, ...): the
// deep layers have few pixels (3034 at 1200x680), so one thread per pixel would leave most SMs idle.
constexpr int kHeadPix = 32, kHeadGroups = 8, kHeadThreads = kHeadPix * kHeadGroups;

// f: [2N, C, P] features of one layer (x images first); partials[i * gridDim.x + block] = this block's sum over its
// pixels of d = sum_c lin[c] * (fx / |fx| - fy / |fy|)^2, |f| = sqrt(kNormEps + sum_c f^2), in double.
__global__ void __launch_bounds__(kHeadThreads)
lpips_head_kernel(const float* __restrict__ f, int N, int C, int P, const float* __restrict__ lin,
                  double* __restrict__ partials) {
    __shared__ double sq[2][kHeadGroups][kHeadPix];
    __shared__ double red[kHeadThreads / 32];
    const int lane = threadIdx.x % kHeadPix, grp = threadIdx.x / kHeadPix;
    const int i = blockIdx.y, p = blockIdx.x * kHeadPix + lane;
    const bool ok = p < P;
    const float* fx = f + (size_t)i * C * P + p;
    const float* fy = f + (size_t)(N + i) * C * P + p;
    double sx = 0.0, sy = 0.0;
    if (ok)
        for (int c = grp; c < C; c += kHeadGroups) {
            const double a = fx[(size_t)c * P], b = fy[(size_t)c * P];
            sx = fma(a, a, sx);
            sy = fma(b, b, sy);
        }
    sq[0][grp][lane] = sx;
    sq[1][grp][lane] = sy;
    __syncthreads();
    sx = 0.0;
    sy = 0.0;
    for (int g = 0; g < kHeadGroups; ++g) {      // the same order in every warp: x and y norms agree bit for bit
        sx += sq[0][g][lane];
        sy += sq[1][g][lane];
    }
    const double nx = sqrt(kNormEps + sx), ny = sqrt(kNormEps + sy);
    double d = 0.0;
    if (ok)
        for (int c = grp; c < C; c += kHeadGroups) {
            const double e = (double)fx[(size_t)c * P] / nx - (double)fy[(size_t)c * P] / ny;
            d = fma((double)lin[c], e * e, d);
        }
    const double s = block_sum<kHeadThreads>(d, red, threadIdx.x);
    if (threadIdx.x == 0) partials[(size_t)i * gridDim.x + blockIdx.x] = s;
}

struct HeadDims {
    int P[kLayers], nblk[kLayers];
    size_t part_off[kLayers];                // offset (doubles) of each layer's [N][nblk] partials
};

// one block: per_image[i] = sum over layers of (sum of the layer's partials of pair i) / P, mean = their average
__global__ void __launch_bounds__(kHeadThreads)
lpips_finalize_kernel(const double* __restrict__ partials, int N, const HeadDims D, double* __restrict__ per_image,
                      double* __restrict__ mean) {
    __shared__ double red[kHeadThreads / 32];
    const int tid = threadIdx.x;
    double total = 0.0;
    for (int i = 0; i < N; ++i) {
        double val = 0.0;
        for (int l = 0; l < kLayers; ++l) {
            const double* part = partials + D.part_off[l] + (size_t)i * D.nblk[l];
            double v = 0.0;
            for (int b = tid; b < D.nblk[l]; b += kHeadThreads) v += part[b];
            const double s = block_sum<kHeadThreads>(v, red, tid);
            if (tid == 0) val += s / (double)D.P[l];
        }
        if (tid == 0) {
            if (per_image) per_image[i] = val;
            total += val;
        }
    }
    if (tid == 0 && mean) *mean = total / (double)N;
}

// ---- plan: feature sizes, workspace carving, packed weight offsets -------------------------------------------------
struct Plan {
    int H1, W1, Hp1, Wp1, Hp2, Wp2;          // conv1 output; after pool 1 (conv2); after pool 2 (conv3..5)
    float* f[kLayers];                       // relu(conv_l) [2N, Cout_l, ...]
    float* pool1;                            // [2N, 64, Hp1, Wp1]
    float* pool2;                            // [2N, 192, Hp2, Wp2]
    double* partials;
    HeadDims D;
    size_t bytes;
};

bool args_ok(int N, int H, int W) {
    if (N < 1 || H < kMinSide || W < kMinSide) return false;
    const long long H1 = (H + 4 - 11) / 4 + 1, W1 = (W + 4 - 11) / 4 + 1;
    return 2LL * N * 64 * H1 * W1 < (1LL << 31) && 2LL * N * 3 * H * W < (1LL << 31);
}

Plan make_plan(int N, int H, int W, void* ws) {
    Plan p;
    p.H1 = (H + 2 * kConv[0].pad - kConv[0].ks) / kConv[0].stride + 1;
    p.W1 = (W + 2 * kConv[0].pad - kConv[0].ks) / kConv[0].stride + 1;
    p.Hp1 = (p.H1 - 3) / 2 + 1; p.Wp1 = (p.W1 - 3) / 2 + 1;
    p.Hp2 = (p.Hp1 - 3) / 2 + 1; p.Wp2 = (p.Wp1 - 3) / 2 + 1;
    const size_t B = 2 * (size_t)N;
    const int P[kLayers] = {p.H1 * p.W1, p.Hp1 * p.Wp1, p.Hp2 * p.Wp2, p.Hp2 * p.Wp2, p.Hp2 * p.Wp2};
    Carver c(ws);
    for (int l = 0; l < kLayers; ++l) p.f[l] = c.take<float>(B * kConv[l].cout * P[l]);
    p.pool1 = c.take<float>(B * kConv[0].cout * P[1]);
    p.pool2 = c.take<float>(B * kConv[1].cout * P[2]);
    size_t off = 0;
    for (int l = 0; l < kLayers; ++l) {
        p.D.P[l] = P[l];
        p.D.nblk[l] = (P[l] + kHeadPix - 1) / kHeadPix;
        p.D.part_off[l] = off;
        off += (size_t)N * p.D.nblk[l];
    }
    p.partials = c.take<double>(off);
    p.bytes = c.used();
    return p;
}

// packed weights: for l = 0..4 the conv weight as [K_l][Cout_l] then its bias [Cout_l]; then lin_0 .. lin_4 [Cout_l]
struct WeightOffsets { size_t w[kLayers], b[kLayers], lin[kLayers], total; };

WeightOffsets weight_offsets() {
    WeightOffsets o;
    size_t off = 0;
    for (int l = 0; l < kLayers; ++l) {
        const ConvSpec& s = kConv[l];
        o.w[l] = off;
        off += (size_t)s.cin * s.ks * s.ks * s.cout;
        o.b[l] = off;
        off += s.cout;
    }
    for (int l = 0; l < kLayers; ++l) { o.lin[l] = off; off += kConv[l].cout; }
    o.total = off;
    return o;
}

template <int KS, int STRIDE, int PAD, bool INPUT>
int launch_conv(const float* in0, const float* in1, int n_split, int B, const ConvSpec& s, int H, int W, int OH, int OW,
                const float* wk, const float* bias, float* out, cudaStream_t st) {
    const int M = B * OH * OW;
    const dim3 grid((M + kBM - 1) / kBM, s.cout / kBN);
    conv_relu_kernel<KS, STRIDE, PAD, INPUT><<<grid, kConvThreads, 0, st>>>(in0, in1, n_split, s.cin, H, W, OH, OW, M,
                                                                            s.cout, wk, bias, out);
    SB_LAUNCH_CHECK("lpips conv_relu_kernel");
    return SB_OK;
}

int launch_pool(const float* in, int planes, int H, int W, int OH, int OW, float* out, cudaStream_t st) {
    const size_t n = (size_t)planes * OH * OW;
    const unsigned blocks = (unsigned)((n + 255) / 256 < 4224 ? (n + 255) / 256 : 4224);
    maxpool_kernel<<<blocks, 256, 0, st>>>(in, planes, H, W, OH, OW, out);
    SB_LAUNCH_CHECK("lpips maxpool_kernel");
    return SB_OK;
}

}  // namespace

}  // namespace sb

using namespace sb;

extern "C" {

SB_API int sb_lpips_weights_floats(size_t* n) {
    if (!n) return SB_ERR_BAD_ARG;
    *n = weight_offsets().total;
    return SB_OK;
}

SB_API int sb_lpips_workspace_bytes(int N, int H, int W, size_t* bytes) {
    if (!bytes || !args_ok(N, H, W)) return SB_ERR_BAD_ARG;
    *bytes = make_plan(N, H, W, nullptr).bytes;
    return SB_OK;
}

SB_API int sb_lpips(const float* x, const float* y, int N, int H, int W, const float* weights, void* workspace,
                    size_t workspace_bytes, double* per_image, double* mean, void* stream) {
    if (!x || !y || !weights || !workspace || (!per_image && !mean) || !args_ok(N, H, W)) return SB_ERR_BAD_ARG;
    if (workspace_bytes < make_plan(N, H, W, nullptr).bytes) return SB_ERR_WORKSPACE;
    const Plan p = make_plan(N, H, W, workspace);
    const WeightOffsets o = weight_offsets();
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int B = 2 * N;
    const float* w = weights;
    int rc;
#define SB_LPIPS_TRY(expr) do { if ((rc = (expr)) != SB_OK) return rc; } while (0)
    SB_LPIPS_TRY((launch_conv<11, 4, 2, true>(x, y, N, B, kConv[0], H, W, p.H1, p.W1, w + o.w[0], w + o.b[0], p.f[0],
                                              st)));
    SB_LPIPS_TRY(launch_pool(p.f[0], B * kConv[0].cout, p.H1, p.W1, p.Hp1, p.Wp1, p.pool1, st));
    SB_LPIPS_TRY((launch_conv<5, 1, 2, false>(p.pool1, p.pool1, B, B, kConv[1], p.Hp1, p.Wp1, p.Hp1, p.Wp1,
                                              w + o.w[1], w + o.b[1], p.f[1], st)));
    SB_LPIPS_TRY(launch_pool(p.f[1], B * kConv[1].cout, p.Hp1, p.Wp1, p.Hp2, p.Wp2, p.pool2, st));
    const float* in = p.pool2;
    for (int l = 2; l < kLayers; ++l) {
        SB_LPIPS_TRY((launch_conv<3, 1, 1, false>(in, in, B, B, kConv[l], p.Hp2, p.Wp2, p.Hp2, p.Wp2, w + o.w[l],
                                                  w + o.b[l], p.f[l], st)));
        in = p.f[l];
    }
#undef SB_LPIPS_TRY
    for (int l = 0; l < kLayers; ++l) {
        lpips_head_kernel<<<dim3(p.D.nblk[l], N), kHeadThreads, 0, st>>>(p.f[l], N, kConv[l].cout, p.D.P[l],
                                                                          w + o.lin[l], p.partials + p.D.part_off[l]);
        SB_LAUNCH_CHECK("lpips_head_kernel");
    }
    lpips_finalize_kernel<<<1, kHeadThreads, 0, st>>>(p.partials, N, p.D, per_image, mean);
    SB_LAUNCH_CHECK("lpips_finalize_kernel");
    return SB_OK;
}

}  // extern "C"
