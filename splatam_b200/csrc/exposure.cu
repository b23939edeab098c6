// exposure.cu -- per-frame affine colour correction (splatam_b200/train_ops.py `exposure`; the rule is stated in
// include/splatam_b200.h and restated in oracle/exposure_numpy.py).
//
//   sb_exposure_apply      one elementwise pass over the flat [3*H*W] image, four values per thread iteration
//                          (float4 when every pointer is 16-byte aligned, scalar otherwise; a float4 may straddle two
//                          channels, so each value picks its own channel); the three gains are computed once per CTA
//                          in double and rounded to float
//   sb_exposure_backward   gx in the same elementwise pass, the six sums as kBlocks fixed CTAs of grid-stride partials
//                          in double (warp shuffles, then warps in order), summed in block order by one finishing
//                          kernel: no atomics, so the result does not change from call to call
#include <cmath>

#include "common.cuh"

namespace sb {

namespace {

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr int kBlocks = SB_EXPOSURE_BLOCKS;   // fixed, so the summation order does not depend on the device
constexpr int kMaxApplyBlocks = 4096;

inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

__device__ __forceinline__ int channel_of(long long i, long long n) { return (int)(i >= n) + (int)(i >= 2 * n); }

__device__ __forceinline__ float pick(int c, float v0, float v1, float v2) { return c == 0 ? v0 : (c == 1 ? v1 : v2); }

// gain[c] = float(exp(+-a_c)) in double, bias[c] = b_c; written by the first three threads of the CTA
__device__ __forceinline__ void load_gains(const float* ab, int inverse, float* gain, float* bias) {
    if (threadIdx.x < 3) {
        const double a = (double)ab[threadIdx.x];
        gain[threadIdx.x] = (float)exp(inverse ? -a : a);
        bias[threadIdx.x] = ab[3 + threadIdx.x];
    }
    __syncthreads();
}

__device__ __forceinline__ float apply_one(float x, float g, float b, int inverse) {
    return inverse ? __fmul_rn(__fsub_rn(x, b), g) : __fadd_rn(__fmul_rn(g, x), b);
}

template <bool kVec>
__global__ void __launch_bounds__(kThreads) apply_kernel(long long n, const float* __restrict__ x,
                                                         const float* __restrict__ ab, int inverse,
                                                         float* __restrict__ y) {
    __shared__ float gain[3], bias[3];
    load_gains(ab, inverse, gain, bias);
    const long long total = 3 * n, quads = (total + 3) / 4;
    for (long long q = blockIdx.x * (long long)kThreads + threadIdx.x; q < quads;
         q += (long long)gridDim.x * kThreads) {
        const long long i0 = 4 * q;
        if (kVec && i0 + 3 < total) {
            const float4 v = reinterpret_cast<const float4*>(x)[q];
            const float in[4] = {v.x, v.y, v.z, v.w};
            float out[4];
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const int c = channel_of(i0 + j, n);
                out[j] = apply_one(in[j], pick(c, gain[0], gain[1], gain[2]), pick(c, bias[0], bias[1], bias[2]),
                                   inverse);
            }
            reinterpret_cast<float4*>(y)[q] = make_float4(out[0], out[1], out[2], out[3]);
        } else {
            for (long long i = i0; i < i0 + 4 && i < total; ++i) {
                const int c = channel_of(i, n);
                y[i] = apply_one(x[i], pick(c, gain[0], gain[1], gain[2]), pick(c, bias[0], bias[1], bias[2]),
                                 inverse);
            }
        }
    }
}

// per value: gx = gain_c gy (float); acc[c] += double(gy) double(x), acc[3 + c] += double(gy)
__device__ __forceinline__ void backward_one(float x, float gy, int c, const float* gain, float& gx, double* acc) {
    gx = __fmul_rn(pick(c, gain[0], gain[1], gain[2]), gy);
    const double p = (double)gy * (double)x, g = (double)gy;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        acc[k] += c == k ? p : 0.0;
        acc[3 + k] += c == k ? g : 0.0;
    }
}

template <bool kVec>
__global__ void __launch_bounds__(kThreads) backward_partials_kernel(long long n, const float* __restrict__ x,
                                                                     const float* __restrict__ ab,
                                                                     const float* __restrict__ gy,
                                                                     float* __restrict__ gx,
                                                                     double* __restrict__ partials) {
    __shared__ float gain[3], bias[3];
    __shared__ double warp_sums[kWarps][6];
    load_gains(ab, 0, gain, bias);
    double acc[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
    const long long total = 3 * n, quads = (total + 3) / 4;
    for (long long q = blockIdx.x * (long long)kThreads + threadIdx.x; q < quads;
         q += (long long)gridDim.x * kThreads) {
        const long long i0 = 4 * q;
        if (kVec && i0 + 3 < total) {
            const float4 xv = reinterpret_cast<const float4*>(x)[q];
            const float4 gv = reinterpret_cast<const float4*>(gy)[q];
            const float xs[4] = {xv.x, xv.y, xv.z, xv.w}, gs[4] = {gv.x, gv.y, gv.z, gv.w};
            float out[4];
#pragma unroll
            for (int j = 0; j < 4; ++j) backward_one(xs[j], gs[j], channel_of(i0 + j, n), gain, out[j], acc);
            reinterpret_cast<float4*>(gx)[q] = make_float4(out[0], out[1], out[2], out[3]);
        } else {
            for (long long i = i0; i < i0 + 4 && i < total; ++i) {
                float o;
                backward_one(x[i], gy[i], channel_of(i, n), gain, o, acc);
                gx[i] = o;
            }
        }
    }
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int k = 0; k < 6; ++k) {
        double v = acc[k];
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) v += __shfl_down_sync(0xffffffffu, v, off);
        if (lane == 0) warp_sums[warp][k] = v;
    }
    __syncthreads();
    if (threadIdx.x < 6) {
        double s = 0.0;
        for (int w = 0; w < kWarps; ++w) s += warp_sums[w][threadIdx.x];
        partials[(size_t)blockIdx.x * 6 + threadIdx.x] = s;
    }
}

// g_ab[c] = exp(a_c) sum_c(gy x), g_ab[3 + c] = sum_c(gy): the kBlocks partials of each sum in block order
__global__ void backward_finish_kernel(const float* __restrict__ ab, const double* __restrict__ partials,
                                       double* __restrict__ g_ab) {
    const int k = threadIdx.x;
    if (k >= 6) return;
    double s = 0.0;
    for (int b = 0; b < kBlocks; ++b) s += partials[(size_t)b * 6 + k];
    g_ab[k] = k < 3 ? exp((double)ab[k]) * s : s;
}

unsigned int apply_blocks(long long n) {
    const long long quads = (3 * n + 3) / 4;
    const long long b = (quads + kThreads - 1) / kThreads;
    return (unsigned int)(b < kMaxApplyBlocks ? b : kMaxApplyBlocks);
}

}  // namespace

}  // namespace sb

using namespace sb;

extern "C" {

SB_API int sb_exposure_workspace_bytes(int height, int width, size_t* bytes) {
    if (height < 1 || width < 1 || !bytes) return SB_ERR_BAD_ARG;
    *bytes = (size_t)kBlocks * 6 * sizeof(double);
    return SB_OK;
}

SB_API int sb_exposure_apply(int height, int width, const float* x, const float* ab, int inverse, float* y,
                             void* stream) {
    if (height < 1 || width < 1 || !x || !ab || !y || (inverse != 0 && inverse != 1)) return SB_ERR_BAD_ARG;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const long long n = (long long)height * width;
    if (aligned16(x) && aligned16(y))
        apply_kernel<true><<<apply_blocks(n), kThreads, 0, st>>>(n, x, ab, inverse, y);
    else
        apply_kernel<false><<<apply_blocks(n), kThreads, 0, st>>>(n, x, ab, inverse, y);
    SB_LAUNCH_CHECK("exposure_apply_kernel");
    return SB_OK;
}

SB_API int sb_exposure_backward(int height, int width, const float* x, const float* ab, const float* gy, float* gx,
                                double* g_ab, void* workspace, size_t workspace_bytes, void* stream) {
    if (height < 1 || width < 1 || !x || !ab || !gy || !gx || !g_ab || !workspace) return SB_ERR_BAD_ARG;
    if (workspace_bytes < (size_t)kBlocks * 6 * sizeof(double)) return SB_ERR_WORKSPACE;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const long long n = (long long)height * width;
    double* partials = static_cast<double*>(workspace);
    if (aligned16(x) && aligned16(gy) && aligned16(gx))
        backward_partials_kernel<true><<<kBlocks, kThreads, 0, st>>>(n, x, ab, gy, gx, partials);
    else
        backward_partials_kernel<false><<<kBlocks, kThreads, 0, st>>>(n, x, ab, gy, gx, partials);
    SB_LAUNCH_CHECK("exposure_backward_partials_kernel");
    backward_finish_kernel<<<1, 32, 0, st>>>(ab, partials, g_ab);
    SB_LAUNCH_CHECK("exposure_backward_finish_kernel");
    return SB_OK;
}

}  // extern "C"
