// viewer.cu -- the pictures of the reference's viewers (R/viz_scripts/final_recon.py, online_recon.py) without a
// window: what Open3D draws from a render's back-projected pixels, from the Gaussian centres and from the camera
// frustums and trajectory, as one uint8 HWC RGB frame at view_scale s times the render size.
//
//   sb_viewer_compose  render [3,h,w] + depth [h,w] (+ silhouette) -> frame [h*s, w*s, 3] and a float depth buffer
//   sb_viewer_points   Gaussian centres as s x s squares, nearest first              -> frame and depth buffer
//   sb_viewer_lines    world-space segments, 1 px wide, depth-tested against the buffer -> drawn over the frame
//
// Pixel rules (this project's; Open3D's exact coverage is not reproduced):
//   * Background: white at infinite depth.  A render pixel with depth <= 0 or NaN is background (Open3D puts its
//     point on the camera centre, where it is not drawn).
//   * Colours: round_half_even(clamp(x, 0, 1) * 255f), NaN -> 0, as eval_frames.cu.
//   * Compose: output pixel (X, Y) shows render pixel (X / s, Y / s).  Back-projected through k and displayed at
//     k * s, render pixel (x, y) lands at (s x, s y), and the points rule below covers exactly that s x s block.
//   * Depth mode: vmax = max over pixels of d where 0 < d < 15, else 0 (matplotlib Normalize(0, max(d * (d < 15)))
//     with NaN pixels left out); index = trunc(float32(d / vmax) * 256), 256 -> 255, vmax == 0 -> 0; d >= 15 white.
//   * Points: camera z = ((r0 x + r1 y) + r2 z) + t per row in float32; points with !(near < z < far) or a
//     non-finite projection u = fx x / z + cx, v = fy y / z + cy are skipped.  The square's top-left pixel is
//     (floor(u + 0.5), floor(v + 0.5)); it covers s x s pixels.  Per pixel the key (float bits of z) << 32 | index
//     wins by atomicMin: the nearest point, ties to the lower index, whatever the launch order.
//   * Lines: endpoints to the camera as points; a segment with both z <= near is dropped, one with one endpoint
//     behind is clipped to z = near.  Projected with k * s, it is drawn by a DDA along its major screen axis: at
//     every pixel centre c + 0.5 of that axis within the segment's span, a = (c + 0.5 - p0) / (p1 - p0), the minor
//     coordinate p0' + a (p1' - p0') is floored, and the camera depth 1 / ((1 - a) / z0 + a / z1) is interpolated
//     perspective-correctly.  A pixel is drawn when that depth is below the depth buffer's; overlapping segments
//     resolve by the same (z, segment index) atomicMin in a separate key buffer, then the winners are written.
#include "common.cuh"

namespace sb {

namespace {

constexpr int kViewThreads = 256;
constexpr int kViewMaxBlocks = 1056;   // 132 SMs x 8
constexpr unsigned long long kNoKey = ~0ull;

__device__ __forceinline__ uint8_t rgb_u8(float x) {
    if (!(x == x)) return 0;
    const float c = fminf(fmaxf(x, 0.f), 1.f);
    return (uint8_t)__float2int_rn(__fmul_rn(c, 255.f));
}

__device__ __forceinline__ bool foreground(float d) { return d > 0.f; }   // false for NaN

__device__ __forceinline__ void put_white(uint8_t* o) { o[0] = o[1] = o[2] = 255; }

inline int grid_for(long long n) {
    const long long b = (n + kViewThreads - 1) / kViewThreads;
    return (int)(b < kViewMaxBlocks ? (b > 0 ? b : 1) : kViewMaxBlocks);
}

// camera-frame coordinates of a world point under a row-major 4x4 w2c, in a fixed float32 operation order
__device__ __forceinline__ float3 to_camera(const float* m, float x, float y, float z) {
    float3 c;
    c.x = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(m[0], x), __fmul_rn(m[1], y)), __fmul_rn(m[2], z)), m[3]);
    c.y = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(m[4], x), __fmul_rn(m[5], y)), __fmul_rn(m[6], z)), m[7]);
    c.z = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(m[8], x), __fmul_rn(m[9], y)), __fmul_rn(m[10], z)), m[11]);
    return c;
}

__global__ void __launch_bounds__(kViewThreads)
depth_vmax_kernel(const float* __restrict__ depth, int n, unsigned int* __restrict__ vmax_bits) {
    float m = 0.f;
    for (int p = blockIdx.x * blockDim.x + threadIdx.x; p < n; p += gridDim.x * blockDim.x) {
        const float d = depth[p];
        if (d > 0.f && d < 15.f) m = fmaxf(m, d);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    // non-negative floats order as their bit patterns
    if ((threadIdx.x & 31) == 0 && m > 0.f) atomicMax(vmax_bits, __float_as_uint(m));
}

__global__ void __launch_bounds__(kViewThreads)
compose_kernel(const float* __restrict__ color, const float* __restrict__ depth, const float* __restrict__ sil,
               int h, int w, int mode, int s, const uint8_t* __restrict__ lut,
               const unsigned int* __restrict__ vmax_bits, uint8_t* __restrict__ out, float* __restrict__ zbuf) {
    __shared__ uint8_t s_lut[256 * 3];
    if (mode == 1) {
        for (int i = threadIdx.x; i < 256 * 3; i += blockDim.x) s_lut[i] = lut[i];
        __syncthreads();
    }
    const int W = w * s;
    const long long n = (long long)W * h * s;
    const int hw = h * w;
    const float vmax = mode == 1 ? __uint_as_float(*vmax_bits) : 0.f;
    for (long long q = blockIdx.x * (long long)blockDim.x + threadIdx.x; q < n; q += (long long)gridDim.x * blockDim.x) {
        const int X = (int)(q % W), Y = (int)(q / W);
        const int p = (Y / s) * w + X / s;
        uint8_t* o = out + 3 * q;
        const float d = depth[p];
        if (!foreground(d) || (mode == 1 && !(d < 15.f))) {
            put_white(o);
            zbuf[q] = foreground(d) ? d : __int_as_float(0x7f800000);
            continue;
        }
        zbuf[q] = d;
        if (mode == 0) {
            o[0] = rgb_u8(color[p]);
            o[1] = rgb_u8(color[hw + p]);
            o[2] = rgb_u8(color[2 * hw + p]);
        } else if (mode == 1) {
            int idx = 0;
            if (vmax > 0.f) {
                const float x = __fmul_rn(__fdiv_rn(d, vmax), 256.f);
                idx = x >= 256.f ? 255 : (int)x;
            }
            o[0] = s_lut[3 * idx]; o[1] = s_lut[3 * idx + 1]; o[2] = s_lut[3 * idx + 2];
        } else {
            const uint8_t g = rgb_u8(__fsub_rn(1.f, sil[p]));
            o[0] = o[1] = o[2] = g;
        }
    }
}

__global__ void __launch_bounds__(kViewThreads)
points_splat_kernel(int P, const float* __restrict__ means, const float* __restrict__ timestep, float t_max,
                    const float* __restrict__ w2c, float fx, float fy, float cx, float cy, int W, int H, int s,
                    float near, float far, unsigned long long* __restrict__ keys) {
    __shared__ float m[12];
    if (threadIdx.x < 12) m[threadIdx.x] = w2c[threadIdx.x];
    __syncthreads();
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < P; i += gridDim.x * blockDim.x) {
        if (timestep && !(timestep[i] <= t_max)) continue;
        const float3 c = to_camera(m, means[3 * i], means[3 * i + 1], means[3 * i + 2]);
        if (!(c.z > near && c.z < far)) continue;
        const float u = __fadd_rn(__fdiv_rn(__fmul_rn(fx, c.x), c.z), cx);
        const float v = __fadd_rn(__fdiv_rn(__fmul_rn(fy, c.y), c.z), cy);
        if (!isfinite(u) || !isfinite(v)) continue;
        const float x0f = floorf(__fadd_rn(u, 0.5f)), y0f = floorf(__fadd_rn(v, 0.5f));
        if (x0f >= (float)W || y0f >= (float)H || x0f + (float)s <= 0.f || y0f + (float)s <= 0.f) continue;
        const int x0 = (int)x0f, y0 = (int)y0f;
        const unsigned long long key = ((unsigned long long)__float_as_uint(c.z) << 32) | (unsigned int)i;
        for (int dy = 0; dy < s; ++dy) {
            const int y = y0 + dy;
            if (y < 0 || y >= H) continue;
            for (int dx = 0; dx < s; ++dx) {
                const int x = x0 + dx;
                if (x < 0 || x >= W) continue;
                unsigned long long* k = keys + (size_t)y * W + x;
                if (key < *k) atomicMin(k, key);
            }
        }
    }
}

__global__ void __launch_bounds__(kViewThreads)
points_resolve_kernel(const unsigned long long* __restrict__ keys, long long n, const float* __restrict__ colors,
                      uint8_t* __restrict__ out, float* __restrict__ zbuf) {
    for (long long q = blockIdx.x * (long long)blockDim.x + threadIdx.x; q < n; q += (long long)gridDim.x * blockDim.x) {
        const unsigned long long key = keys[q];
        uint8_t* o = out + 3 * q;
        if (key == kNoKey) {
            put_white(o);
            zbuf[q] = __int_as_float(0x7f800000);
            continue;
        }
        const unsigned int i = (unsigned int)(key & 0xffffffffu);
        o[0] = rgb_u8(colors[3 * (size_t)i]);
        o[1] = rgb_u8(colors[3 * (size_t)i + 1]);
        o[2] = rgb_u8(colors[3 * (size_t)i + 2]);
        zbuf[q] = __uint_as_float((unsigned int)(key >> 32));
    }
}

// one warp per segment; lanes stride over the major-axis pixel centres
__global__ void __launch_bounds__(kViewThreads)
lines_splat_kernel(int S, const float* __restrict__ seg, const float* __restrict__ w2c, float fx, float fy, float cx,
                   float cy, int W, int H, float near, const float* __restrict__ zbuf,
                   unsigned long long* __restrict__ keys) {
    __shared__ float m[12];
    if (threadIdx.x < 12) m[threadIdx.x] = w2c[threadIdx.x];
    __syncthreads();
    const int lane = threadIdx.x & 31;
    const int warps = gridDim.x * (blockDim.x >> 5);
    for (int j = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); j < S; j += warps) {
        const float* e = seg + 6 * (size_t)j;
        float3 a = to_camera(m, e[0], e[1], e[2]);
        float3 b = to_camera(m, e[3], e[4], e[5]);
        if (!(a.z > near) && !(b.z > near)) continue;
        if (!(a.z > near) || !(b.z > near)) {
            if (!(a.z > near)) { const float3 t = a; a = b; b = t; }   // a in front, b behind
            const float f = __fdiv_rn(__fsub_rn(near, a.z), __fsub_rn(b.z, a.z));
            b.x = __fadd_rn(a.x, __fmul_rn(f, __fsub_rn(b.x, a.x)));
            b.y = __fadd_rn(a.y, __fmul_rn(f, __fsub_rn(b.y, a.y)));
            b.z = near;
        }
        const float u0 = __fadd_rn(__fdiv_rn(__fmul_rn(fx, a.x), a.z), cx);
        const float v0 = __fadd_rn(__fdiv_rn(__fmul_rn(fy, a.y), a.z), cy);
        const float u1 = __fadd_rn(__fdiv_rn(__fmul_rn(fx, b.x), b.z), cx);
        const float v1 = __fadd_rn(__fdiv_rn(__fmul_rn(fy, b.y), b.z), cy);
        if (!isfinite(u0) || !isfinite(v0) || !isfinite(u1) || !isfinite(v1)) continue;
        const float du = __fsub_rn(u1, u0), dv = __fsub_rn(v1, v0);
        if (du == 0.f && dv == 0.f) continue;
        const bool xmajor = fabsf(du) >= fabsf(dv);
        const float p0 = xmajor ? u0 : v0, p1 = xmajor ? u1 : v1, q0 = xmajor ? v0 : u0;
        const float dp = xmajor ? du : dv, dq = xmajor ? dv : du;
        const int nmaj = xmajor ? W : H, nmin = xmajor ? H : W;
        float lo = ceilf(__fsub_rn(fminf(p0, p1), 0.5f)), hi = floorf(__fsub_rn(fmaxf(p0, p1), 0.5f));
        lo = fmaxf(lo, 0.f);
        hi = fminf(hi, (float)(nmaj - 1));
        if (lo > hi) continue;
        const float iz0 = __fdiv_rn(1.f, a.z), iz1 = __fdiv_rn(1.f, b.z);
        for (int c = (int)lo + lane; c <= (int)hi; c += 32) {
            const float t = __fdiv_rn(__fsub_rn(__fadd_rn((float)c, 0.5f), p0), dp);
            const float r = floorf(__fadd_rn(q0, __fmul_rn(t, dq)));
            if (!(r >= 0.f && r < (float)nmin)) continue;
            const int X = xmajor ? c : (int)r, Y = xmajor ? (int)r : c;
            const float z = __fdiv_rn(1.f, __fadd_rn(__fmul_rn(__fsub_rn(1.f, t), iz0), __fmul_rn(t, iz1)));
            const size_t q = (size_t)Y * W + X;
            if (!(z < zbuf[q])) continue;
            const unsigned long long key = ((unsigned long long)__float_as_uint(z) << 32) | (unsigned int)j;
            if (key < keys[q]) atomicMin(keys + q, key);
        }
    }
}

__global__ void __launch_bounds__(kViewThreads)
lines_resolve_kernel(const unsigned long long* __restrict__ keys, long long n, const uint8_t* __restrict__ colors,
                     uint8_t* __restrict__ out) {
    for (long long q = blockIdx.x * (long long)blockDim.x + threadIdx.x; q < n; q += (long long)gridDim.x * blockDim.x) {
        const unsigned long long key = keys[q];
        if (key == kNoKey) continue;
        const unsigned int j = (unsigned int)(key & 0xffffffffu);
        out[3 * q] = colors[3 * j];
        out[3 * q + 1] = colors[3 * j + 1];
        out[3 * q + 2] = colors[3 * j + 2];
    }
}

}  // namespace

}  // namespace sb

using namespace sb;

extern "C" {

SB_API int sb_viewer_compose(const float* color, const float* depth, const float* sil, int h, int w, int mode,
                             int view_scale, const uint8_t* lut, unsigned int* vmax_bits, uint8_t* out, float* zbuf,
                             void* stream) {
    if (h < 1 || w < 1 || view_scale < 1 || mode < 0 || mode > 2 || !depth || !out || !zbuf ||
        (mode == 0 && !color) || (mode == 1 && (!lut || !vmax_bits)) || (mode == 2 && !sil) ||
        (long long)h * w * view_scale * view_scale >= (1LL << 31) / 3)
        return SB_ERR_BAD_ARG;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const long long n = (long long)h * w * view_scale * view_scale;
    if (mode == 1) {
        SB_CUDA_CHECK(cudaMemsetAsync(vmax_bits, 0, sizeof(unsigned int), st));
        depth_vmax_kernel<<<grid_for((long long)h * w), kViewThreads, 0, st>>>(depth, h * w, vmax_bits);
        SB_LAUNCH_CHECK("depth_vmax_kernel");
    }
    compose_kernel<<<grid_for(n), kViewThreads, 0, st>>>(color, depth, sil, h, w, mode, view_scale, lut, vmax_bits,
                                                         out, zbuf);
    SB_LAUNCH_CHECK("compose_kernel");
    return SB_OK;
}

SB_API int sb_viewer_points(int P, const float* means, const float* colors, const float* timestep, float t_max,
                            const float* w2c, float fx, float fy, float cx, float cy, int width, int height,
                            int view_scale, float near, float far, unsigned long long* keys, uint8_t* out, float* zbuf,
                            void* stream) {
    if (P < 0 || width < 1 || height < 1 || view_scale < 1 || !(near >= 0.f) || !(far > near) || !w2c || !keys ||
        !out || !zbuf || (P > 0 && (!means || !colors)) || (long long)width * height >= (1LL << 31) / 3)
        return SB_ERR_BAD_ARG;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const long long n = (long long)width * height;
    SB_CUDA_CHECK(cudaMemsetAsync(keys, 0xff, sizeof(unsigned long long) * n, st));
    if (P > 0) {
        points_splat_kernel<<<grid_for(P), kViewThreads, 0, st>>>(P, means, timestep, t_max, w2c, fx, fy, cx, cy,
                                                                  width, height, view_scale, near, far, keys);
        SB_LAUNCH_CHECK("points_splat_kernel");
    }
    points_resolve_kernel<<<grid_for(n), kViewThreads, 0, st>>>(keys, n, colors, out, zbuf);
    SB_LAUNCH_CHECK("points_resolve_kernel");
    return SB_OK;
}

SB_API int sb_viewer_lines(int S, const float* segments, const uint8_t* colors, const float* w2c, float fx, float fy,
                           float cx, float cy, int width, int height, float near, const float* zbuf,
                           unsigned long long* keys, uint8_t* out, void* stream) {
    if (S < 0 || width < 1 || height < 1 || !(near > 0.f) || !w2c || !zbuf || !keys || !out ||
        (S > 0 && (!segments || !colors)) || (long long)width * height >= (1LL << 31) / 3)
        return SB_ERR_BAD_ARG;
    if (S == 0) return SB_OK;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const long long n = (long long)width * height;
    SB_CUDA_CHECK(cudaMemsetAsync(keys, 0xff, sizeof(unsigned long long) * n, st));
    const int warps_per_block = kViewThreads / 32;
    long long blocks = ((long long)S + warps_per_block - 1) / warps_per_block;
    if (blocks > kViewMaxBlocks) blocks = kViewMaxBlocks;
    lines_splat_kernel<<<(int)blocks, kViewThreads, 0, st>>>(S, segments, w2c, fx, fy, cx, cy, width, height, near,
                                                             zbuf, keys);
    SB_LAUNCH_CHECK("lines_splat_kernel");
    lines_resolve_kernel<<<grid_for(n), kViewThreads, 0, st>>>(keys, n, colors, out);
    SB_LAUNCH_CHECK("lines_resolve_kernel");
    return SB_OK;
}

}  // extern "C"
