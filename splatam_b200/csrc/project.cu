// project.cu -- stage 1 of the forward: per-Gaussian 3D->2D projection, screen-space covariance,
// conic, radius, tile rectangle (FORWARD::preprocessCUDA, X/cuda_rasterizer/forward.cu:155-256,
// with in_frustum/getRect/ndc2Pix of X/cuda_rasterizer/auxiliary.h:41-56,139-163), followed by the
// depth ordering of the Gaussians.  Also sb_mark_visible (checkFrustum, rasterizer_impl.cu:54-66).
//
// Bit-exactness: the tile/depth sort keys must equal the reference's, so every float that feeds
// `depth`, `radius` or the pixel centre is computed with the exact operation sequence that nvcc
// 12.9 emits for the reference source (read off the SASS of the reference build; the sequence is
// written out with explicit __f*_rn intrinsics so this file's own contraction cannot change it).
// Division, reciprocal and square root are IEEE correctly-rounded in both builds.
#include "common.cuh"
#include "radix_sort.cuh"
#include <cub/device/device_scan.cuh>
#include <cub/iterator/counting_input_iterator.cuh>
#include <cub/iterator/transform_input_iterator.cuh>

namespace sb {

namespace {

constexpr int kProjThreads = 256;

// Cooperative, coalesced load of a [P,3] float array slice (256 rows) into shared memory.
// Uses 128-bit loads when the base pointer is 16-B aligned (a block's slice starts at a multiple
// of 3072 B), scalar loads otherwise (views with odd storage offsets).
__device__ __forceinline__ void stage_aos3(float* __restrict__ dst, const float* __restrict__ src,
                                           int first_row, int P, bool aligned16) {
    const int nfloat = min(kProjThreads, P - first_row) * 3;
    const float* base = src + (size_t)first_row * 3;
    if (aligned16) {
        const int nvec = nfloat >> 2;
        for (int i = threadIdx.x; i < nvec; i += kProjThreads)
            reinterpret_cast<float4*>(dst)[i] = __ldg(reinterpret_cast<const float4*>(base) + i);
        for (int i = (nvec << 2) + threadIdx.x; i < nfloat; i += kProjThreads) dst[i] = __ldg(base + i);
    } else {
        for (int i = threadIdx.x; i < nfloat; i += kProjThreads) dst[i] = __ldg(base + i);
    }
}

struct Cov3 { float c0, c1, c2, c3, c4, c5; };

// Sigma = (S R)^T (S R) from scale*modifier and the quaternion AS GIVEN (no normalisation),
// X/cuda_rasterizer/forward.cu:118-152, operation order from the reference SASS.
__device__ __forceinline__ Cov3 cov3d_from_scale_rot(float sx_, float sy_, float sz_, float mod, float4 q) {
    const float r = q.x, x = q.y, y = q.z, z = q.w;
    const float xz = __fmul_rn(x, z), rx = __fmul_rn(r, x), rz = __fmul_rn(r, z);
    const float yy = __fmul_rn(y, y), zz = __fmul_rn(z, z);
    const float xz_p_ry = __fmaf_rn(r, y, xz), xz_m_ry = __fmaf_rn(-r, y, xz);
    const float yz_m_rx = __fmaf_rn(y, z, -rx), yz_p_rx = __fmaf_rn(y, z, rx);
    const float xy_m_rz = __fmaf_rn(x, y, -rz), xy_p_rz = __fmaf_rn(x, y, rz);
    const float xx_p_yy = __fmaf_rn(x, x, yy), xx_p_zz = __fmaf_rn(x, x, zz), yy_p_zz = __fadd_rn(yy, zz);
    // R[c][r] (GLM column-major constructor)
    const float R00 = __fsub_rn(1.f, __fadd_rn(yy_p_zz, yy_p_zz));
    const float R01 = __fadd_rn(xy_m_rz, xy_m_rz), R02 = __fadd_rn(xz_p_ry, xz_p_ry);
    const float R10 = __fadd_rn(xy_p_rz, xy_p_rz);
    const float R11 = __fsub_rn(1.f, __fadd_rn(xx_p_zz, xx_p_zz));
    const float R12 = __fadd_rn(yz_m_rx, yz_m_rx);
    const float R20 = __fadd_rn(xz_m_ry, xz_m_ry), R21 = __fadd_rn(yz_p_rx, yz_p_rx);
    const float R22 = __fsub_rn(1.f, __fadd_rn(xx_p_yy, xx_p_yy));
    const float sx = __fmul_rn(sx_, mod), sy = __fmul_rn(sy_, mod), sz = __fmul_rn(sz_, mod);
    // M = S * R : M[c][r] = s_r * R[c][r]
    const float M00 = __fmul_rn(sx, R00), M01 = __fmul_rn(sy, R01), M02 = __fmul_rn(sz, R02);
    const float M10 = __fmul_rn(sx, R10), M11 = __fmul_rn(sy, R11), M12 = __fmul_rn(sz, R12);
    const float M20 = __fmul_rn(sx, R20), M21 = __fmul_rn(sy, R21), M22 = __fmul_rn(sz, R22);
    Cov3 o;
    o.c0 = __fmaf_rn(M02, M02, __fmaf_rn(M00, M00, __fmul_rn(M01, M01)));
    o.c1 = __fmaf_rn(M02, M12, __fmaf_rn(M00, M10, __fmul_rn(M01, M11)));
    o.c2 = __fmaf_rn(M02, M22, __fmaf_rn(M00, M20, __fmul_rn(M01, M21)));
    o.c3 = __fmaf_rn(M12, M12, __fmaf_rn(M10, M10, __fmul_rn(M11, M11)));
    o.c4 = __fmaf_rn(M12, M22, __fmaf_rn(M10, M20, __fmul_rn(M11, M21)));
    o.c5 = __fmaf_rn(M22, M22, __fmaf_rn(M20, M20, __fmul_rn(M21, M21)));
    return o;
}

// EWA screen-space covariance + 0.3 low-pass (X/cuda_rasterizer/forward.cu:74-113).
__device__ __forceinline__ float3 cov2d_exact(float px, float py, float pz, float focal_x, float focal_y,
                                              float tan_fovx, float tan_fovy, const Cov3& v,
                                              const float* __restrict__ vm) {
    const float tz = xform_row(vm, 2, px, py, pz);
    const float tx = xform_row(vm, 0, px, py, pz);
    const float ty = xform_row(vm, 1, px, py, pz);
    const float limx = __fmul_rn(tan_fovx, 1.3f), limy = __fmul_rn(tan_fovy, 1.3f);
    const float cx = fminf(fmaxf(__fdiv_rn(tx, tz), -limx), limx);
    const float cy = fminf(fmaxf(__fdiv_rn(ty, tz), -limy), limy);
    const float tz2 = __fmul_rn(tz, tz);
    const float J00 = __fdiv_rn(focal_x, tz);
    const float J02 = __fdiv_rn(__fmul_rn(__fmul_rn(tz, -cx), focal_x), tz2);
    const float J11 = __fdiv_rn(focal_y, tz);
    const float J12 = __fdiv_rn(__fmul_rn(__fmul_rn(tz, -cy), focal_y), tz2);
    // T = W * J  (third column of J is zero)
    const float T00 = __fmaf_rn(vm[2], J02, __fmul_rn(vm[0], J00));
    const float T01 = __fmaf_rn(vm[6], J02, __fmul_rn(vm[4], J00));
    const float T02 = __fmaf_rn(vm[10], J02, __fmul_rn(vm[8], J00));
    const float T10 = __fmaf_rn(vm[2], J12, __fmul_rn(vm[1], J11));
    const float T11 = __fmaf_rn(vm[6], J12, __fmul_rn(vm[5], J11));
    const float T12 = __fmaf_rn(vm[10], J12, __fmul_rn(vm[9], J11));
    // A = T^T * Vrk^T
    const float A00 = __fmaf_rn(T02, v.c2, __fmaf_rn(T00, v.c0, __fmul_rn(T01, v.c1)));
    const float A10 = __fmaf_rn(T02, v.c4, __fmaf_rn(T00, v.c1, __fmul_rn(T01, v.c3)));
    const float A20 = __fmaf_rn(T02, v.c5, __fmaf_rn(T00, v.c2, __fmul_rn(T01, v.c4)));
    const float A01 = __fmaf_rn(T12, v.c2, __fmaf_rn(T10, v.c0, __fmul_rn(T11, v.c1)));
    const float A11 = __fmaf_rn(T12, v.c4, __fmaf_rn(T10, v.c1, __fmul_rn(T11, v.c3)));
    const float A21 = __fmaf_rn(T12, v.c5, __fmaf_rn(T10, v.c2, __fmul_rn(T11, v.c4)));
    // cov = A * T, upper-left 2x2
    float3 cov;
    cov.x = __fadd_rn(__fmaf_rn(T02, A20, __fmaf_rn(T00, A00, __fmul_rn(T01, A10))), 0.3f);
    cov.y = __fmaf_rn(T02, A21, __fmaf_rn(T00, A01, __fmul_rn(T01, A11)));
    cov.z = __fadd_rn(__fmaf_rn(T12, A21, __fmaf_rn(T10, A01, __fmul_rn(T11, A11))), 0.3f);
    return cov;
}

// ndc2Pix is evaluated in double by the reference (double literals, auxiliary.h:41-44); nvcc fuses
// (v+1.0)*S-1.0 into one DFMA.
__device__ __forceinline__ float ndc_to_pix(float v, int S) {
    return (float)__dmul_rn(__fma_rn(__dadd_rn((double)v, 1.0), (double)S, -1.0), 0.5);
}

__global__ void __launch_bounds__(kProjThreads)
project_kernel(int P,
               const float* __restrict__ means3D, const float* __restrict__ opacities,
               const float* __restrict__ scales, const float4* __restrict__ rotations,
               const float* __restrict__ cov3D_precomp,
               const float* __restrict__ viewmatrix, const float* __restrict__ projmatrix,
               int W, int H, float tan_fovx, float tan_fovy, float focal_x, float focal_y,
               float scale_modifier, uint32_t grid_x, uint32_t grid_y, bool prefiltered,
               bool means_al16, bool scales_al16, bool rot_al16,
               int32_t* __restrict__ radii, uint32_t* __restrict__ depth_key,
               uint32_t* __restrict__ tiles_touched, float4* __restrict__ geom, uint2* __restrict__ rect) {
    __shared__ __align__(16) float s_mean[kProjThreads * 3];
    __shared__ __align__(16) float s_scale[kProjThreads * 3];
    __shared__ float s_vm[16], s_pm[16];
    const int first = blockIdx.x * kProjThreads;
    stage_aos3(s_mean, means3D, first, P, means_al16);
    if (scales != nullptr) stage_aos3(s_scale, scales, first, P, scales_al16);
    if (threadIdx.x < 16) s_vm[threadIdx.x] = __ldg(viewmatrix + threadIdx.x);
    else if (threadIdx.x < 32) s_pm[threadIdx.x - 16] = __ldg(projmatrix + threadIdx.x - 16);
    __syncthreads();

    // Near-plane test for every Gaussian, then block-level compaction of the survivors: a Gaussian behind the camera
    // only gets its four "culled" words written, and the projection / covariance path below runs on whole warps of
    // survivors instead of dragging every warp through it for a few live lanes (a SLAM map seen from one frame
    // has a large share of its Gaussians behind or beside the camera).
    __shared__ uint16_t s_list[kProjThreads];
    __shared__ uint32_t s_wcount[kProjThreads / 32];
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    const int gidx = first + tid;
    bool front = false;
    if (gidx < P) {
        front = xform_row(s_vm, 2, s_mean[3 * tid], s_mean[3 * tid + 1], s_mean[3 * tid + 2]) > 0.2f;
        if (!front) {
            // in_frustum(): a culled point with `prefiltered` set traps in the reference (auxiliary.h:156-160).
            if (prefiltered) __trap();
            radii[gidx] = 0;
#ifndef SB_PROBE_PROJECT_RADII_ONLY
            depth_key[gidx] = kCulledKey;
            tiles_touched[gidx] = 0u;
#endif
        }
    }
    const uint32_t ball = __ballot_sync(0xffffffffu, front);
    if (lane == 0) s_wcount[wid] = (uint32_t)__popc(ball);
    __syncthreads();
    uint32_t base = 0, total = 0;
#pragma unroll
    for (int w = 0; w < kProjThreads / 32; ++w) { const uint32_t c = s_wcount[w]; base += (w < wid) ? c : 0u; total += c; }
    if (front) s_list[base + __popc(ball & ((1u << lane) - 1u))] = (uint16_t)tid;
    __syncthreads();
    if ((uint32_t)tid >= total) return;
    const int src = (int)s_list[tid];              // this thread now owns Gaussian first + src (in front of the camera)
    const int idx = first + src;

    int32_t out_radius = 0;
    uint32_t out_tiles = 0, out_key = kCulledKey;
    float4 gA = make_float4(0.f, 0.f, -1.f, -1.f), gB = make_float4(0.f, 0.f, 0.f, 0.f);
    uint2 out_rect = make_uint2(0u, 0u);

    const float px = s_mean[3 * src], py = s_mean[3 * src + 1], pz = s_mean[3 * src + 2];
    const float depth = xform_row(s_vm, 2, px, py, pz);
    {
        const float hom_x = xform_row(s_pm, 0, px, py, pz);
        const float hom_y = xform_row(s_pm, 1, px, py, pz);
        const float hom_w = xform_row(s_pm, 3, px, py, pz);
        const float p_w = __frcp_rn(__fadd_rn(hom_w, 0.0000001f));
        const float proj_x = __fmul_rn(hom_x, p_w), proj_y = __fmul_rn(hom_y, p_w);

        Cov3 c3;
        if (cov3D_precomp != nullptr) {
            const float* c = cov3D_precomp + (size_t)idx * 6;
            c3.c0 = __ldg(c); c3.c1 = __ldg(c + 1); c3.c2 = __ldg(c + 2);
            c3.c3 = __ldg(c + 3); c3.c4 = __ldg(c + 4); c3.c5 = __ldg(c + 5);
        } else {
            float4 q;
            if (rot_al16) q = __ldg(rotations + idx);
            else { const float* rp = reinterpret_cast<const float*>(rotations) + (size_t)idx * 4;
                   q = make_float4(__ldg(rp), __ldg(rp + 1), __ldg(rp + 2), __ldg(rp + 3)); }
            c3 = cov3d_from_scale_rot(s_scale[3 * src], s_scale[3 * src + 1], s_scale[3 * src + 2], scale_modifier, q);
        }
        const float3 cov = cov2d_exact(px, py, pz, focal_x, focal_y, tan_fovx, tan_fovy, c3, s_vm);
        const float det = __fmaf_rn(cov.x, cov.z, -__fmul_rn(cov.y, cov.y));
        if (det != 0.0f) {
            const float det_inv = __frcp_rn(det);
            const float conic_x = __fmul_rn(cov.z, det_inv);
            const float conic_y = __fmul_rn(cov.y, -det_inv);
            const float conic_z = __fmul_rn(cov.x, det_inv);
            const float mid = __fmul_rn(__fadd_rn(cov.x, cov.z), 0.5f);
            const float root = __fsqrt_rn(fmaxf(__fmaf_rn(mid, mid, -det), 0.1f));
            const float lam = fmaxf(__fadd_rn(mid, root), __fsub_rn(mid, root));
            const int radius = __float2int_ru(__fmul_rn(__fsqrt_rn(lam), 3.f));
            const float rf = (float)radius;
            const float pix_x = ndc_to_pix(proj_x, W), pix_y = ndc_to_pix(proj_y, H);
            // getRect(): float math, truncating conversion, clamp to the grid (auxiliary.h:46-56)
            const int ix0 = (int)__fmul_rn(__fsub_rn(pix_x, rf), 0.0625f);
            const int iy0 = (int)__fmul_rn(__fsub_rn(pix_y, rf), 0.0625f);
            const int ix1 = (int)__fmul_rn(__fadd_rn(__fadd_rn(__fadd_rn(pix_x, rf), 16.f), -1.f), 0.0625f);
            const int iy1 = (int)__fmul_rn(__fadd_rn(__fadd_rn(__fadd_rn(pix_y, rf), 16.f), -1.f), 0.0625f);
            const uint32_t x0 = min(grid_x, (uint32_t)max(0, ix0)), y0 = min(grid_y, (uint32_t)max(0, iy0));
            const uint32_t x1 = min(grid_x, (uint32_t)max(0, ix1)), y1 = min(grid_y, (uint32_t)max(0, iy1));
            const uint32_t ntiles = (x1 - x0) * (y1 - y0);
            if (ntiles != 0u) {
                const float op = __ldg(opacities + idx);
                out_radius = radius;
                out_tiles = ntiles;
                out_key = __float_as_uint(depth);
                out_rect = make_uint2(x0 | (y0 << 16), x1 | (y1 << 16));
                // Conservative axis-aligned half-extents of the set of pixels that can pass the
                // reference's `alpha >= 1/255` test (forward.cu:342-350): q(d) = -power <= tau with
                // tau = ln(255*opacity), inflated by (a) 1e-3 absolute + 1e-3 relative slack, (b) a
                // bound on the float evaluation error of `power` over every pixel the reference can
                // pair with this Gaussian (|d| < radius + 16 in its tile rectangle).  hx = hy = -1
                // means "contributes nowhere" (opacity < 1/255); 1e30 means "do not cull".
                float hx = -1.f, hy = -1.f;
                if ((double)op * 255.0 >= 0.999) {
                    const double a = conic_x, b = conic_y, c = conic_z;
                    const double reach = (double)radius + 17.0;
                    const double eg = 4e-6 * (fabs(a) + fabs(c) + 2.0 * fabs(b)) * reach * reach;
                    double tau = log((double)op * 255.0);
                    tau = tau + 1e-3 + 1e-3 * fabs(tau) + eg;
                    const double dc = a * c - b * b;
                    if (dc > 0.0 && a > 0.0 && c > 0.0) {
                        hx = (float)(sqrt(2.0 * tau * c / dc) * 1.0001 + 2e-3);
                        hy = (float)(sqrt(2.0 * tau * a / dc) * 1.0001 + 2e-3);
                        if (!(hx < 1e30f)) hx = 1e30f;
                        if (!(hy < 1e30f)) hy = 1e30f;
                    } else {
                        hx = hy = 1e30f;
                    }
                }
                gA = make_float4(pix_x, pix_y, hx, hy);
                gB = make_float4(conic_x, conic_y, conic_z, op);
            }
        }
    }
#ifdef SB_PROBE_PROJECT_RADII_ONLY
    {   // tools/stage_bounds.py's variant: every result but the radius stays live (a store that is never taken), so
        // its time is the arithmetic and the input traffic without the geometry stores
        const uint32_t h = __float_as_uint(gA.x) ^ __float_as_uint(gA.y) ^ __float_as_uint(gA.z) ^
                           __float_as_uint(gA.w) ^ __float_as_uint(gB.x) ^ __float_as_uint(gB.y) ^
                           __float_as_uint(gB.z) ^ __float_as_uint(gB.w) ^ out_rect.x ^ out_rect.y ^ out_key ^ out_tiles;
        radii[idx] = h == 0x7fc00001u ? -1 : out_radius;
        return;
    }
#endif
    radii[idx] = out_radius;
    depth_key[idx] = out_key;
    tiles_touched[idx] = out_tiles;
    if (out_tiles != 0u) {          // geometry and rectangle are only ever read for Gaussians that touch a tile
        geom[2 * (size_t)idx] = gA;
        geom[2 * (size_t)idx + 1] = gB;
        rect[idx] = out_rect;
    }
}

__global__ void __launch_bounds__(256)
mark_visible_kernel(int P, const float* __restrict__ means3D, const float* __restrict__ vm,
                    uint8_t* __restrict__ present) {
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= P) return;
    const float px = __ldg(means3D + 3 * (size_t)idx), py = __ldg(means3D + 3 * (size_t)idx + 1),
                pz = __ldg(means3D + 3 * (size_t)idx + 2);
    present[idx] = (xform_row(vm, 2, px, py, pz) <= 0.2f) ? 0 : 1;  // in_frustum(): `!(z <= 0.2f)`
}

// header[0] = num_rendered, header[2] = 1 if it exceeds the caller's capacity (sync-free mode)
__global__ void finalize_count_kernel(const uint32_t* __restrict__ last_offset, int32_t* __restrict__ header, int cap) {
    const uint32_t R = *last_offset;
    header[0] = (int32_t)min(R, 0x7fffffffu);
    header[2] = (R > (uint32_t)cap) ? 1 : 0;
}

struct TilesInDepthOrder {
    const uint32_t* tiles_touched;
    const uint32_t* sorted_idx;
    __host__ __device__ __forceinline__ uint32_t operator()(uint32_t i) const {
        return tiles_touched[sorted_idx[i]];
    }
};

}  // namespace

size_t geometry_scan_temp_bytes(int P) {
    size_t scan_bytes = 0;
    TilesInDepthOrder op{nullptr, nullptr};
    cub::TransformInputIterator<uint32_t, TilesInDepthOrder, cub::CountingInputIterator<uint32_t>> it(
        cub::CountingInputIterator<uint32_t>(0u), op);
    cub::DeviceScan::InclusiveSum(nullptr, scan_bytes, it, (uint32_t*)nullptr, P);
    return scan_bytes;
}

int launch_project(const sb_settings& s, int P, const float* means3D, const float* opacities,
                   const float* scales, const float* rotations, const float* cov3D_precomp,
                   int32_t* radii, const GeometryWs& g, cudaStream_t st) {
    const int W = s.image_width, H = s.image_height;
    const float focal_y = H / (2.0f * s.tanfovy), focal_x = W / (2.0f * s.tanfovx);  // rasterizer_impl.cu:222-223
    const uint32_t gx = (W + kTile - 1) / kTile, gy = (H + kTile - 1) / kTile;
    auto al16 = [](const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; };
    ScopedStage _p(kStProject, st);
    project_kernel<<<(P + kProjThreads - 1) / kProjThreads, kProjThreads, 0, st>>>(
        P, means3D, opacities, scales, reinterpret_cast<const float4*>(rotations), cov3D_precomp,
        s.viewmatrix, s.projmatrix, W, H, s.tanfovx, s.tanfovy, focal_x, focal_y, s.scale_modifier,
        gx, gy, s.prefiltered != 0, al16(means3D), al16(scales), al16(rotations),
        radii, g.depth_key, g.tiles_touched, g.geom, g.rect);
    SB_LAUNCH_CHECK("project_kernel");
    return SB_OK;
}

// Orders the Gaussians by (depth bits, index) -- a stable LSD sort of P 32-bit keys -- and scans
// tiles_touched in that order.  A later stable sort of the emitted instances by tile id alone then
// reproduces the reference's single 64-bit (tile|depth) sort of rasterizer_impl.cu:304-309 exactly
// (ties in the reference resolve by emission order == Gaussian index).
int launch_depth_order(int P, const GeometryWs& g, cudaStream_t st) {
    { ScopedStage _p(kStDepthSort, st);
      // payload = the Gaussian's index, synthesised by the first pass; depth_key is left intact
      const int rc = radix_sort_pairs(g.depth_key, nullptr, g.sorted_key, g.sorted_idx, P, nullptr, 0, 32, g.sort_temp,
                                      g.sort_temp_bytes, st);
      if (rc != SB_OK) return rc; }
    TilesInDepthOrder op{g.tiles_touched, g.sorted_idx};
    cub::TransformInputIterator<uint32_t, TilesInDepthOrder, cub::CountingInputIterator<uint32_t>> it(
        cub::CountingInputIterator<uint32_t>(0u), op);
    size_t tb = g.scan_temp_bytes;
    ScopedStage _p(kStDepthScan, st);
    SB_CUDA_CHECK(cub::DeviceScan::InclusiveSum(g.scan_temp, tb, it, g.offsets, P, st));
    return SB_OK;
}

int launch_finalize_count(int P, const GeometryWs& g, int capacity, cudaStream_t st) {
    finalize_count_kernel<<<1, 1, 0, st>>>(g.offsets + (P - 1), g.header, capacity);
    SB_LAUNCH_CHECK("finalize_count_kernel");
    return SB_OK;
}

int launch_mark_visible(int P, const float* means3D, const float* viewmatrix, uint8_t* present,
                        cudaStream_t st) {
    mark_visible_kernel<<<(P + 255) / 256, 256, 0, st>>>(P, means3D, viewmatrix, present);
    SB_LAUNCH_CHECK("mark_visible_kernel");
    return SB_OK;
}

}  // namespace sb
