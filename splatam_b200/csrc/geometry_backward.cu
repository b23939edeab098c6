// geometry_backward.cu -- per-Gaussian tail of the backward: conic -> cov2D -> {cov3D, mean3D},
// mean2D -> mean3D through the projection, cov3D -> {scale, quaternion}
// (computeCov2DCUDA, BACKWARD::preprocessCUDA, computeCov3D of X/cuda_rasterizer/backward.cu:144-396),
// fused into ONE kernel that also unpacks the blend accumulator rows into the six gradient tensors
// SplaTAM consumes (so none of them needs a zero-fill; the reference zero-fills nine,
// X/rasterize_points.cu:150-158).  cov3D is recomputed from scale/quaternion instead of being
// round-tripped through HBM (the reference stores 24 B per Gaussian in forward to re-read here).
#include "common.cuh"

namespace sb {

namespace {

// Gaussians (threads) per block.  Each block loads, computes, then stores through its shared-memory stage; registers
// allow 24 resident warps per SM, and small blocks keep those phases of different blocks overlapping (on the H100,
// config 3: 0.078 ms at 256, 0.075 at 128, 0.074 at 64).
constexpr int kGbThreads = 64;

// Block-wide copy of n staged floats to dst[off .. off+n): 16-byte stores when the destination is 16-byte aligned
// (off is a multiple of kGbThreads rows, so only the array base decides), scalar stores for the tail / unaligned bases.
__device__ __forceinline__ void copy_out(float* __restrict__ dst, const float* __restrict__ stage, size_t off, int n,
                                         int tid) {
    float* d = dst + off;
    int done = 0;
    if ((reinterpret_cast<uintptr_t>(d) & 15u) == 0u) {
        const int n4 = n >> 2;
        for (int i = tid; i < n4; i += kGbThreads)
            reinterpret_cast<float4*>(d)[i] = reinterpret_cast<const float4*>(stage)[i];
        done = n4 << 2;
    }
    for (int i = done + tid; i < n; i += kGbThreads) d[i] = stage[i];
}

__global__ void __launch_bounds__(kGbThreads, 768 / kGbThreads)
geometry_backward_kernel(int P, const float* __restrict__ means3D, const float* __restrict__ colors,
                         const float* __restrict__ scales, const float* __restrict__ rotations,
                         const float* __restrict__ cov3D_precomp, const int32_t* __restrict__ radii,
                         const float* __restrict__ view, const float* __restrict__ proj,
                         float h_x, float h_y, float tan_fovx, float tan_fovy, float mod,
                         const float* __restrict__ accum, int accum_stride,
                         float* __restrict__ dL_dmeans3D, float* __restrict__ dL_dmeans2D,
                         float* __restrict__ dL_dcolors, float* __restrict__ dL_dcolors2,
                         float* __restrict__ dL_dopacity,
                         float* __restrict__ dL_dscales, float* __restrict__ dL_drot,
                         float* __restrict__ dL_dcov3D) {
    (void)colors;
    __shared__ float vm[16], pm[16];
    __shared__ uint16_t s_list[kGbThreads];
    __shared__ uint32_t s_wcount[kGbThreads / 32];
    if (threadIdx.x < 16) vm[threadIdx.x] = __ldg(view + threadIdx.x);
    else if (threadIdx.x < 32) pm[threadIdx.x - 16] = __ldg(proj + threadIdx.x - 16);
    // Block-level compaction of the visible Gaussians.  Off-screen Gaussians only get zeros written; when most of
    // the map is off-screen (a SLAM map seen from one frame) a visible lane would otherwise drag its whole warp
    // through the ~800-instruction path below at 1/32 utilisation.  Compacted, the visible ones fill whole warps.
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    const int gidx = blockIdx.x * kGbThreads + tid;
    const bool vis = gidx < P && radii[gidx] > 0;
    const uint32_t ball = __ballot_sync(0xffffffffu, vis);
    if (lane == 0) s_wcount[wid] = (uint32_t)__popc(ball);
    __syncthreads();
    uint32_t base = 0, total = 0;
#pragma unroll
    for (int w = 0; w < kGbThreads / 32; ++w) { const uint32_t c = s_wcount[w]; base += (w < wid) ? c : 0u; total += c; }
    if (vis) s_list[base + __popc(ball & ((1u << lane) - 1u))] = (uint16_t)tid;
    __syncthreads();
    // Outputs are staged in shared memory (one slot per Gaussian of the block) and written out by the whole block
    // with contiguous 16-byte stores: the per-thread AoS stores (3-6 strided scalar stores per array) cost ~3x the
    // L2 write transactions of the bytes they move, and this kernel is store-bound when most Gaussians are culled.
    __shared__ __align__(16) float s_o3[5][3 * kGbThreads];      // means3D, means2D, colors, colors2, scales
    __shared__ __align__(16) float s_rot[4 * kGbThreads];
    __shared__ __align__(16) float s_cov[6 * kGbThreads];
    __shared__ __align__(16) float s_op[kGbThreads];
    if (gidx < P && !vis) {
#pragma unroll
        for (int a = 0; a < 5; ++a) { s_o3[a][3 * tid] = 0.f; s_o3[a][3 * tid + 1] = 0.f; s_o3[a][3 * tid + 2] = 0.f; }
        s_rot[4 * tid] = 0.f; s_rot[4 * tid + 1] = 0.f; s_rot[4 * tid + 2] = 0.f; s_rot[4 * tid + 3] = 0.f;
        s_op[tid] = 0.f;
        if (dL_dcov3D) {
#pragma unroll
            for (int k = 0; k < 6; ++k) s_cov[6 * tid + k] = 0.f;
        }
    }
    const bool has_work = (uint32_t)tid < total;
    const int src = has_work ? (int)s_list[tid] : 0;
    const int idx = blockIdx.x * kGbThreads + src;                     // a visible Gaussian (radii[idx] > 0) when has_work
    const size_t i3 = 3 * (size_t)idx, i4 = 4 * (size_t)idx, i6 = 6 * (size_t)idx;

    float gm[3] = {0.f, 0.f, 0.f}, gm2[2] = {0.f, 0.f}, gc[3] = {0.f, 0.f, 0.f}, gop = 0.f;
    float gc2[3] = {0.f, 0.f, 0.f}, gm2_out[2] = {0.f, 0.f};   // second colour set; means2D sink (first set only)
    float gs[3] = {0.f, 0.f, 0.f}, gq[4] = {0.f, 0.f, 0.f, 0.f}, gcov[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};

    if (has_work) {
        const float4* arow = reinterpret_cast<const float4*>(accum + (size_t)idx * accum_stride);
        const float4 a0 = __ldg(arow), a1 = __ldg(arow + 1), a2 = __ldg(arow + 2);
        gm2[0] = a0.x; gm2[1] = a0.y;
        gm2_out[0] = a0.x; gm2_out[1] = a0.y;
        const float dconic_x = a0.z, dconic_y = a0.w, dconic_z = a1.x;
        gop = a1.y; gc[0] = a1.z; gc[1] = a1.w; gc[2] = a2.x;
        if (accum_stride == kAccumStride2) {
            const float4 a3 = __ldg(arow + 3);
            gc2[0] = a2.y; gc2[1] = a2.z; gc2[2] = a2.w;
            gm2_out[0] = a3.x; gm2_out[1] = a3.y;
        }

        const float mx = __ldg(means3D + i3), my = __ldg(means3D + i3 + 1), mz = __ldg(means3D + i3 + 2);

        // ---- 3D covariance (recomputed) and the pieces its backward needs ----
        float c3[6];
        float R[3][3] = {{0.f}}, M[3][3] = {{0.f}}, s[3] = {0.f, 0.f, 0.f};   // [c][r]
        float qr = 0.f, qx = 0.f, qy = 0.f, qz = 0.f;
        const bool from_scale_rot = (cov3D_precomp == nullptr);
        if (from_scale_rot) {
            qr = __ldg(rotations + i4); qx = __ldg(rotations + i4 + 1);
            qy = __ldg(rotations + i4 + 2); qz = __ldg(rotations + i4 + 3);
            s[0] = mod * __ldg(scales + i3); s[1] = mod * __ldg(scales + i3 + 1); s[2] = mod * __ldg(scales + i3 + 2);
            R[0][0] = 1.f - 2.f * (qy * qy + qz * qz); R[0][1] = 2.f * (qx * qy - qr * qz); R[0][2] = 2.f * (qx * qz + qr * qy);
            R[1][0] = 2.f * (qx * qy + qr * qz); R[1][1] = 1.f - 2.f * (qx * qx + qz * qz); R[1][2] = 2.f * (qy * qz - qr * qx);
            R[2][0] = 2.f * (qx * qz - qr * qy); R[2][1] = 2.f * (qy * qz + qr * qx); R[2][2] = 1.f - 2.f * (qx * qx + qy * qy);
#pragma unroll
            for (int c = 0; c < 3; ++c)
#pragma unroll
                for (int r = 0; r < 3; ++r) M[c][r] = s[r] * R[c][r];
            // Sigma[c][r] = sum_k M[r][k] * M[c][k]
            c3[0] = M[0][0] * M[0][0] + M[0][1] * M[0][1] + M[0][2] * M[0][2];
            c3[1] = M[0][0] * M[1][0] + M[0][1] * M[1][1] + M[0][2] * M[1][2];
            c3[2] = M[0][0] * M[2][0] + M[0][1] * M[2][1] + M[0][2] * M[2][2];
            c3[3] = M[1][0] * M[1][0] + M[1][1] * M[1][1] + M[1][2] * M[1][2];
            c3[4] = M[1][0] * M[2][0] + M[1][1] * M[2][1] + M[1][2] * M[2][2];
            c3[5] = M[2][0] * M[2][0] + M[2][1] * M[2][1] + M[2][2] * M[2][2];
        } else {
#pragma unroll
            for (int k = 0; k < 6; ++k) c3[k] = __ldg(cov3D_precomp + i6 + k);
        }

        // ---- computeCov2DCUDA (backward.cu:144-274) ----
        float tx = vm[0] * mx + vm[4] * my + vm[8] * mz + vm[12];
        float ty = vm[1] * mx + vm[5] * my + vm[9] * mz + vm[13];
        const float tz = vm[2] * mx + vm[6] * my + vm[10] * mz + vm[14];
        const float limx = 1.3f * tan_fovx, limy = 1.3f * tan_fovy;
        const float txtz = tx / tz, tytz = ty / tz;
        tx = fminf(limx, fmaxf(-limx, txtz)) * tz;
        ty = fminf(limy, fmaxf(-limy, tytz)) * tz;
        const float x_grad_mul = (txtz < -limx || txtz > limx) ? 0.f : 1.f;
        const float y_grad_mul = (tytz < -limy || tytz > limy) ? 0.f : 1.f;
        const float J00 = h_x / tz, J02 = -(h_x * tx) / (tz * tz), J11 = h_y / tz, J12 = -(h_y * ty) / (tz * tz);
        // T[c][r] = W[0][r]*J[c][0] + W[1][r]*J[c][1] + W[2][r]*J[c][2],  W[k][r] = vm[k + 4r]
        const float T00 = vm[0] * J00 + vm[2] * J02, T01 = vm[4] * J00 + vm[6] * J02, T02 = vm[8] * J00 + vm[10] * J02;
        const float T10 = vm[1] * J11 + vm[2] * J12, T11 = vm[5] * J11 + vm[6] * J12, T12 = vm[9] * J11 + vm[10] * J12;
        // rows of T^T * Vrk: u0k = sum_j T0j V[j][k], u1k = sum_j T1j V[j][k]
        const float u00 = T00 * c3[0] + T01 * c3[1] + T02 * c3[2];
        const float u01 = T00 * c3[1] + T01 * c3[3] + T02 * c3[4];
        const float u02 = T00 * c3[2] + T01 * c3[4] + T02 * c3[5];
        const float u10 = T10 * c3[0] + T11 * c3[1] + T12 * c3[2];
        const float u11 = T10 * c3[1] + T11 * c3[3] + T12 * c3[4];
        const float u12 = T10 * c3[2] + T11 * c3[4] + T12 * c3[5];
        const float a = u00 * T00 + u01 * T01 + u02 * T02 + 0.3f;
        const float b = u10 * T00 + u11 * T01 + u12 * T02;
        const float c = u10 * T10 + u11 * T11 + u12 * T12 + 0.3f;

        const float denom = a * c - b * b;
        float dL_da = 0.f, dL_db = 0.f, dL_dc = 0.f;
        const float denom2inv = 1.0f / ((denom * denom) + 0.0000001f);
        if (denom2inv != 0.f) {
            dL_da = denom2inv * (-c * c * dconic_x + 2.f * b * c * dconic_y + (denom - a * c) * dconic_z);
            dL_dc = denom2inv * (-a * a * dconic_z + 2.f * a * b * dconic_y + (denom - a * c) * dconic_x);
            dL_db = denom2inv * 2.f * (b * c * dconic_x - (denom + 2.f * b * b) * dconic_y + a * b * dconic_z);
            gcov[0] = T00 * T00 * dL_da + T00 * T10 * dL_db + T10 * T10 * dL_dc;
            gcov[3] = T01 * T01 * dL_da + T01 * T11 * dL_db + T11 * T11 * dL_dc;
            gcov[5] = T02 * T02 * dL_da + T02 * T12 * dL_db + T12 * T12 * dL_dc;
            gcov[1] = 2.f * T00 * T01 * dL_da + (T00 * T11 + T01 * T10) * dL_db + 2.f * T10 * T11 * dL_dc;
            gcov[2] = 2.f * T00 * T02 * dL_da + (T00 * T12 + T02 * T10) * dL_db + 2.f * T10 * T12 * dL_dc;
            gcov[4] = 2.f * T02 * T01 * dL_da + (T01 * T12 + T02 * T11) * dL_db + 2.f * T11 * T12 * dL_dc;
        }
        const float dT00 = 2.f * u00 * dL_da + u10 * dL_db, dT01 = 2.f * u01 * dL_da + u11 * dL_db,
                    dT02 = 2.f * u02 * dL_da + u12 * dL_db;
        const float dT10 = 2.f * u10 * dL_dc + u00 * dL_db, dT11 = 2.f * u11 * dL_dc + u01 * dL_db,
                    dT12 = 2.f * u12 * dL_dc + u02 * dL_db;
        const float dJ00 = vm[0] * dT00 + vm[4] * dT01 + vm[8] * dT02;
        const float dJ02 = vm[2] * dT00 + vm[6] * dT01 + vm[10] * dT02;
        const float dJ11 = vm[1] * dT10 + vm[5] * dT11 + vm[9] * dT12;
        const float dJ12 = vm[2] * dT10 + vm[6] * dT11 + vm[10] * dT12;
        const float itz = 1.f / tz, itz2 = itz * itz, itz3 = itz2 * itz;
        const float dtx = x_grad_mul * -h_x * itz2 * dJ02;
        const float dty = y_grad_mul * -h_y * itz2 * dJ12;
        const float dtz = -h_x * itz2 * dJ00 - h_y * itz2 * dJ11 + (2.f * h_x * tx) * itz3 * dJ02 +
                          (2.f * h_y * ty) * itz3 * dJ12;
        gm[0] = vm[0] * dtx + vm[1] * dty + vm[2] * dtz;
        gm[1] = vm[4] * dtx + vm[5] * dty + vm[6] * dtz;
        gm[2] = vm[8] * dtx + vm[9] * dty + vm[10] * dtz;

        // ---- BACKWARD::preprocessCUDA: mean2D -> mean3D through the projection (backward.cu:366-387) ----
        const float hw_ = pm[3] * mx + pm[7] * my + pm[11] * mz + pm[15];
        const float m_w = 1.0f / (hw_ + 0.0000001f);
        const float mul1 = (pm[0] * mx + pm[4] * my + pm[8] * mz + pm[12]) * m_w * m_w;
        const float mul2 = (pm[1] * mx + pm[5] * my + pm[9] * mz + pm[13]) * m_w * m_w;
        gm[0] += (pm[0] * m_w - pm[3] * mul1) * gm2[0] + (pm[1] * m_w - pm[3] * mul2) * gm2[1];
        gm[1] += (pm[4] * m_w - pm[7] * mul1) * gm2[0] + (pm[5] * m_w - pm[7] * mul2) * gm2[1];
        gm[2] += (pm[8] * m_w - pm[11] * mul1) * gm2[0] + (pm[9] * m_w - pm[11] * mul2) * gm2[1];

        // ---- computeCov3D backward (backward.cu:278-341) ----
        if (from_scale_rot) {
            // dL_dSigma[c][r] (symmetric), dL_dM = 2 * M * dL_dSigma : dM[c][r] = sum_k 2 M[k][r] dS[c][k]
            const float dS[3][3] = {{gcov[0], 0.5f * gcov[1], 0.5f * gcov[2]},
                                    {0.5f * gcov[1], gcov[3], 0.5f * gcov[4]},
                                    {0.5f * gcov[2], 0.5f * gcov[4], gcov[5]}};
            float dM[3][3];
#pragma unroll
            for (int cc = 0; cc < 3; ++cc)
#pragma unroll
                for (int r = 0; r < 3; ++r)
                    dM[cc][r] = 2.f * (M[0][r] * dS[cc][0] + M[1][r] * dS[cc][1] + M[2][r] * dS[cc][2]);
            // dL_dscale_i = dot(Rt[i], dL_dMt[i]) = sum_r R[r][i] * dM[r][i]
#pragma unroll
            for (int i = 0; i < 3; ++i) gs[i] = R[0][i] * dM[0][i] + R[1][i] * dM[1][i] + R[2][i] * dM[2][i];
            // dMt[c][r] = s_c * dM[r][c], each product rounded on its own: a multiply fused into the differences
            // below would leave its rounding residue in them, so an isotropic Gaussian with an identity quaternion
            // (whose quaternion gradient is exactly zero) would get float noise that changes with the summation order
            // of the blend's atomics from run to run.
            float dMt[3][3];
#pragma unroll
            for (int cc = 0; cc < 3; ++cc)
#pragma unroll
                for (int r = 0; r < 3; ++r) dMt[cc][r] = __fmul_rn(s[cc], dM[r][cc]);
            gq[0] = 2.f * qz * (dMt[0][1] - dMt[1][0]) + 2.f * qy * (dMt[2][0] - dMt[0][2]) + 2.f * qx * (dMt[1][2] - dMt[2][1]);
            gq[1] = 2.f * qy * (dMt[1][0] + dMt[0][1]) + 2.f * qz * (dMt[2][0] + dMt[0][2]) + 2.f * qr * (dMt[1][2] - dMt[2][1]) - 4.f * qx * (dMt[2][2] + dMt[1][1]);
            gq[2] = 2.f * qx * (dMt[1][0] + dMt[0][1]) + 2.f * qr * (dMt[2][0] - dMt[0][2]) + 2.f * qz * (dMt[1][2] + dMt[2][1]) - 4.f * qy * (dMt[2][2] + dMt[0][0]);
            gq[3] = 2.f * qr * (dMt[0][1] - dMt[1][0]) + 2.f * qx * (dMt[2][0] + dMt[0][2]) + 2.f * qy * (dMt[1][2] + dMt[2][1]) - 4.f * qz * (dMt[1][1] + dMt[0][0]);
        }
    }

    if (has_work) {
        float* o;
        o = &s_o3[0][3 * src]; o[0] = gm[0]; o[1] = gm[1]; o[2] = gm[2];
        o = &s_o3[1][3 * src]; o[0] = gm2_out[0]; o[1] = gm2_out[1]; o[2] = 0.f;
        o = &s_o3[2][3 * src]; o[0] = gc[0]; o[1] = gc[1]; o[2] = gc[2];
        o = &s_o3[3][3 * src]; o[0] = gc2[0]; o[1] = gc2[1]; o[2] = gc2[2];
        o = &s_o3[4][3 * src]; o[0] = gs[0]; o[1] = gs[1]; o[2] = gs[2];
        o = &s_rot[4 * src]; o[0] = gq[0]; o[1] = gq[1]; o[2] = gq[2]; o[3] = gq[3];
        s_op[src] = gop;
        if (dL_dcov3D) {
#pragma unroll
            for (int k = 0; k < 6; ++k) s_cov[6 * src + k] = gcov[k];
        }
    }
    __syncthreads();
    const int rows = min(kGbThreads, P - blockIdx.x * kGbThreads);
    const size_t row0 = (size_t)blockIdx.x * kGbThreads;
    copy_out(dL_dmeans3D, s_o3[0], row0 * 3, rows * 3, tid);
    copy_out(dL_dmeans2D, s_o3[1], row0 * 3, rows * 3, tid);
    copy_out(dL_dcolors, s_o3[2], row0 * 3, rows * 3, tid);
    if (dL_dcolors2) copy_out(dL_dcolors2, s_o3[3], row0 * 3, rows * 3, tid);
    if (dL_dscales) copy_out(dL_dscales, s_o3[4], row0 * 3, rows * 3, tid);
    if (dL_drot) copy_out(dL_drot, s_rot, row0 * 4, rows * 4, tid);
    copy_out(dL_dopacity, s_op, row0, rows, tid);
    if (dL_dcov3D) copy_out(dL_dcov3D, s_cov, row0 * 6, rows * 6, tid);
}

}  // namespace

int launch_geometry_backward(const sb_settings& s, int P, const float* means3D, const float* colors,
                             const float* scales, const float* rotations, const float* cov3D_precomp,
                             const int32_t* radii, const float* accum, int accum_stride,
                             float* dL_dmeans3D, float* dL_dmeans2D, float* dL_dcolors, float* dL_dcolors2,
                             float* dL_dopacity, float* dL_dscales, float* dL_drotations,
                             float* dL_dcov3D, cudaStream_t st) {
    const float focal_y = s.image_height / (2.0f * s.tanfovy), focal_x = s.image_width / (2.0f * s.tanfovx);
    ScopedStage _p(kStGeomBwd, st);
    geometry_backward_kernel<<<(P + kGbThreads - 1) / kGbThreads, kGbThreads, 0, st>>>(
        P, means3D, colors, scales, rotations, cov3D_precomp, radii, s.viewmatrix, s.projmatrix, focal_x,
        focal_y, s.tanfovx, s.tanfovy, s.scale_modifier, accum, accum_stride, dL_dmeans3D, dL_dmeans2D, dL_dcolors,
        dL_dcolors2, dL_dopacity, dL_dscales, dL_drotations, dL_dcov3D);
    SB_LAUNCH_CHECK("geometry_backward_kernel");
    return SB_OK;
}

}  // namespace sb
