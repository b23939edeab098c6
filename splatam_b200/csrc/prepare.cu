// prepare.cu -- SplaTAM's per-iteration PyTorch glue around the rasterizer as two kernels
// (SURVEY.md section 8(f) row N2; reference: transform_to_frame, transformed_params2rendervar,
// transformed_params2depthplussilhouette, get_depth_and_silhouette -- R/utils/slam_helpers.py:124-139,
// 196-304 -- about 20 elementwise kernels plus a 4x4 sgemm over P points, twice with autograd).
//
// forward : raw parameters (world means, un-normalised quaternions, logit opacities, log scales) + the
//           frame's rel_w2c  ->  the five operator inputs (camera-frame means, normalised rotations,
//           sigmoid opacities, exp scales tiled x3) and the depth/silhouette colours [z, 1, z^2].
// backward: gradients of those six tensors -> gradients of the raw parameters, plus the 3x4 gradient
//           of rel_w2c and the gradient of the (normalised) camera quaternion, block-reduced in double and
//           added with 16 double atomics per CTA (camera-pose gradients for tracking: at SplaTAM's map sizes
//           these are sums of ~1M products that cancel most of each other once tracking has converged).
#include "common.cuh"

namespace sb {

namespace {

struct Quat { float w, x, y, z; };

__device__ __forceinline__ Quat qmul(const Quat& a, const Quat& b) {   // Hamilton product (slam_helpers.py:24-31)
    return {a.w * b.w - a.x * b.x - a.y * b.y - a.z * b.z, a.w * b.x + a.x * b.w + a.y * b.z - a.z * b.y,
            a.w * b.y - a.x * b.z + a.y * b.w + a.z * b.x, a.w * b.z + a.x * b.y - a.y * b.x + a.z * b.w};
}
// F.normalize: x / max(|x|, 1e-12).  The returned inverse norm is negative when the clamp is active (|x| < 1e-12):
// the divisor is then the constant 1e-12 and the backward must not project out the radial component.
__device__ __forceinline__ Quat qnormalize(const Quat& q, float* inv_norm) {
    const float r = sqrtf(q.w * q.w + q.x * q.x + q.y * q.y + q.z * q.z);
    const float inv = 1.f / fmaxf(r, 1e-12f);
    *inv_norm = r < 1e-12f ? -inv : inv;
    return {q.w * inv, q.x * inv, q.y * inv, q.z * inv};
}
// backward of y = x/|x| : g_x = (g_y - y (y.g_y)) / |x| ; of the clamped branch y = x/1e-12 : g_x = g_y / 1e-12
__device__ __forceinline__ Quat qnormalize_bwd(const Quat& y, float inv_norm, const Quat& g) {
    const float d = inv_norm < 0.f ? 0.f : y.w * g.w + y.x * g.x + y.y * g.y + y.z * g.z;
    const float inv = fabsf(inv_norm);
    return {(g.w - y.w * d) * inv, (g.x - y.x * d) * inv, (g.y - y.y * d) * inv, (g.z - y.z * d) * inv};
}

__global__ void __launch_bounds__(256)
prepare_forward_kernel(int P, int scale_dim, const float* __restrict__ means, const float* __restrict__ unnorm,
                       const float* __restrict__ logit, const float* __restrict__ log_scales,
                       const float* __restrict__ rel, const float* __restrict__ cam_rot,
                       const float* __restrict__ w2c0, float* __restrict__ means_cam, float* __restrict__ rot,
                       float* __restrict__ opac, float* __restrict__ scales3, float* __restrict__ dcols) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P) return;
    const size_t i3 = 3 * (size_t)i, i4 = 4 * (size_t)i;
    const float px = __ldg(means + i3), py = __ldg(means + i3 + 1), pz = __ldg(means + i3 + 2);
    const float cx = rel[0] * px + rel[1] * py + rel[2] * pz + rel[3];
    const float cy = rel[4] * px + rel[5] * py + rel[6] * pz + rel[7];
    const float cz = rel[8] * px + rel[9] * py + rel[10] * pz + rel[11];
    means_cam[i3] = cx; means_cam[i3 + 1] = cy; means_cam[i3 + 2] = cz;
    Quat u = {__ldg(unnorm + i4), __ldg(unnorm + i4 + 1), __ldg(unnorm + i4 + 2), __ldg(unnorm + i4 + 3)};
    float inv;
    Quat q = qnormalize(u, &inv);
    if (scale_dim == 3) {   // anisotropic: rotate into the camera frame, then the rendervar's normalize
        const Quat c = {cam_rot[0], cam_rot[1], cam_rot[2], cam_rot[3]};
        q = qnormalize(qmul(c, q), &inv);
    }
    rot[i4] = q.w; rot[i4 + 1] = q.x; rot[i4 + 2] = q.y; rot[i4 + 3] = q.z;
    opac[i] = 1.f / (1.f + expf(-__ldg(logit + i)));
    if (scale_dim == 1) {
        const float s = expf(__ldg(log_scales + i));
        scales3[i3] = s; scales3[i3 + 1] = s; scales3[i3 + 2] = s;
    } else {
        scales3[i3] = expf(__ldg(log_scales + i3)); scales3[i3 + 1] = expf(__ldg(log_scales + i3 + 1));
        scales3[i3 + 2] = expf(__ldg(log_scales + i3 + 2));
    }
    const float z = w2c0[8] * cx + w2c0[9] * cy + w2c0[10] * cz + w2c0[11];
    dcols[i3] = z; dcols[i3 + 1] = 1.f; dcols[i3 + 2] = z * z;
}

__global__ void __launch_bounds__(256)
prepare_backward_kernel(int P, int scale_dim, int want_pose, const float* __restrict__ means,
                        const float* __restrict__ unnorm, const float* __restrict__ rel,
                        const float* __restrict__ cam_rot, const float* __restrict__ w2c0,
                        const float* __restrict__ means_cam, const float* __restrict__ opac,
                        const float* __restrict__ scales3,
                        const float* __restrict__ g_means_cam, const float* __restrict__ g_rot,
                        const float* __restrict__ g_opac, const float* __restrict__ g_scales3,
                        const float* __restrict__ g_dcols,
                        float* __restrict__ g_means, float* __restrict__ g_unnorm, float* __restrict__ g_logit,
                        float* __restrict__ g_log_scales, double* __restrict__ g_pose /* [16]: 12 rel + 4 cam_rot */) {
    __shared__ double red[16][8];
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    float pose[16];
#pragma unroll
    for (int k = 0; k < 16; ++k) pose[k] = 0.f;
    if (i < P) {
        const size_t i3 = 3 * (size_t)i, i4 = 4 * (size_t)i;
        // camera-frame mean gradient, incl. the depth colours' dependence on z
        float gx = g_means_cam ? g_means_cam[i3] : 0.f, gy = g_means_cam ? g_means_cam[i3 + 1] : 0.f,
              gz = g_means_cam ? g_means_cam[i3 + 2] : 0.f;
        if (g_dcols) {
            const float cx = means_cam[i3], cy = means_cam[i3 + 1], cz = means_cam[i3 + 2];
            const float z = w2c0[8] * cx + w2c0[9] * cy + w2c0[10] * cz + w2c0[11];
            const float gzc = g_dcols[i3] + 2.f * z * g_dcols[i3 + 2];
            gx += w2c0[8] * gzc; gy += w2c0[9] * gzc; gz += w2c0[10] * gzc;
        }
        g_means[i3] = rel[0] * gx + rel[4] * gy + rel[8] * gz;
        g_means[i3 + 1] = rel[1] * gx + rel[5] * gy + rel[9] * gz;
        g_means[i3 + 2] = rel[2] * gx + rel[6] * gy + rel[10] * gz;
        if (want_pose) {
            const float px = __ldg(means + i3), py = __ldg(means + i3 + 1), pz = __ldg(means + i3 + 2);
            pose[0] = gx * px; pose[1] = gx * py; pose[2] = gx * pz; pose[3] = gx;
            pose[4] = gy * px; pose[5] = gy * py; pose[6] = gy * pz; pose[7] = gy;
            pose[8] = gz * px; pose[9] = gz * py; pose[10] = gz * pz; pose[11] = gz;
        }
        // opacity / scale
        const float op = opac[i];
        g_logit[i] = g_opac ? g_opac[i] * op * (1.f - op) : 0.f;
        if (scale_dim == 1) {
            g_log_scales[i] = g_scales3 ? (g_scales3[i3] + g_scales3[i3 + 1] + g_scales3[i3 + 2]) * scales3[i3] : 0.f;
        } else {
#pragma unroll
            for (int k = 0; k < 3; ++k) g_log_scales[i3 + k] = g_scales3 ? g_scales3[i3 + k] * scales3[i3 + k] : 0.f;
        }
        // rotation
        Quat g = {0.f, 0.f, 0.f, 0.f};
        if (g_rot) g = {g_rot[i4], g_rot[i4 + 1], g_rot[i4 + 2], g_rot[i4 + 3]};
        const Quat u = {__ldg(unnorm + i4), __ldg(unnorm + i4 + 1), __ldg(unnorm + i4 + 2), __ldg(unnorm + i4 + 3)};
        float inv1;
        const Quat y1 = qnormalize(u, &inv1);
        if (scale_dim == 3) {
            const Quat c = {cam_rot[0], cam_rot[1], cam_rot[2], cam_rot[3]};
            const Quat qm = qmul(c, y1);
            float inv2;
            const Quat y2 = qnormalize(qm, &inv2);
            const Quat gq = qnormalize_bwd(y2, inv2, g);
            // qm = c * y1 (Hamilton): d/dy1 = conj(c) * gq ; d/dc = gq * conj(y1)
            const Quat cc = {c.w, -c.x, -c.y, -c.z}, yc = {y1.w, -y1.x, -y1.y, -y1.z};
            g = qmul(cc, gq);
            if (want_pose) { const Quat gc = qmul(gq, yc); pose[12] = gc.w; pose[13] = gc.x; pose[14] = gc.y; pose[15] = gc.z; }
        }
        const Quat gu = qnormalize_bwd(y1, inv1, g);
        g_unnorm[i4] = gu.w; g_unnorm[i4 + 1] = gu.x; g_unnorm[i4 + 2] = gu.y; g_unnorm[i4 + 3] = gu.z;
    }
    if (!want_pose) return;
    // CTA reduction of the 16 pose sums in double: warp shuffle, then 8 warp partials in shared memory
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int k = 0; k < 16; ++k) {
        double v = pose[k];
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
        if (lane == 0) red[k][warp] = v;
    }
    __syncthreads();
    if (threadIdx.x < 16) {
        double v = 0.0;
#pragma unroll
        for (int w = 0; w < 8; ++w) v += red[threadIdx.x][w];
        atomicAdd(g_pose + threadIdx.x, v);
    }
}

}  // namespace

}  // namespace sb

using namespace sb;

extern "C" {

SB_API int sb_prepare_forward(int P, int scale_dim, const float* means3D, const float* unnorm_rotations,
                              const float* logit_opacities, const float* log_scales, const float* rel_w2c,
                              const float* cam_rot, const float* w2c0, float* means_cam, float* rotations,
                              float* opacities, float* scales3, float* depth_sil_colors, void* stream) {
    if (P < 0 || (scale_dim != 1 && scale_dim != 3)) return SB_ERR_BAD_ARG;
    if (P == 0) return SB_OK;
    if (!means3D || !unnorm_rotations || !logit_opacities || !log_scales || !rel_w2c || !cam_rot || !w2c0 ||
        !means_cam || !rotations || !opacities || !scales3 || !depth_sil_colors)
        return SB_ERR_BAD_ARG;
    prepare_forward_kernel<<<(P + 255) / 256, 256, 0, static_cast<cudaStream_t>(stream)>>>(
        P, scale_dim, means3D, unnorm_rotations, logit_opacities, log_scales, rel_w2c, cam_rot, w2c0, means_cam,
        rotations, opacities, scales3, depth_sil_colors);
    SB_LAUNCH_CHECK("prepare_forward_kernel");
    return SB_OK;
}

SB_API int sb_prepare_backward(int P, int scale_dim, int want_pose, const float* means3D,
                               const float* unnorm_rotations, const float* rel_w2c, const float* cam_rot,
                               const float* w2c0, const float* means_cam, const float* opacities,
                               const float* scales3, const float* g_means_cam, const float* g_rotations,
                               const float* g_opacities, const float* g_scales3, const float* g_depth_sil_colors,
                               float* g_means3D, float* g_unnorm_rotations, float* g_logit_opacities,
                               float* g_log_scales, double* g_pose16, void* stream) {
    if (P < 0 || (scale_dim != 1 && scale_dim != 3)) return SB_ERR_BAD_ARG;
    if (P == 0) return SB_OK;
    if (!means3D || !unnorm_rotations || !rel_w2c || !cam_rot || !w2c0 || !means_cam || !opacities || !scales3 ||
        !g_means3D || !g_unnorm_rotations || !g_logit_opacities || !g_log_scales || (want_pose && !g_pose16))
        return SB_ERR_BAD_ARG;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (want_pose) SB_CUDA_CHECK(cudaMemsetAsync(g_pose16, 0, 16 * sizeof(double), st));
    prepare_backward_kernel<<<(P + 255) / 256, 256, 0, st>>>(
        P, scale_dim, want_pose, means3D, unnorm_rotations, rel_w2c, cam_rot, w2c0, means_cam, opacities, scales3,
        g_means_cam, g_rotations, g_opacities, g_scales3, g_depth_sil_colors, g_means3D, g_unnorm_rotations,
        g_logit_opacities, g_log_scales, g_pose16);
    SB_LAUNCH_CHECK("prepare_backward_kernel");
    return SB_OK;
}

}  // extern "C"
