// eval_frames.cu -- the four images the reference's final and novel-view evaluations save per frame with
// save_frames=True (R/utils/eval_helpers.py:509-528, 755-774), as uint8 HWC RGB, the layout a PNG decodes into:
//   0  rendered RGB     cv2.imwrite of float32 clamp(im, 0, 1) * 255: saturate_cast<uchar>, i.e. round half to even,
//                       NaN -> 0
//   1  rendered depth   cv2.applyColorMap(np.clip(d / 6, 0, 1) * 255 -> astype(uint8), COLORMAP_JET), d = depth_sil[0]
//   2  ground-truth RGB as 0, from gt_im
//   3  ground-truth depth as 1, from gt_depth
// Every step is the float32 operation numpy / cv2 perform, rounded as they round: an IEEE division by 6 (not a
// multiply by a reciprocal), a float32 multiply by 255, a truncating cast.  The colormap is a 256-entry RGB table the
// caller passes (evaluate.jet_lut).
#include "common.cuh"

namespace sb {

namespace {

constexpr int kFramesThreads = 256;
constexpr int kFramesMaxBlocks = 1056;   // 132 SMs x 8

// cv2's saturate_cast<uchar>(float) of clamp(x, 0, 1) * 255: cvRound (round half to even); NaN -> 0
__device__ __forceinline__ uint8_t rgb_u8(float x) {
    if (!(x == x)) return 0;
    const float c = fminf(fmaxf(x, 0.f), 1.f);
    return (uint8_t)__float2int_rn(__fmul_rn(c, 255.f));
}

// np.clip(d / 6, 0, 1) * 255 cast to uint8 (truncation); numpy's NaN -> uint8 cast gives 0 on x86-64
__device__ __forceinline__ int depth_idx(float d) {
    const float n = __fdiv_rn(d, 6.f);
    if (!(n == n)) return 0;
    return (int)__fmul_rn(fminf(fmaxf(n, 0.f), 1.f), 255.f);
}

__global__ void __launch_bounds__(kFramesThreads)
eval_frames_kernel(const float* __restrict__ im, const float* __restrict__ depth, const float* __restrict__ gt_im,
                   const float* __restrict__ gt_depth, int HW, const uint8_t* __restrict__ lut,
                   uint8_t* __restrict__ out) {
    __shared__ uint8_t s_lut[256 * 3];
    for (int i = threadIdx.x; i < 256 * 3; i += blockDim.x) s_lut[i] = lut[i];
    __syncthreads();
    uint8_t* o_im = out;
    uint8_t* o_d = out + (size_t)3 * HW;
    uint8_t* o_gt = out + (size_t)6 * HW;
    uint8_t* o_gd = out + (size_t)9 * HW;
    for (int p = blockIdx.x * blockDim.x + threadIdx.x; p < HW; p += gridDim.x * blockDim.x) {
        const size_t q = (size_t)3 * p;
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            o_im[q + c] = rgb_u8(im[(size_t)c * HW + p]);
            o_gt[q + c] = rgb_u8(gt_im[(size_t)c * HW + p]);
        }
        const int a = 3 * depth_idx(depth[p]), b = 3 * depth_idx(gt_depth[p]);
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            o_d[q + c] = s_lut[a + c];
            o_gd[q + c] = s_lut[b + c];
        }
    }
}

}  // namespace

}  // namespace sb

using namespace sb;

extern "C" {

SB_API int sb_eval_frames_u8(const float* im, const float* depth_sil, const float* gt_im, const float* gt_depth, int H,
                             int W, const uint8_t* lut, uint8_t* out, void* stream) {
    if (!im || !depth_sil || !gt_im || !gt_depth || !lut || !out || H < 1 || W < 1 ||
        (long long)H * W >= (1LL << 31) / 12)
        return SB_ERR_BAD_ARG;
    const int HW = H * W;
    const int blocks = (HW + kFramesThreads - 1) / kFramesThreads < kFramesMaxBlocks
                           ? (HW + kFramesThreads - 1) / kFramesThreads : kFramesMaxBlocks;
    eval_frames_kernel<<<blocks, kFramesThreads, 0, static_cast<cudaStream_t>(stream)>>>(im, depth_sil, gt_im,
                                                                                        gt_depth, HW, lut, out);
    SB_LAUNCH_CHECK("eval_frames_kernel");
    return SB_OK;
}

}  // extern "C"
