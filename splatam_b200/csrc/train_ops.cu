// train_ops.cu -- the two per-iteration PyTorch costs that dominate SplaTAM's mapping step once the
// rasterizer is fast (SURVEY.md section 8(f) row N3), as hand-written kernels:
//   * fused Adam over the packed (flat) Gaussian parameter buffer with per-segment learning rates
//     (reference: torch.optim.Adam over 5-7 param groups, R/scripts/splatam.py:160-166,869);
//   * fused image loss  0.8*L1 + 0.2*(1-SSIM)  and its gradient w.r.t. the rendered image
//     (reference: l1_loss_v1 + calc_ssim, R/scripts/splatam.py:290, R/utils/slam_external.py:54-97 --
//     five depthwise 11x11 convolutions forward and their autograd backward).
#include "common.cuh"

namespace sb {

namespace {

constexpr int kMaxSeg = 16;
struct AdamSegs { uint32_t end[kMaxSeg]; float lr[kMaxSeg]; int n; };

// Device-resident optimizer clock of the guarded step: the step count only advances on steps that are applied, and the
// bias-correction scalars are formed from it on the device (one thread), so a skipped step leaves NO trace.
struct AdamClock { int t; int skipped; float bc2_sqrt; float neg_step[kMaxSeg]; };
struct AdamLrs { double lr[kMaxSeg]; int n; };

__global__ void adam_clock_kernel(AdamClock* __restrict__ clk, const float* __restrict__ skip_if_nonzero, AdamLrs segs,
                                  double beta1, double beta2) {
    if (skip_if_nonzero != nullptr && *skip_if_nonzero != 0.f) { clk->skipped += 1; return; }
    const int t = clk->t + 1;
    clk->t = t;
    const double bc1 = 1.0 - pow(beta1, (double)t), bc2 = 1.0 - pow(beta2, (double)t);
    clk->bc2_sqrt = (float)sqrt(bc2);
    for (int k = 0; k < segs.n; ++k) clk->neg_step[k] = (float)(-(segs.lr[k] / bc1));   // as sb_adam_step forms it
}

// GUARDED == true: the per-segment step sizes and bc2_sqrt come from the device clock and the whole update is a no-op
// when *skip_if_nonzero != 0 (the sync-free rasterizer overflowed its instance capacity: gradients are incomplete).
template <bool GUARDED>
__global__ void __launch_bounds__(256)
adam_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m, float* __restrict__ v,
            size_t n, AdamSegs segs, float w1, float beta2, float w2, float eps, float bc2_sqrt,
            const AdamClock* __restrict__ clk, const float* __restrict__ skip_if_nonzero) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    __shared__ float s_neg[kMaxSeg + 1];      // guarded mode: the clock's step sizes, fetched once per CTA
    if (GUARDED) {
        if (skip_if_nonzero != nullptr && __ldg(skip_if_nonzero) != 0.f) return;      // uniform over the grid
        if (threadIdx.x <= kMaxSeg) s_neg[threadIdx.x] = threadIdx.x < kMaxSeg ? clk->neg_step[threadIdx.x] : clk->bc2_sqrt;
        __syncthreads();
        bc2_sqrt = s_neg[kMaxSeg];
    }
    if (i >= n) return;
    float neg_step = 0.f;            // -(lr / bias_correction1) of this element's segment
#pragma unroll 4
    for (int k = 0; k < segs.n; ++k)
        if (i < segs.end[k]) { neg_step = GUARDED ? s_neg[k] : segs.lr[k]; break; }
    const float gi = g[i];
    // torch.optim.Adam's math, op for op: lerp_(g, 1-b1); mul_(b2).addcmul_(g, g, 1-b2); sqrt / bc2_sqrt + eps; addcdiv_
    const float mi = fmaf(w1, gi - m[i], m[i]);
    const float vi = fmaf(w2 * gi, gi, v[i] * beta2);
    m[i] = mi; v[i] = vi;
    const float denom = sqrtf(vi) / bc2_sqrt + eps;
    p[i] = fmaf(neg_step, mi / denom, p[i]);
}

// ---- fused 0.8*L1 + 0.2*(1-SSIM) ----------------------------------------------------------------------
constexpr int kTW = 32, kTH = 8, kR = 5, kWin = 11;     // output tile 32x8, 11-tap separable Gaussian
constexpr int kPW = kTW + 2 * kR, kPH = kTH + 2 * kR;   // padded tile 42 x 18
// The 11 window weights travel as a by-value kernel argument (constant bank of the launch): no per-device symbol to
// initialise, nothing to copy during a CUDA-graph capture, safe from any thread.
struct GaussWin { float w[kWin]; };

// Forward: per pixel/channel SSIM map terms; writes the three partial-derivative maps needed by the
// backward (dS/dmu1, dS/dE[x^2], dS/dE[xy]) and accumulates sum(ssim) and sum|x-y| into sums[0..1].  With `keep`
// (uint8 [H,W]) a pixel whose byte is 0 adds nothing and gets zero derivative maps, and sums[2] counts the kept pixels;
// NULL keeps every pixel and leaves sums[2] alone.
__global__ void __launch_bounds__(kTW * kTH)
ssim_l1_forward_kernel(const float* __restrict__ x, const float* __restrict__ y, int C, int H, int W,
                       float* __restrict__ dmu, float* __restrict__ de11, float* __restrict__ de12,
                       double* __restrict__ sums, const GaussWin win, const uint8_t* __restrict__ keep) {
    __shared__ float sx[kPH][kPW], sy[kPH][kPW];
    __shared__ float h[5][kPH][kTW];     // horizontally filtered x, y, xx, yy, xy
    __shared__ float red[3][kTW * kTH / 32];
    const int c = blockIdx.z, x0 = blockIdx.x * kTW, y0 = blockIdx.y * kTH;
    const float* xc = x + (size_t)c * H * W;
    const float* yc = y + (size_t)c * H * W;
    const int tid = threadIdx.y * kTW + threadIdx.x;
    for (int i = tid; i < kPH * kPW; i += kTW * kTH) {
        const int r = i / kPW, q = i % kPW, gy = y0 + r - kR, gx = x0 + q - kR;
        const bool in = gy >= 0 && gy < H && gx >= 0 && gx < W;          // zero padding (conv2d padding=5)
        sx[r][q] = in ? __ldg(xc + (size_t)gy * W + gx) : 0.f;
        sy[r][q] = in ? __ldg(yc + (size_t)gy * W + gx) : 0.f;
    }
    __syncthreads();
    for (int i = tid; i < kPH * kTW; i += kTW * kTH) {
        const int r = i / kTW, q = i % kTW;
        float a = 0.f, b = 0.f, aa = 0.f, bb = 0.f, ab = 0.f;
#pragma unroll
        for (int k = 0; k < kWin; ++k) {
            const float w = win.w[k], xv = sx[r][q + k], yv = sy[r][q + k];
            a = fmaf(w, xv, a); b = fmaf(w, yv, b);
            aa = fmaf(w, xv * xv, aa); bb = fmaf(w, yv * yv, bb); ab = fmaf(w, xv * yv, ab);
        }
        h[0][r][q] = a; h[1][r][q] = b; h[2][r][q] = aa; h[3][r][q] = bb; h[4][r][q] = ab;
    }
    __syncthreads();
    const int px = x0 + threadIdx.x, py = y0 + threadIdx.y;
    float ssim = 0.f, l1 = 0.f, kept = 0.f;
    if (px < W && py < H) {
        const bool k = keep == nullptr || keep[(size_t)py * W + px] != 0;
        kept = k ? 1.f : 0.f;
        float mu1 = 0.f, mu2 = 0.f, e11 = 0.f, e22 = 0.f, e12 = 0.f;
#pragma unroll
        for (int k = 0; k < kWin; ++k) {
            const float w = win.w[k];
            mu1 = fmaf(w, h[0][threadIdx.y + k][threadIdx.x], mu1);
            mu2 = fmaf(w, h[1][threadIdx.y + k][threadIdx.x], mu2);
            e11 = fmaf(w, h[2][threadIdx.y + k][threadIdx.x], e11);
            e22 = fmaf(w, h[3][threadIdx.y + k][threadIdx.x], e22);
            e12 = fmaf(w, h[4][threadIdx.y + k][threadIdx.x], e12);
        }
        const float C1 = 0.01f * 0.01f, C2 = 0.03f * 0.03f;
        const float s1 = e11 - mu1 * mu1, s2 = e22 - mu2 * mu2, s12 = e12 - mu1 * mu2;
        const float a1 = 2.f * mu1 * mu2 + C1, a2 = 2.f * s12 + C2, b1 = mu1 * mu1 + mu2 * mu2 + C1, b2 = s1 + s2 + C2;
        const float inv = 1.f / (b1 * b2);
        ssim = a1 * a2 * inv;
        const size_t o = (size_t)c * H * W + (size_t)py * W + px;
        // total derivatives w.r.t. mu1 (incl. through sigma terms), E[x^2], E[xy]
        dmu[o] = k ? 2.f * mu2 * (a2 - a1) * inv - ssim * 2.f * mu1 * (1.f / b1 - 1.f / b2) : 0.f;
        de11[o] = k ? -ssim / b2 : 0.f;
        de12[o] = k ? 2.f * a1 * inv : 0.f;
        l1 = k ? fabsf(sx[threadIdx.y + kR][threadIdx.x + kR] - sy[threadIdx.y + kR][threadIdx.x + kR]) : 0.f;
        ssim = k ? ssim : 0.f;
    }
    // block reduction of the two sums
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
        ssim += __shfl_xor_sync(0xffffffffu, ssim, off);
        l1 += __shfl_xor_sync(0xffffffffu, l1, off);
        kept += __shfl_xor_sync(0xffffffffu, kept, off);
    }
    if ((tid & 31) == 0) { red[0][tid >> 5] = ssim; red[1][tid >> 5] = l1; red[2][tid >> 5] = kept; }
    __syncthreads();
    if (tid == 0) {
        float a = 0.f, b = 0.f, n = 0.f;
        for (int i = 0; i < kTW * kTH / 32; ++i) { a += red[0][i]; b += red[1][i]; n += red[2][i]; }
        atomicAdd(&sums[0], (double)a);
        atomicAdd(&sums[1], (double)b);
        if (keep != nullptr && c == 0) atomicAdd(&sums[2], (double)n);
    }
}

// Backward: grad_x = gscale_ssim * (conv(dmu) + 2 x conv(de11) + y conv(de12)) + gscale_l1 * sign(x - y).  With
// `keep` the sign term is zero where keep is 0 and n = C * the kept count of the forward (sums[2]).
__global__ void __launch_bounds__(kTW * kTH)
ssim_l1_backward_kernel(const float* __restrict__ x, const float* __restrict__ y, const float* __restrict__ dmu,
                        const float* __restrict__ de11, const float* __restrict__ de12, int C, int H, int W,
                        const float* __restrict__ grad_out, float w_ssim, float w_l1, float* __restrict__ gx,
                        const GaussWin win, const uint8_t* __restrict__ keep, const double* __restrict__ sums) {
    __shared__ float s[3][kPH][kPW];
    __shared__ float h[3][kPH][kTW];
    const int c = blockIdx.z, x0 = blockIdx.x * kTW, y0 = blockIdx.y * kTH;
    const size_t plane = (size_t)c * H * W;
    const int tid = threadIdx.y * kTW + threadIdx.x;
    for (int i = tid; i < kPH * kPW; i += kTW * kTH) {
        const int r = i / kPW, q = i % kPW, gy = y0 + r - kR, gxx = x0 + q - kR;
        const bool in = gy >= 0 && gy < H && gxx >= 0 && gxx < W;
        const size_t o = plane + (size_t)gy * W + gxx;
        s[0][r][q] = in ? __ldg(dmu + o) : 0.f;
        s[1][r][q] = in ? __ldg(de11 + o) : 0.f;
        s[2][r][q] = in ? __ldg(de12 + o) : 0.f;
    }
    __syncthreads();
    for (int i = tid; i < kPH * kTW; i += kTW * kTH) {
        const int r = i / kTW, q = i % kTW;
        float a = 0.f, b = 0.f, d = 0.f;
#pragma unroll
        for (int k = 0; k < kWin; ++k) {
            const float w = win.w[k];
            a = fmaf(w, s[0][r][q + k], a); b = fmaf(w, s[1][r][q + k], b); d = fmaf(w, s[2][r][q + k], d);
        }
        h[0][r][q] = a; h[1][r][q] = b; h[2][r][q] = d;
    }
    __syncthreads();
    const int px = x0 + threadIdx.x, py = y0 + threadIdx.y;
    if (px >= W || py >= H) return;
    float a = 0.f, b = 0.f, d = 0.f;
#pragma unroll
    for (int k = 0; k < kWin; ++k) {
        const float w = win.w[k];
        a = fmaf(w, h[0][threadIdx.y + k][threadIdx.x], a);
        b = fmaf(w, h[1][threadIdx.y + k][threadIdx.x], b);
        d = fmaf(w, h[2][threadIdx.y + k][threadIdx.x], d);
    }
    const size_t o = plane + (size_t)py * W + px;
    const float xv = x[o], yv = y[o], go = __ldg(grad_out);
    // with `keep`, an empty kept set gives zero gradient (n >= C), not 0/0
    const float n = keep == nullptr ? (float)C * (float)H * (float)W : (float)C * (float)fmax(sums[2], 1.0);
    // loss = w_l1 * mean|x-y| + w_ssim * (1 - mean(ssim))
    const float diff = xv - yv;
    const bool k = keep == nullptr || keep[(size_t)py * W + px] != 0;
    const float sgn = !k ? 0.f : (diff > 0.f ? 1.f : (diff < 0.f ? -1.f : 0.f));
    gx[o] = go * (w_l1 * sgn / n - w_ssim * (a + 2.f * xv * b + yv * d) / n);
}

// ---- fused silhouette/validity-masked L1 losses of get_loss (R/scripts/splatam.py:254-288) ---------------
// mask = (gt_depth > 0) & !isnan(depth) & !isnan(depth_sq - depth^2) [& (silhouette > sil_thres)]
// sums[0] = sum |gt_depth - depth| * mask, sums[1] = sum mask, sums[2] = sum_ch |gt_im - im| * mask
__device__ __forceinline__ bool loss_mask(float gd, float d, float sil, float dsq, float sil_thres, int use_sil) {
    const float unc = dsq - d * d;
    bool m = gd > 0.f && !isnan(d) && !isnan(unc);
    if (use_sil) m = m && (sil > sil_thres);
    return m;
}

__global__ void __launch_bounds__(256)
masked_l1_forward_kernel(const float* __restrict__ depth_sil, const float* __restrict__ gt_depth,
                         const float* __restrict__ im, const float* __restrict__ gt_im, int HW, float sil_thres,
                         int use_sil, double* __restrict__ sums, const uint8_t* __restrict__ keep) {
    __shared__ float red[3][8];
    float sd = 0.f, sm = 0.f, si = 0.f;
    for (int p = blockIdx.x * blockDim.x + threadIdx.x; p < HW; p += gridDim.x * blockDim.x) {
        const float d = depth_sil[p], gd = gt_depth[p];
        if (loss_mask(gd, d, depth_sil[HW + p], depth_sil[2 * HW + p], sil_thres, use_sil) && (!keep || keep[p])) {
            sd += fabsf(gd - d); sm += 1.f;
            if (im) si += fabsf(gt_im[p] - im[p]) + fabsf(gt_im[HW + p] - im[HW + p]) + fabsf(gt_im[2 * HW + p] - im[2 * HW + p]);
        }
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
        sd += __shfl_xor_sync(0xffffffffu, sd, off); sm += __shfl_xor_sync(0xffffffffu, sm, off);
        si += __shfl_xor_sync(0xffffffffu, si, off);
    }
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (lane == 0) { red[0][warp] = sd; red[1][warp] = sm; red[2][warp] = si; }
    __syncthreads();
    if (threadIdx.x < 3) {
        float v = 0.f;
        for (int w = 0; w < 8; ++w) v += red[threadIdx.x][w];
        atomicAdd(&sums[threadIdx.x], (double)v);
    }
}

// grad_depth_sil[0] = g_d * sign(d - gt) * mask * (mean ? 1/count : 1); channels 1, 2 get zero (the uncertainty
// and the silhouette mask are detached in the reference); grad_im[ch] = g_i * sign(im - gt) * mask.
__global__ void __launch_bounds__(256)
masked_l1_backward_kernel(const float* __restrict__ depth_sil, const float* __restrict__ gt_depth,
                          const float* __restrict__ im, const float* __restrict__ gt_im, int HW, float sil_thres,
                          int use_sil, int depth_mean, const double* __restrict__ sums,
                          const float* __restrict__ g_depth, const float* __restrict__ g_im,
                          float* __restrict__ grad_depth_sil, float* __restrict__ grad_im,
                          const uint8_t* __restrict__ keep) {
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= HW) return;
    const float d = depth_sil[p], gd = gt_depth[p];
    const bool m = loss_mask(gd, d, depth_sil[HW + p], depth_sil[2 * HW + p], sil_thres, use_sil) && (!keep || keep[p]);
    float scale = g_depth ? __ldg(g_depth) : 0.f;
    if (depth_mean) scale = scale / (float)(keep ? fmax(sums[1], 1.0) : sums[1]);
    const float diff = d - gd;
    grad_depth_sil[p] = m ? scale * (diff > 0.f ? 1.f : (diff < 0.f ? -1.f : 0.f)) : 0.f;
    grad_depth_sil[HW + p] = 0.f;
    grad_depth_sil[2 * HW + p] = 0.f;
    if (grad_im) {
        const float gi = g_im ? __ldg(g_im) : 0.f;
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            const float df = im[c * HW + p] - gt_im[c * HW + p];
            grad_im[c * HW + p] = m ? gi * (df > 0.f ? 1.f : (df < 0.f ? -1.f : 0.f)) : 0.f;
        }
    }
}


}  // namespace

}  // namespace sb

using namespace sb;

extern "C" {

SB_API int sb_adam_step(float* params, const float* grads, float* exp_avg, float* exp_avg_sq, size_t n,
                        const uint32_t* seg_end, const double* seg_lr, int num_segments, int step, double beta1,
                        double beta2, double eps, void* stream) {
    if (!params || !grads || !exp_avg || !exp_avg_sq || !seg_end || !seg_lr || num_segments < 1 ||
        num_segments > kMaxSeg || step < 1)
        return SB_ERR_BAD_ARG;
    if (n == 0) return SB_OK;
    // scalars are formed in double and rounded to float once, as torch does with its Python-float hyper-parameters
    const double bc1 = 1.0 - pow(beta1, step), bc2 = 1.0 - pow(beta2, step);
    AdamSegs segs;
    segs.n = num_segments;
    for (int k = 0; k < num_segments; ++k) { segs.end[k] = seg_end[k]; segs.lr[k] = (float)(-(seg_lr[k] / bc1)); }
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    adam_kernel<false><<<(unsigned)((n + 255) / 256), 256, 0, st>>>(params, grads, exp_avg, exp_avg_sq, n, segs,
                                                                     (float)(1.0 - beta1), (float)beta2,
                                                                     (float)(1.0 - beta2), (float)eps, (float)sqrt(bc2),
                                                                     nullptr, nullptr);
    SB_LAUNCH_CHECK("adam_kernel");
    return SB_OK;
}

SB_API size_t sb_adam_clock_bytes(void) { return sizeof(AdamClock); }

SB_API int sb_adam_step_guarded(float* params, const float* grads, float* exp_avg, float* exp_avg_sq, size_t n,
                                const uint32_t* seg_end, const double* seg_lr, int num_segments, void* clock_dev,
                                const float* skip_if_nonzero, double beta1, double beta2, double eps, void* stream) {
    if (!params || !grads || !exp_avg || !exp_avg_sq || !seg_end || !seg_lr || !clock_dev || num_segments < 1 ||
        num_segments > kMaxSeg)
        return SB_ERR_BAD_ARG;
    if (n == 0) return SB_OK;
    AdamSegs segs;
    segs.n = num_segments;
    AdamLrs lrs;
    lrs.n = num_segments;
    for (int k = 0; k < num_segments; ++k) { segs.end[k] = seg_end[k]; segs.lr[k] = 0.f; lrs.lr[k] = seg_lr[k]; }
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    AdamClock* clk = static_cast<AdamClock*>(clock_dev);
    adam_clock_kernel<<<1, 1, 0, st>>>(clk, skip_if_nonzero, lrs, beta1, beta2);
    SB_LAUNCH_CHECK("adam_clock_kernel");
    adam_kernel<true><<<(unsigned)((n + 255) / 256), 256, 0, st>>>(params, grads, exp_avg, exp_avg_sq, n, segs,
                                                                    (float)(1.0 - beta1), (float)beta2,
                                                                    (float)(1.0 - beta2), (float)eps, 0.f, clk,
                                                                    skip_if_nonzero);
    SB_LAUNCH_CHECK("adam_kernel");
    return SB_OK;
}

/* sums: 3 device doubles (zeroed here).  im / gt_im may be NULL (mapping: the RGB term uses the SSIM loss). */
static int masked_l1_forward(const uint8_t* keep, const float* depth_sil, const float* gt_depth, const float* im,
                             const float* gt_im, int H, int W, float sil_thres, int use_sil, double* sums,
                             void* stream) {
    if (!depth_sil || !gt_depth || !sums || H < 1 || W < 1 || ((im != nullptr) != (gt_im != nullptr))) return SB_ERR_BAD_ARG;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    SB_CUDA_CHECK(cudaMemsetAsync(sums, 0, 3 * sizeof(double), st));
    const int HW = H * W;
    const int blocks = (HW + 255) / 256 < 528 ? (HW + 255) / 256 : 528;   // 132 SMs x 4
    masked_l1_forward_kernel<<<blocks, 256, 0, st>>>(depth_sil, gt_depth, im, gt_im, HW, sil_thres, use_sil, sums,
                                                     keep);
    SB_LAUNCH_CHECK("masked_l1_forward_kernel");
    return SB_OK;
}

static int masked_l1_backward(const uint8_t* keep, const float* depth_sil, const float* gt_depth, const float* im,
                              const float* gt_im, int H, int W, float sil_thres, int use_sil, int depth_mean,
                              const double* sums, const float* g_depth, const float* g_im, float* grad_depth_sil,
                              float* grad_im, void* stream) {
    if (!depth_sil || !gt_depth || !sums || !grad_depth_sil || H < 1 || W < 1) return SB_ERR_BAD_ARG;
    if (grad_im && (!im || !gt_im)) return SB_ERR_BAD_ARG;
    const int HW = H * W;
    masked_l1_backward_kernel<<<(HW + 255) / 256, 256, 0, static_cast<cudaStream_t>(stream)>>>(
        depth_sil, gt_depth, im, gt_im, HW, sil_thres, use_sil, depth_mean, sums, g_depth, g_im, grad_depth_sil, grad_im,
        keep);
    SB_LAUNCH_CHECK("masked_l1_backward_kernel");
    return SB_OK;
}

SB_API int sb_masked_l1_forward(const float* depth_sil, const float* gt_depth, const float* im, const float* gt_im,
                                int H, int W, float sil_thres, int use_sil, double* sums, void* stream) {
    return masked_l1_forward(nullptr, depth_sil, gt_depth, im, gt_im, H, W, sil_thres, use_sil, sums, stream);
}

SB_API int sb_masked_l1_backward(const float* depth_sil, const float* gt_depth, const float* im, const float* gt_im,
                                 int H, int W, float sil_thres, int use_sil, int depth_mean, const double* sums,
                                 const float* g_depth, const float* g_im, float* grad_depth_sil, float* grad_im,
                                 void* stream) {
    return masked_l1_backward(nullptr, depth_sil, gt_depth, im, gt_im, H, W, sil_thres, use_sil, depth_mean, sums,
                              g_depth, g_im, grad_depth_sil, grad_im, stream);
}

SB_API int sb_masked_l1_keep_forward(const uint8_t* keep, const float* depth_sil, const float* gt_depth,
                                     const float* im, const float* gt_im, int H, int W, float sil_thres, int use_sil,
                                     double* sums, void* stream) {
    if (!keep) return SB_ERR_BAD_ARG;
    return masked_l1_forward(keep, depth_sil, gt_depth, im, gt_im, H, W, sil_thres, use_sil, sums, stream);
}

SB_API int sb_masked_l1_keep_backward(const uint8_t* keep, const float* depth_sil, const float* gt_depth,
                                      const float* im, const float* gt_im, int H, int W, float sil_thres, int use_sil,
                                      int depth_mean, const double* sums, const float* g_depth, const float* g_im,
                                      float* grad_depth_sil, float* grad_im, void* stream) {
    if (!keep) return SB_ERR_BAD_ARG;
    return masked_l1_backward(keep, depth_sil, gt_depth, im, gt_im, H, W, sil_thres, use_sil, depth_mean, sums,
                              g_depth, g_im, grad_depth_sil, grad_im, stream);
}

// slam_external.gaussian(): float32 exp values divided by their float32 sum (R/utils/slam_external.py:54-57).  The
// sum is accumulated in double and rounded once: that is the value torch's float32 sum gives for these 11 weights,
// where a left-to-right float sum lands one ulp lower and would filter with a slightly different window.
static GaussWin gauss_window() {
    GaussWin g;
    for (int i = 0; i < kWin; ++i) g.w[i] = (float)exp(-(double)((i - kWin / 2) * (i - kWin / 2)) / (2.0 * 1.5 * 1.5));
    double ds = 0.0;
    for (int i = 0; i < kWin; ++i) ds += g.w[i];
    const float fs = (float)ds;
    for (int i = 0; i < kWin; ++i) g.w[i] = g.w[i] / fs;
    return g;
}

SB_API size_t sb_image_loss_workspace_floats(int C, int H, int W) { return (size_t)3 * C * H * W; }

/* loss terms of  w_l1*mean|x-y| + w_ssim*(1-mean(SSIM(x,y))) : writes sums[0]=sum(ssim map), sums[1]=sum|x-y|
 * (device doubles, zeroed here) and the partial-derivative maps into `work` (3*C*H*W floats). */
static int image_loss_forward(const uint8_t* keep, const float* x, const float* y, int C, int H, int W, float* work,
                              double* sums, void* stream) {
    if (!x || !y || !work || !sums || C < 1 || H < 1 || W < 1) return SB_ERR_BAD_ARG;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    SB_CUDA_CHECK(cudaMemsetAsync(sums, 0, (keep ? 3 : 2) * sizeof(double), st));
    const size_t n = (size_t)C * H * W;
    dim3 grid((W + kTW - 1) / kTW, (H + kTH - 1) / kTH, C), block(kTW, kTH);
    ssim_l1_forward_kernel<<<grid, block, 0, st>>>(x, y, C, H, W, work, work + n, work + 2 * n, sums, gauss_window(),
                                                   keep);
    SB_LAUNCH_CHECK("ssim_l1_forward_kernel");
    return SB_OK;
}

static int image_loss_backward(const uint8_t* keep, const double* sums, const float* x, const float* y, int C, int H,
                               int W, const float* work, const float* grad_out, float w_ssim, float w_l1,
                               float* grad_x, void* stream) {
    if (!x || !y || !work || !grad_out || !grad_x || C < 1 || H < 1 || W < 1) return SB_ERR_BAD_ARG;
    const size_t n = (size_t)C * H * W;
    dim3 grid((W + kTW - 1) / kTW, (H + kTH - 1) / kTH, C), block(kTW, kTH);
    ssim_l1_backward_kernel<<<grid, block, 0, static_cast<cudaStream_t>(stream)>>>(
        x, y, work, work + n, work + 2 * n, C, H, W, grad_out, w_ssim, w_l1, grad_x, gauss_window(), keep, sums);
    SB_LAUNCH_CHECK("ssim_l1_backward_kernel");
    return SB_OK;
}

SB_API int sb_image_loss_forward(const float* x, const float* y, int C, int H, int W, float* work, double* sums,
                                 void* stream) {
    return image_loss_forward(nullptr, x, y, C, H, W, work, sums, stream);
}

SB_API int sb_image_loss_backward(const float* x, const float* y, int C, int H, int W, const float* work,
                                  const float* grad_out, float w_ssim, float w_l1, float* grad_x, void* stream) {
    return image_loss_backward(nullptr, nullptr, x, y, C, H, W, work, grad_out, w_ssim, w_l1, grad_x, stream);
}

SB_API int sb_image_loss_keep_forward(const uint8_t* keep, const float* x, const float* y, int C, int H, int W,
                                      float* work, double* sums, void* stream) {
    if (!keep) return SB_ERR_BAD_ARG;
    return image_loss_forward(keep, x, y, C, H, W, work, sums, stream);
}

SB_API int sb_image_loss_keep_backward(const uint8_t* keep, const float* x, const float* y, int C, int H, int W,
                                       const float* work, const double* sums, const float* grad_out, float w_ssim,
                                       float w_l1, float* grad_x, void* stream) {
    if (!keep || !sums) return SB_ERR_BAD_ARG;
    return image_loss_backward(keep, sums, x, y, C, H, W, work, grad_out, w_ssim, w_l1, grad_x, stream);
}

}  // extern "C"
