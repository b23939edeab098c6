// blend_forward.cu -- stage 2b of the forward: front-to-back per-pixel alpha-composite of colour,
// median depth, final transmittance and contributor count (FORWARD::renderCUDA,
// X/cuda_rasterizer/forward.cu:261-393).
//
// One CTA per 16x16 tile (the tile size is part of the sort-key contract).  Warp 8 is a TMA
// producer: one elected lane streams the tile's contiguous range of sorted SoA splat records
// (recA/recB/recC, 16 B each) into a 4-stage shared-memory ring with cp.async.bulk + mbarrier
// complete_tx.  Warps 0-7 each own an 8x4 pixel sub-rectangle and consume the ring independently
// (no __syncthreads in the loop):
//   1. each lane reads ONE staged record's coverage bit for the warp's pixel rectangle (recA.z, computed once per
//      tile instance by binning.cu from the conservative ellipse-vs-rectangle test); __ballot_sync gives the
//      survivors of 32 Gaussians at once;
//   2. only survivors are evaluated per pixel, with exactly the reference's float operation order
//      (dx,dy,power,expf,alpha,test_T,fma accumulate), so colour / final_T / n_contrib are
//      bit-identical -- culled pairs are precisely pairs the reference skips (alpha < 1/255);
//   3. a warp whose 32 pixels are all saturated (T < 1e-4) stops evaluating (warp-vote early-out).
//
// kStats = true replays the same walk over a finished render's workspaces and writes no image: per Gaussian it counts
// the (pixel) pairs it blended (alpha >= 1/255, test_T >= 1e-4), the pairs it ended (test_T < 1e-4: it sets `done`),
// and atomicMax-es the bits of its largest weight alpha * T.  Each survivor step folds its 32 lanes with one ballot
// per count and one __reduce_max_sync, then one lane issues at most three integer atomics (deterministic).
#include "common.cuh"
#include "pipeline.cuh"

namespace sb {

namespace {

constexpr int kBatch = 128;           // records per pipeline stage
constexpr int kStages = 4;
constexpr int kConsumerWarps = 8;
constexpr int kBlendThreads = (kConsumerWarps + 1) * 32;

// NCH = 3: one colour set (the reference operator).  NCH = 6: two colour sets blended in one pass over
// the same geometry (SplaTAM's RGB render + depth/silhouette render, R/scripts/splatam.py:249,253).
template <int NCH>
struct __align__(128) FwdSmem {
    float4 A[kStages][kBatch];
    float4 B[kStages][kBatch];
    float4 C[kStages][kBatch];
    float4 D[NCH == 6 ? kStages : 1][NCH == 6 ? kBatch : 1];
    uint64_t full[kStages];
    uint64_t empty[kStages];
};

template <int NCH, int kMinBlocks, bool kStats = false>
__global__ void __launch_bounds__(kBlendThreads, kMinBlocks)
blend_forward_kernel(const uint2* __restrict__ ranges, const float4* __restrict__ recA,
                     const float4* __restrict__ recB, const float4* __restrict__ recC,
                     const float4* __restrict__ recD,
                     const uint32_t* __restrict__ depth_key, int W, int H, uint32_t grid_x,
                     const float* __restrict__ bg, float* __restrict__ out_color,
                     float* __restrict__ out_color2,
                     float* __restrict__ out_depth, float* __restrict__ final_T,
                     uint32_t* __restrict__ n_contrib, const int32_t* __restrict__ overflow_flag,
                     uint32_t* __restrict__ st_blended = nullptr, uint32_t* __restrict__ st_ended = nullptr,
                     uint32_t* __restrict__ st_max_weight = nullptr) {
    __shared__ FwdSmem<NCH> sm;
    // an overflowed sync-free render had truncated lists: its statistics add nothing (block-uniform exit)
    if (kStats && overflow_flag != nullptr && __ldg(overflow_flag) != 0) return;
    const uint32_t tile = blockIdx.x;
    const uint2 range = ranges[tile];
    const int n = (int)(range.y - range.x);
    const int nb = (n + kBatch - 1) / kBatch;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

    if (threadIdx.x == 0) {
        for (int s = 0; s < kStages; ++s) { mbar_init(&sm.full[s], 1); mbar_init(&sm.empty[s], kConsumerWarps); }
        mbar_fence_init();
    }
    __syncthreads();

    if (warp == kConsumerWarps) {
        // ---- TMA producer ----
        if (lane == 0) {
            for (int k = 0; k < nb; ++k) {
                const int s = k % kStages;
                if (k >= kStages) mbar_wait(&sm.empty[s], ((k / kStages) - 1) & 1);
                const int cnt = min(kBatch, n - k * kBatch);
                const uint32_t bytes = (uint32_t)cnt * 16u;
                const size_t src = (size_t)range.x + (size_t)k * kBatch;
                mbar_arrive_expect_tx(&sm.full[s], (NCH == 6 ? 4u : 3u) * bytes);
                tma_load_1d(sm.A[s], recA + src, bytes, &sm.full[s]);
                tma_load_1d(sm.B[s], recB + src, bytes, &sm.full[s]);
                tma_load_1d(sm.C[s], recC + src, bytes, &sm.full[s]);
                if (NCH == 6) tma_load_1d(sm.D[s], recD + src, bytes, &sm.full[s]);
            }
        }
        return;
    }

    // ---- consumers: warp w owns pixels [x0, x0+8) x [y0, y0+4) of the tile ----
    const uint32_t tx = tile % grid_x, ty = tile / grid_x;
    const int x0 = (int)tx * kTile + (warp & 1) * 8, y0 = (int)ty * kTile + (warp >> 1) * 4;
    const int px = x0 + (lane & 7), py = y0 + (lane >> 3);
    const bool inside = px < W && py < H;
    const float pxf = (float)px, pyf = (float)py;
    const uint32_t wbit = 1u << warp;   // this warp's bit of the records' coverage masks

    float T = 1.0f, C0 = 0.f, C1 = 0.f, C2 = 0.f, E0 = 0.f, E1 = 0.f, E2 = 0.f;
    float D = 15.0f;  // median depth default (forward.cu:308)
    uint32_t last = 0;
    bool done = !inside;
    bool warp_done = __all_sync(0xffffffffu, done);

    for (int k = 0; k < nb; ++k) {
        const int s = k % kStages;
        mbar_wait(&sm.full[s], (k / kStages) & 1);
        if (!warp_done) {
            const int cnt = min(kBatch, n - k * kBatch);
            for (int c = 0; c < cnt && !warp_done; c += 32) {
                const int jl = c + lane;
                const bool hit = jl < cnt && (__float_as_uint(sm.A[s][jl].z) & wbit) != 0u;
                uint32_t mask = __ballot_sync(0xffffffffu, hit);
                while (mask) {
                    const int j = c + (__ffs(mask) - 1);
                    mask &= mask - 1;
                    bool st_b = false, st_e = false;
                    uint32_t st_w = 0u;
                    if (!done) {
                        const float4 a = sm.A[s][j];
                        const float4 q = sm.B[s][j];
                        const float dx = __fsub_rn(a.x, pxf), dy = __fsub_rn(a.y, pyf);
                        const float sxy = __fmaf_rn(dx, __fmul_rn(dx, q.x), __fmul_rn(dy, __fmul_rn(dy, q.z)));
                        const float power = __fmaf_rn(sxy, -0.5f, -__fmul_rn(dy, __fmul_rn(dx, q.y)));
                        if (!(power > 0.0f)) {
                            const float alpha = fminf(__fmul_rn(q.w, expf(power)), 0.99f);
                            if (!(alpha < 1.0f / 255.0f)) {
                                const float test_T = __fmul_rn(T, __fsub_rn(1.0f, alpha));
                                if (test_T < 0.0001f) {
                                    done = true;
                                    if (kStats) st_e = true;
                                } else if (kStats) {
                                    st_b = true;
                                    st_w = __float_as_uint(__fmul_rn(alpha, T));
                                    T = test_T;
                                } else {
                                    const float4 col = sm.C[s][j];
                                    C0 = __fmaf_rn(T, __fmul_rn(alpha, col.x), C0);
                                    C1 = __fmaf_rn(T, __fmul_rn(alpha, col.y), C1);
                                    C2 = __fmaf_rn(T, __fmul_rn(alpha, col.z), C2);
                                    if (NCH == 6) {
                                        const float4 ex = sm.D[s][j];
                                        E0 = __fmaf_rn(T, __fmul_rn(alpha, ex.x), E0);
                                        E1 = __fmaf_rn(T, __fmul_rn(alpha, ex.y), E1);
                                        E2 = __fmaf_rn(T, __fmul_rn(alpha, ex.z), E2);
                                    }
                                    if (T > 0.5f && test_T < 0.5f)
                                        D = __uint_as_float(__ldg(depth_key + __float_as_uint(col.w)));
                                    T = test_T;
                                    last = (uint32_t)(k * kBatch + j + 1);
                                }
                            }
                        }
                    }
                    if (kStats) {
                        const uint32_t nbl = __popc(__ballot_sync(0xffffffffu, st_b));
                        const uint32_t nen = __popc(__ballot_sync(0xffffffffu, st_e));
                        const uint32_t wmax = __reduce_max_sync(0xffffffffu, st_w);
                        if (lane == 0 && (nbl | nen) != 0u) {
                            const uint32_t g = __float_as_uint(sm.C[s][j].w);
                            if (nbl) atomicAdd(st_blended + g, nbl);
                            if (nen) atomicAdd(st_ended + g, nen);
                            if (wmax) atomicMax(st_max_weight + g, wmax);
                        }
                    }
                }
                warp_done = __all_sync(0xffffffffu, done);
            }
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(&sm.empty[s]);
    }

    if (!kStats && inside) {
        const size_t pix = (size_t)py * W + px, hw = (size_t)H * W;
        // sync-free mode: if the scene needed more tile instances than the caller's capacity, the lists are truncated;
        // poison the images so that an incomplete render can never be mistaken for a valid one
        if (overflow_flag != nullptr && __ldg(overflow_flag) != 0) { C0 = C1 = C2 = E0 = E1 = E2 = __int_as_float(0x7fc00000); }
        final_T[pix] = T;
        n_contrib[pix] = last;
        out_color[pix] = __fmaf_rn(__ldg(bg), T, C0);
        out_color[hw + pix] = __fmaf_rn(__ldg(bg + 1), T, C1);
        out_color[2 * hw + pix] = __fmaf_rn(__ldg(bg + 2), T, C2);
        if (NCH == 6) {
            out_color2[pix] = __fmaf_rn(__ldg(bg), T, E0);
            out_color2[hw + pix] = __fmaf_rn(__ldg(bg + 1), T, E1);
            out_color2[2 * hw + pix] = __fmaf_rn(__ldg(bg + 2), T, E2);
        }
        out_depth[pix] = D;
    }
}

}  // namespace

int launch_blend_forward(const sb_settings& s, int R, const GeometryWs& g, const BinningWs& b,
                         const ImageWs& img, float* out_color, float* out_color2, float* out_depth,
                         const int32_t* overflow_flag, cudaStream_t st) {
    (void)R;
    const int W = s.image_width, H = s.image_height;
    const uint32_t gx = (W + kTile - 1) / kTile, gy = (H + kTile - 1) / kTile;
    ScopedStage _p(kStBlendFwd, st);
    if (out_color2 != nullptr)
        blend_forward_kernel<6, 4><<<gx * gy, kBlendThreads, 0, st>>>(img.ranges, b.recA, b.recB, b.recC, b.recD,
                                                                      g.depth_key, W, H, gx, s.bg, out_color,
                                                                      out_color2, out_depth, img.final_T,
                                                                      img.n_contrib, overflow_flag);
    else
        blend_forward_kernel<3, 5><<<gx * gy, kBlendThreads, 0, st>>>(img.ranges, b.recA, b.recB, b.recC, nullptr,
                                                                      g.depth_key, W, H, gx, s.bg, out_color,
                                                                      nullptr, out_depth, img.final_T,
                                                                      img.n_contrib, overflow_flag);
    SB_LAUNCH_CHECK("blend_forward_kernel");
    return SB_OK;
}

int launch_blend_stats(const sb_settings& s, const BinningWs& b, const ImageWs& img, const int32_t* overflow_flag,
                       uint32_t* blended, uint32_t* ended, uint32_t* max_weight_bits, cudaStream_t st) {
    const int W = s.image_width, H = s.image_height;
    const uint32_t gx = (W + kTile - 1) / kTile, gy = (H + kTile - 1) / kTile;
    // the walk reads geometry (recA, recB) and the index (recC.w) only, so one instantiation serves both colour sets
    blend_forward_kernel<3, 5, true><<<gx * gy, kBlendThreads, 0, st>>>(img.ranges, b.recA, b.recB, b.recC, nullptr,
                                                                        nullptr, W, H, gx, nullptr, nullptr, nullptr,
                                                                        nullptr, nullptr, nullptr, overflow_flag,
                                                                        blended, ended, max_weight_bits);
    SB_LAUNCH_CHECK("blend_forward_kernel<stats>");
    return SB_OK;
}

}  // namespace sb
