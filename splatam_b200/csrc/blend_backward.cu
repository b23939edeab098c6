// blend_backward.cu -- backward of the alpha-composite (BACKWARD::renderCUDA,
// X/cuda_rasterizer/backward.cu:399-557): walks every tile's sorted list back-to-front from the last
// contributor, rebuilds T as the reference does (T /= 1-alpha), and produces per-Gaussian
// dL/d{mean2D.xy, conic.xx/xy/yy, opacity, colour rgb}.
//
// One CTA per 16x16 tile: a TMA producer warp streams the tile's sorted splat records into a shared-memory
// ring (as blend_forward.cu); 8 autonomous consumer warps own one 8x4 pixel rectangle each.  The reference
// issues 9 global float atomics per contributing (pixel, Gaussian) pair (backward.cu:523-554) from a loop
// in which, on SplaTAM-sized splats, only ~10 of a warp's 32 pixels lie inside any one Gaussian.  Here the
// work of a warp is split by what it depends on, over a WINDOW of KW mask-culled survivors at a time:
//
//   gather   (lane = record)  : ballot-cull 32 staged records with their coverage bit for the warp's rectangle
//                               (recA.z, binning.cu's conservative ellipse-vs-rectangle test), compact survivors
//                               into the window;
//   evaluate (lane = pixel, lock-step over the window's slots): the part that needs no running state --
//                               G = exp(power), opacity*G, the skip decisions with the forward's exact float
//                               sequence, and c.dL/dpixel -- parked in a [slot][pixel] matrix in shared
//                               memory, plus a per-lane bit mask of the slots that blend this pixel;
//   chain    (lane = pixel, every lane walks ITS OWN mask bits): the sequential part -- T /= (1-alpha),
//                               the colour seen behind the Gaussian (as a scalar: only its dot product with
//                               dL/dpixel is ever used), dL/dalpha -> w = G dL/dG and ca = alpha T, written
//                               back into the matrix.  A lane never spends an iteration on a Gaussian that
//                               does not cover its pixel: 1.8-2.0x fewer iterations than a warp-lock-stepped walk
//                               on the 1M-Gaussian bench (tools/lane_window_model.py);
//   reduce   (lane = Gaussian, two lanes per slot): sweep the slot's 32 pixels, accumulate raw moments in
//                               pixel coordinates local to the rectangle and the colour sums in registers at full
//                               lane utilisation, shift the moments to the Gaussian's centre once per slot, and
//                               flush them with 16-byte vector reductions (REDG.E.ADD.F32x4) per (warp, Gaussian).
#include "common.cuh"
#include "pipeline.cuh"

namespace sb {

namespace {

constexpr int kBatch = 64;            // records per ring stage
template <int NCH> constexpr int stages_of() { return NCH == 6 ? 4 : 8; }   // ring depth (4 record arrays per stage at NCH 6)
constexpr int kConsumerWarps = 8;
constexpr int kBlendThreads = (kConsumerWarps + 1) * 32;
constexpr int kRow = 33;              // matrix row stride in cells: column sweeps (reduce) are conflict-free

// One matrix cell per (window slot, pixel): {opacity*G -> w, c.dL -> ca}; for NCH == 6 the cell holds the sums over
// both colour sets {opacity*G -> w, (c.dL + e.dL2) -> ca} and a second float matrix q3 holds {c.dL -> w of the first
// set}.  12 B per (slot, pixel) instead of a padded float4 keeps two CTAs per SM resident.
using Cell = float2;

template <int NCH, int KW>
struct __align__(128) BwdSmem {
    static constexpr int kStages = stages_of<NCH>();
    float4 A[kStages][kBatch];
    float4 B[kStages][kBatch];
    float4 C[kStages][kBatch];
    float4 D[NCH == 6 ? kStages : 1][NCH == 6 ? kBatch : 1];
    uint64_t full[kStages];
    uint64_t empty[kStages];
    uint32_t nmax;
    uint32_t pad[15];
    // per consumer warp: the window's records ...
    float4 WA[kConsumerWarps][KW];     // {pixel x, pixel y, bits(list index), -}
    float4 WB[kConsumerWarps][KW];     // {conic.x, conic.y, conic.z, opacity}
    float4 WC[kConsumerWarps][KW];     // {r, g, b, bits(Gaussian id)}
    float4 WD[NCH == 6 ? kConsumerWarps : 1][NCH == 6 ? KW : 1];   // second colour set
    // ... the [slot][pixel] matrix and dL/dpixel of the warp's 32 pixels
    Cell q[kConsumerWarps][KW][kRow];
    float q3[NCH == 6 ? kConsumerWarps : 1][NCH == 6 ? KW : 1][kRow];
    float4 dL[kConsumerWarps][NCH == 6 ? 2 : 1][32];
};

// 1/x for x in [0.01, 1]: MUFU.RCP + one Newton step (error < 1 ulp; the reference divides, IEEE).
__device__ __forceinline__ float fast_rcp(float x) {
    float r;
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
    return fmaf(r, fmaf(-x, r, 1.0f), r);
}

// 16-byte vector reduction into global memory (sm_90+; SASS REDG.E.ADD.F32x4).
__device__ __forceinline__ void red_add_v4(float* addr, float a, float b, float c, float d) {
    asm volatile("red.relaxed.gpu.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(addr), "f"(a), "f"(b), "f"(c),
                 "f"(d)
                 : "memory");
}

// Takes the first slot left in `rest` (bit 31 - s stands for slot s) out of it and returns s, or -1 when `rest` is
// empty: bfind.shiftamt (SASS FLO.U32.SH) is the leading-zero count, 0xffffffff for 0, and shr.b32 clamps its shift,
// so the empty case needs no branch.
__device__ __forceinline__ int pop_slot(uint32_t& rest) {
    uint32_t s, bit;
    asm("bfind.shiftamt.u32 %0, %1;" : "=r"(s) : "r"(rest));
    asm("shr.b32 %0, 0x80000000, %1;" : "=r"(bit) : "r"(s));
    rest ^= bit;
    return (int)s;
}

// Phase timing of the instrumented build (tools/blend_phases.py compiles this file with -DSB_PROBE_BLEND_PHASES;
// the shipped library has none of it).  Every consumer warp sums clock64() deltas per phase and adds them to
// g_probe_cycles at its end; each CTA leaves its %globaltimer start and end in g_probe_cta_ns.
enum ProbePhase { kPhWait, kPhGather, kPhEvaluate, kPhChain, kPhReduce, kNumPhases };
#ifdef SB_PROBE_BLEND_PHASES
constexpr int kProbeMaxTiles = 1 << 16;
__device__ unsigned long long g_probe_cycles[kNumPhases];
__device__ unsigned long long g_probe_cta_ns[2][kProbeMaxTiles];
__device__ __forceinline__ unsigned long long globaltimer_ns() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}
struct PhaseClock {
    long long t, acc[kNumPhases];
    __device__ __forceinline__ void start() {
        for (int p = 0; p < kNumPhases; ++p) acc[p] = 0;
        t = clock64();
    }
    __device__ __forceinline__ void lap(int p) { const long long n = clock64(); acc[p] += n - t; t = n; }
    __device__ __forceinline__ void flush(int lane, uint32_t tile) {
        if (lane != 0) return;
        for (int p = 0; p < kNumPhases; ++p) atomicAdd(&g_probe_cycles[p], (unsigned long long)acc[p]);
        if (tile < kProbeMaxTiles) atomicMax(&g_probe_cta_ns[1][tile], globaltimer_ns());
    }
};
#else
struct PhaseClock {
    __device__ __forceinline__ void start() {}
    __device__ __forceinline__ void lap(int) {}
    __device__ __forceinline__ void flush(int, uint32_t) {}
};
#endif

// Per-pixel running state of the back-to-front walk (one lane = one pixel).
template <int NCH>
struct PixelState {
    float T;            // transmittance in front of the Gaussian being processed
    float A;            // (colour accumulated behind) . dL/dpixel        (accum_rec, backward.cu:513-518)
    float last_alpha;   // alpha of the previous (deeper) contributor
    float last_cd;      // (its colour) . dL/dpixel
    float A1, last_cd1; // NCH == 6: the same for the first colour set alone
};

// evaluate + chain + reduce over the first `count` slots of the warp's window.
template <int NCH, int KW>
__device__ __forceinline__ void process_window(BwdSmem<NCH, KW>& sm, const int warp, const int lane, const int count,
                                               const float pxf, const float pyf, const uint32_t nc,
                                               const float4 dLa, const float4 dLb, const float T_final,
                                               const float bg_dot, const float bg_dot1, PixelState<NCH>& st,
                                               const float fx0, const float fy0, const float ddelx_dx,
                                               const float ddely_dy, float* __restrict__ accum, PhaseClock& clk) {
    constexpr uint32_t full = 0xffffffffu;
    constexpr int kStride = NCH == 6 ? kAccumStride2 : kAccumStride;
    __syncwarp();
    clk.lap(kPhGather);
    Cell* const qcol = &sm.q[warp][0][lane];          // this pixel's column, row stride kRow cells
    float* const q3col = &sm.q3[NCH == 6 ? warp : 0][0][lane];

    // ---- evaluate: lock-step over the slots, lane = pixel (same float sequence as the forward so the skip
    //      decisions agree, backward.cu:491-500) ----
    uint32_t mymask = 0u;
    float4 wa = sm.WA[warp][0], q = sm.WB[warp][0], col = sm.WC[warp][0];
    float4 ex = make_float4(0.f, 0.f, 0.f, 0.f);
    if constexpr (NCH == 6) ex = sm.WD[NCH == 6 ? warp : 0][0];
#pragma unroll 2
    for (int s = 0; s < count; ++s) {
        // software pipeline: the next slot's records are in flight while this slot is evaluated
        const int sn = min(s + 1, KW - 1);
        const float4 wa_n = sm.WA[warp][sn], q_n = sm.WB[warp][sn], col_n = sm.WC[warp][sn];
        float4 ex_n = make_float4(0.f, 0.f, 0.f, 0.f);
        if constexpr (NCH == 6) ex_n = sm.WD[NCH == 6 ? warp : 0][NCH == 6 ? sn : 0];
        const float dx = __fsub_rn(wa.x, pxf), dy = __fsub_rn(wa.y, pyf);
        const float sxy = __fmaf_rn(dx, __fmul_rn(dx, q.x), __fmul_rn(dy, __fmul_rn(dy, q.z)));
        const float power = __fmaf_rn(sxy, -0.5f, -__fmul_rn(dy, __fmul_rn(dx, q.y)));
        const float G = expf(power);
        const float Gop = __fmul_rn(q.w, G);
        const float alpha = fminf(Gop, 0.99f);
        const bool active = (__float_as_uint(wa.z) < nc) && !(power > 0.0f) && !(alpha < 1.0f / 255.0f);
        const float cd1 = fmaf(col.z, dLa.z, fmaf(col.y, dLa.y, col.x * dLa.x));
        if constexpr (NCH == 6) {
            const float cdS = fmaf(ex.z, dLb.z, fmaf(ex.y, dLb.y, fmaf(ex.x, dLb.x, cd1)));
            float2 v = make_float2(0.f, 0.f);
            if (active) { v.x = Gop; v.y = cdS; }
            qcol[s * kRow] = v;
            q3col[s * kRow] = active ? cd1 : 0.f;
        } else {
            float2 v = make_float2(0.f, 0.f);
            if (active) { v.x = Gop; v.y = cd1; }
            qcol[s * kRow] = v;
        }
        mymask |= (active ? 1u : 0u) << s;
        wa = wa_n; q = q_n; col = col_n; ex = ex_n;
    }

    clk.lap(kPhEvaluate);

    // ---- chain: each lane walks its own contributors, deepest first (slot order = back to front) ----
    //      A lane whose contributors are used up steps on an all-zero cell, so the step needs no branch: alpha = 0
    //      gives ir = 1 exactly (fast_rcp(1) = 1), so T does not change; A (and A1) take the deeper contributor's
    //      term one step early and then add 0 * 0, which is the value the next contributor would have computed,
    //      bit for bit (A is never -0: it starts at +0 and a sum of two terms is -0 only if both are).  Only the
    //      stores are predicated.
    const int iters = (int)__reduce_max_sync(full, (uint32_t)__popc(mymask));
    {
        uint32_t rest = __brev(mymask);
        // the next contributor's cell is loaded before this one's chain step (hides the shared-memory latency)
        int s = pop_slot(rest);
        Cell v = make_float2(0.f, 0.f);
        float v3 = 0.f;
        if (s >= 0) {
            v = qcol[s * kRow];
            if constexpr (NCH == 6) v3 = q3col[s * kRow];
        }
        for (int it = 0; it < iters; ++it) {
            const int s_n = pop_slot(rest);
            Cell v_n = make_float2(0.f, 0.f);
            float v3_n = 0.f;
            if (s_n >= 0) {
                v_n = qcol[s_n * kRow];
                if constexpr (NCH == 6) v3_n = q3col[s_n * kRow];
            }
            const float Gop = v.x, cd = v.y;
            const float alpha = fminf(Gop, 0.99f);
            const float ir = fast_rcp(1.f - alpha);
            st.T = st.T * ir;                                     // T = T / (1 - alpha)
            const float ca = alpha * st.T;                        // dchannel_dcolor
            const float om = 1.f - st.last_alpha;
            st.A = fmaf(st.last_alpha, st.last_cd, om * st.A);
            const float tb = T_final * ir;
            const float dL_dalpha = fmaf(cd - st.A, st.T, -tb * bg_dot);
            st.last_cd = cd;
            if constexpr (NCH == 6) {
                const float cd1 = v3;
                st.A1 = fmaf(st.last_alpha, st.last_cd1, om * st.A1);
                const float dL_dalpha1 = fmaf(cd1 - st.A1, st.T, -tb * bg_dot1);
                st.last_cd1 = cd1;
                if (s >= 0) q3col[s * kRow] = Gop * dL_dalpha1;
            }
            if (s >= 0) qcol[s * kRow] = make_float2(Gop * dL_dalpha, ca);
            st.last_alpha = alpha;
            s = s_n; v = v_n; v3 = v3_n;
        }
    }
    __syncwarp();
    clk.lap(kPhChain);

    // ---- reduce: lanes (sl, part) = (lane & 15, lane >> 4) sweep pixels [16 part, 16 part + 16) of slot
    //      16 round + sl ----
    const int sl = lane & 15, part = lane >> 4;
#pragma unroll 1
    for (int r0 = 0; r0 < count; r0 += 16) {
        const int slot = r0 + sl;
        const bool live = slot < count;
        const int sc = live ? slot : 0;                 // dead lanes sweep slot 0 and discard the result
        const float4 wa = sm.WA[warp][sc], q = sm.WB[warp][sc];
        const float gxr = wa.x - fx0, gyr = (wa.y - fy0) - (float)(2 * part);
        const Cell* qrow = &sm.q[warp][sc][16 * part];
        const float4* dl = &sm.dL[warp][0][16 * part];
        // Raw moments in pixel coordinates local to the half-rectangle (8x2 pixels) and centred on its middle:
        // lx = px - 3.5 in [-3.5, 3.5] is a constant of the unrolled row sweep and ly = py - 0.5 = -+0.5 one of the
        // row, so a pixel costs one add and two FMAs with immediates for all six moment sums (ly^2 = 1/4 makes
        // sum w ly^2 = Sw / 4, and sum w lx ly is taken per row).  The row loop stays rolled: unrolling both rows
        // lets the compiler hoist all 16 pixels' loads and spills at <3,16,3>'s 72-register budget.
        float Sw = 0.f, Sx = 0.f, Sy = 0.f, Sxyl = 0.f, XX = 0.f, C0 = 0.f, C1 = 0.f, C2 = 0.f;
        float E0 = 0.f, E1 = 0.f, E2 = 0.f, Rw = 0.f, Rly = 0.f, RX = 0.f;   // NCH == 6 only
#pragma unroll 1
        for (int row = 0; row < 2; ++row) {
            const float ly = (float)row - 0.5f;
            float W = 0.f, X = 0.f, Wr = 0.f;
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                const int it = 8 * row + i;
                const Cell v = qrow[it];
                const float4 d = dl[it];
                const float w = v.x, ca = v.y;
                const float lx = (float)i - 3.5f;
                W += w; X = fmaf(w, lx, X); XX = fmaf(w, lx * lx, XX);
                C0 = fmaf(ca, d.x, C0); C1 = fmaf(ca, d.y, C1); C2 = fmaf(ca, d.z, C2);
                if constexpr (NCH == 6) {
                    const float wr = sm.q3[NCH == 6 ? warp : 0][NCH == 6 ? sc : 0][16 * part + it];
                    const float4 d2 = sm.dL[warp][NCH == 6 ? 1 : 0][16 * part + it];
                    Wr += wr; RX = fmaf(wr, lx, RX);
                    E0 = fmaf(ca, d2.x, E0); E1 = fmaf(ca, d2.y, E1); E2 = fmaf(ca, d2.z, E2);
                }
            }
            Sw += W; Sy = fmaf(ly, W, Sy); Sx += X; Sxyl = fmaf(ly, X, Sxyl);
            if constexpr (NCH == 6) { Rw += Wr; Rly = fmaf(ly, Wr, Rly); }
        }
        // Moments about the Gaussian's centre (gx, gy) in the same frame, dx = gx - lx, dy = gy - ly.  Shifting the
        // raw moments cancels terms of size gx^2 Sw, with |gx| <= 3.5 + the splat's reach past the rectangle; the
        // rounding error is a few ulps of gx^2 Sw, against the ulps of the per-pixel sums it replaces.  Centring
        // the local frame (rather than taking the corner pixel as 0) keeps gx small when the centre is inside.
        const float gx = gxr - 3.5f, gy = gyr - 0.5f;
        float Swx = fmaf(gx, Sw, -Sx), Swy = fmaf(gy, Sw, -Sy);
        float Sxx = fmaf(gx, Swx - Sx, XX);                       // sum w dx^2
        float Syy = fmaf(gy, Swy - Sy, 0.25f * Sw);               // sum w dy^2
        float Sxy = fmaf(gx, Swy, fmaf(-gy, Sx, Sxyl));           // sum w dx dy
        float Rx = 0.f, Ry = 0.f;
        if constexpr (NCH == 6) { Rx = fmaf(gx, Rw, -RX); Ry = fmaf(gy, Rw, -Rly); }
        Sw += __shfl_xor_sync(full, Sw, 16);   Swx += __shfl_xor_sync(full, Swx, 16);
        Swy += __shfl_xor_sync(full, Swy, 16); Sxx += __shfl_xor_sync(full, Sxx, 16);
        Sxy += __shfl_xor_sync(full, Sxy, 16); Syy += __shfl_xor_sync(full, Syy, 16);
        C0 += __shfl_xor_sync(full, C0, 16);   C1 += __shfl_xor_sync(full, C1, 16);
        C2 += __shfl_xor_sync(full, C2, 16);
        if constexpr (NCH == 6) {
            E0 += __shfl_xor_sync(full, E0, 16); E1 += __shfl_xor_sync(full, E1, 16);
            E2 += __shfl_xor_sync(full, E2, 16); Rx += __shfl_xor_sync(full, Rx, 16);
            Ry += __shfl_xor_sync(full, Ry, 16);
        }
        if (live && part == 0) {
            // dG/ddelx = -G (dx a + dy b), dG/ddely = -G (dy c + dx b)   (backward.cu:539-546)
            const float a = q.x, b = q.y, c = q.z, op = q.w;
            float* row = accum + (size_t)__float_as_uint(sm.WC[warp][sc].w) * kStride;
            // row = {dmean2D.x, dmean2D.y, dconic.xx, dconic.xy | dconic.yy, dopacity, dcolor.r, .g | .b, ...}
            red_add_v4(row, -(a * Swx + b * Swy) * ddelx_dx, -(c * Swy + b * Swx) * ddely_dy, -0.5f * Sxx,
                       -0.5f * Sxy);
            // G dL/dalpha = w / opacity  (dL/dG = opacity dL/dalpha)
            red_add_v4(row + 4, -0.5f * Syy, Sw / op, C0, C1);
            if constexpr (NCH == 6) {
                red_add_v4(row + 8, C2, E0, E1, E2);
                red_add_v4(row + 12, -(a * Rx + b * Ry) * ddelx_dx, -(c * Ry + b * Rx) * ddely_dy, 0.f, 0.f);
            } else {
                atomicAdd(row + 8, C2);
            }
        }
    }
    __syncwarp();
    clk.lap(kPhReduce);
}

template <int NCH, int KW, int kMinBlocks>
__global__ void __launch_bounds__(kBlendThreads, kMinBlocks)
blend_backward_kernel(const uint2* __restrict__ ranges, const float4* __restrict__ recA,
                      const float4* __restrict__ recB, const float4* __restrict__ recC,
                      const float4* __restrict__ recD,
                      int W, int H, uint32_t grid_x, const float* __restrict__ bg,
                      const float* __restrict__ final_T, const uint32_t* __restrict__ n_contrib,
                      const float* __restrict__ dL_dpix, const float* __restrict__ dL_dpix2,
                      float* __restrict__ accum) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    BwdSmem<NCH, KW>& sm = *reinterpret_cast<BwdSmem<NCH, KW>*>(smem_raw);
    constexpr uint32_t full = 0xffffffffu;
    constexpr int kStages = stages_of<NCH>();
    const uint32_t tile = blockIdx.x;
    const uint2 range = ranges[tile];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

#ifdef SB_PROBE_BLEND_PHASES
    if (threadIdx.x == 0 && tile < kProbeMaxTiles) {
        g_probe_cta_ns[0][tile] = globaltimer_ns();
        g_probe_cta_ns[1][tile] = 0ull;
    }
#endif
    if (threadIdx.x == 0) {
        for (int s = 0; s < kStages; ++s) { mbar_init(&sm.full[s], 1); mbar_init(&sm.empty[s], kConsumerWarps); }
        sm.nmax = 0u;
        mbar_fence_init();
    }
    __syncthreads();

    const uint32_t tx = tile % grid_x, ty = tile / grid_x;
    const int x0 = (int)tx * kTile + (warp & 1) * 8, y0 = (int)ty * kTile + (warp >> 1) * 4;
    const int px = x0 + (lane & 7), py = y0 + (lane >> 3);
    const bool inside = (warp < kConsumerWarps) && px < W && py < H;
    const size_t pix = (size_t)py * W + px, hw = (size_t)H * W;
    const float T_final = inside ? final_T[pix] : 0.f;
    const uint32_t nc = inside ? n_contrib[pix] : 0u;
    const uint32_t warp_nc = __reduce_max_sync(full, nc);
    if (lane == 0 && warp_nc > 0u) atomicMax(&sm.nmax, warp_nc);
    float4 dLa = make_float4(0.f, 0.f, 0.f, 0.f), dLb = make_float4(0.f, 0.f, 0.f, 0.f);
    if (inside) { dLa.x = dL_dpix[pix]; dLa.y = dL_dpix[hw + pix]; dLa.z = dL_dpix[2 * hw + pix]; }
    if (NCH == 6 && inside) { dLb.x = dL_dpix2[pix]; dLb.y = dL_dpix2[hw + pix]; dLb.z = dL_dpix2[2 * hw + pix]; }
    if (warp < kConsumerWarps) {
        sm.dL[warp][0][lane] = dLa;
        if (NCH == 6) sm.dL[warp][NCH == 6 ? 1 : 0][lane] = dLb;
    }
    __syncthreads();
    const int m = (int)sm.nmax;                 // entries [0, m) of the tile list can matter
    const int nb = (m + kBatch - 1) / kBatch;

    if (warp == kConsumerWarps) {
        if (lane == 0) {
            for (int k = 0; k < nb; ++k) {
                const int s = k % kStages;
                if (k >= kStages) mbar_wait(&sm.empty[s], ((k / kStages) - 1) & 1);
                const int hi = m - k * kBatch, cnt = min(kBatch, hi), lo = hi - cnt;
                const uint32_t bytes = (uint32_t)cnt * 16u;
                const size_t src = (size_t)range.x + (size_t)lo;
                mbar_arrive_expect_tx(&sm.full[s], (NCH == 6 ? 4u : 3u) * bytes);
                tma_load_1d(sm.A[s], recA + src, bytes, &sm.full[s]);
                tma_load_1d(sm.B[s], recB + src, bytes, &sm.full[s]);
                tma_load_1d(sm.C[s], recC + src, bytes, &sm.full[s]);
                if (NCH == 6) tma_load_1d(sm.D[s], recD + src, bytes, &sm.full[s]);
            }
        }
        return;
    }

    const float pxf = (float)px, pyf = (float)py;
    const float fx0 = (float)x0, fy0 = (float)y0;
    const float bg0 = __ldg(bg), bg1 = __ldg(bg + 1), bg2 = __ldg(bg + 2);
    const float bg_dot1 = bg0 * dLa.x + bg1 * dLa.y + bg2 * dLa.z;
    const float bg_dot = NCH == 6 ? bg_dot1 + (bg0 * dLb.x + bg1 * dLb.y + bg2 * dLb.z) : bg_dot1;
    const float ddelx_dx = 0.5f * W, ddely_dy = 0.5f * H;  // pixel -> NDC (backward.cu:452-453)
    PixelState<NCH> st;
    st.T = T_final; st.A = 0.f; st.last_alpha = 0.f; st.last_cd = 0.f; st.A1 = 0.f; st.last_cd1 = 0.f;
    int wcount = 0;                                    // survivors in the window (warp-uniform)
    const uint32_t lt_mask = (1u << lane) - 1u;
    PhaseClock clk;
    clk.start();

    for (int k = 0; k < nb; ++k) {
        const int s = k % kStages;
        clk.lap(kPhGather);
        mbar_wait(&sm.full[s], (k / kStages) & 1);
        clk.lap(kPhWait);
        const int hi = m - k * kBatch, cnt = min(kBatch, hi), lo = hi - cnt;
        if (lo < (int)warp_nc) {
            for (int c = 0; c < cnt; c += 32) {
                const int jl = cnt - 1 - (c + lane);       // ascending lane = descending list index
                bool hit = jl >= 0 && lo + jl < (int)warp_nc &&
                           ((__float_as_uint(sm.A[s][jl].z) >> warp) & 1u) != 0u;   // coverage bit of this warp
                uint32_t mask = __ballot_sync(full, hit);
                while (mask != 0u) {
                    const int pos = wcount + __popc(mask & lt_mask);
                    const bool take = hit && pos < KW;
                    if (take) {
                        const float4 a = sm.A[s][jl];
                        sm.WA[warp][pos] = make_float4(a.x, a.y, __uint_as_float((uint32_t)(lo + jl)), 0.f);
                        sm.WB[warp][pos] = sm.B[s][jl];
                        sm.WC[warp][pos] = sm.C[s][jl];
                        if (NCH == 6) sm.WD[NCH == 6 ? warp : 0][NCH == 6 ? pos : 0] = sm.D[NCH == 6 ? s : 0][NCH == 6 ? jl : 0];
                    }
                    const int nhit = __popc(mask);
                    const int ntake = min(nhit, KW - wcount);
                    wcount += ntake;
                    hit = hit && !take;
                    if (wcount == KW) {
                        process_window<NCH, KW>(sm, warp, lane, KW, pxf, pyf, nc, dLa, dLb, T_final, bg_dot, bg_dot1,
                                                st, fx0, fy0, ddelx_dx, ddely_dy, accum, clk);
                        wcount = 0;
                    }
                    mask = (ntake == nhit) ? 0u : __ballot_sync(full, hit);
                }
            }
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(&sm.empty[s]);
    }
    if (wcount > 0)
        process_window<NCH, KW>(sm, warp, lane, wcount, pxf, pyf, nc, dLa, dLb, T_final, bg_dot, bg_dot1, st, fx0,
                                fy0, ddelx_dx, ddely_dy, accum, clk);
    clk.lap(kPhGather);
    clk.flush(lane, tile);
}

}  // namespace

#ifdef SB_PROBE_BLEND_PHASES
// Instrumented build only: copies the phase totals (kNumPhases values) and the first `ntiles` CTA start / end times
// to the host, then zeroes the totals.
extern "C" SB_API int sb_probe_blend_phases(unsigned long long* cycles, unsigned long long* cta_start,
                                            unsigned long long* cta_end, int ntiles) {
    if (ntiles < 0 || ntiles > kProbeMaxTiles) return SB_ERR_BAD_ARG;
    const size_t nt = (size_t)ntiles * sizeof(unsigned long long);
    if (cudaMemcpyFromSymbol(cycles, g_probe_cycles, sizeof(g_probe_cycles)) != cudaSuccess ||
        cudaMemcpyFromSymbol(cta_start, g_probe_cta_ns, nt, 0) != cudaSuccess ||
        cudaMemcpyFromSymbol(cta_end, g_probe_cta_ns, nt, sizeof(g_probe_cta_ns[0])) != cudaSuccess)
        return SB_ERR_CUDA;
    const unsigned long long zero[kNumPhases] = {};
    return cudaMemcpyToSymbol(g_probe_cycles, zero, sizeof(zero)) == cudaSuccess ? SB_OK : SB_ERR_CUDA;
}
#endif

int launch_blend_backward(const sb_settings& s, int R, const BinningWs& b, const ImageWs& img,
                          const float* dL_dout_color, const float* dL_dout_color2, float* accum,
                          cudaStream_t st) {
    if (R <= 0) return SB_OK;
    const int W = s.image_width, H = s.image_height;
    const uint32_t gx = (W + kTile - 1) / kTile, gy = (H + kTile - 1) / kTile;
#define SB_LAUNCH_BWD(NCH, KW, MB)                                                                              \
    do {                                                                                                        \
        SB_CUDA_CHECK(cudaFuncSetAttribute(blend_backward_kernel<NCH, KW, MB>,                                  \
                                           cudaFuncAttributeMaxDynamicSharedMemorySize,                         \
                                           (int)sizeof(BwdSmem<NCH, KW>)));                                     \
        ScopedStage _p(kStBlendBwd, st);                                                                        \
        blend_backward_kernel<NCH, KW, MB><<<gx * gy, kBlendThreads, sizeof(BwdSmem<NCH, KW>), st>>>(           \
            img.ranges, b.recA, b.recB, b.recC, b.recD, W, H, gx, s.bg, img.final_T, img.n_contrib, dL_dout_color, \
            dL_dout_color2, accum);                                                                             \
    } while (0)
    if (dL_dout_color2 != nullptr) SB_LAUNCH_BWD(6, 16, 2);
    else SB_LAUNCH_BWD(3, 16, 3);
#undef SB_LAUNCH_BWD
    SB_LAUNCH_CHECK("blend_backward_kernel");
    return SB_OK;
}

}  // namespace sb
