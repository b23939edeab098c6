// binning.cu -- stage 2a of the forward: per-tile duplication, tile sort, tile ranges and the
// sorted SoA splat records (duplicateWithKeys + SortPairs + identifyTileRanges,
// X/cuda_rasterizer/rasterizer_impl.cu:70-138,284-319).
//
// Two-level ordering instead of the reference's single 64-bit sort: the Gaussians were already
// ordered by (depth bits, index) in launch_depth_order; instances are emitted in that order (tiles
// row-major inside one Gaussian, as the reference emits them) and then STABLY sorted by tile id
// alone.  The result -- instance list ordered by (tile, depth bits, index) -- is bit-identical to the
// reference's sorted point_list / point_list_keys, at 2 radix passes over 8-B pairs instead of 6
// passes over 12-B pairs.  The sort itself is this repo's own (radix_sort.cu).
#include "common.cuh"
#include "radix_sort.cuh"

namespace sb {

namespace {

// One warp per 32 consecutive depth-ordered Gaussians.  Their runs of instances are contiguous in the output (the
// scan's offsets), so the warp walks the span they cover together, lane l writing slots base + l: every store
// instruction writes 32 consecutive words.  A Gaussian's tile count is the difference of neighbouring offsets, so only
// the rectangles of Gaussians that touch a tile are gathered (one 8-B entry each).  A slot's Gaussian is the first lane
// whose run ends after it, found by a 5-step bisection over the lanes' run ends (shuffles); its tile is the slot's
// index in that run, row-major over the Gaussian's rectangle, as the reference emits them.  Slots at or past `cap`
// (capacity of the instance arrays in the sync-free mode, else 2^32-1) are not written.
__global__ void __launch_bounds__(256)
emit_instances_kernel(int P, const uint32_t* __restrict__ sorted_idx, const uint32_t* __restrict__ offsets,
                      const uint2* __restrict__ rect, uint32_t grid_x, uint32_t cap, uint32_t* __restrict__ tile_out,
                      uint32_t* __restrict__ val_out) {
    const int lane = threadIdx.x & 31;
    const int i0 = (blockIdx.x * blockDim.x + threadIdx.x) & ~31;
    if (i0 >= P) return;
    const int i = min(i0 + lane, P - 1);             // lanes past P repeat the last Gaussian with an empty run
    const uint32_t end = __ldg(offsets + i);         // inclusive scan: end of this Gaussian's run
    const uint32_t prev = __shfl_up_sync(0xffffffffu, end, 1);
    const uint32_t start = lane == 0 ? (i0 == 0 ? 0u : __ldg(offsets + i0 - 1)) : prev;
    const uint32_t g = __ldg(sorted_idx + i);
    const uint2 t = end != start ? __ldg(rect + g) : make_uint2(0u, 0u);
    const uint32_t span0 = __shfl_sync(0xffffffffu, start, 0);
    const uint32_t span1 = min(__shfl_sync(0xffffffffu, end, 31), cap);
    for (uint32_t base = span0; base < span1; base += 32u) {
        const uint32_t o = base + (uint32_t)lane;
        int j = 0;
#pragma unroll
        for (int step = 16; step > 0; step >>= 1)
            if (__shfl_sync(0xffffffffu, end, j + step - 1) <= o) j += step;
        const uint32_t k = o - __shfl_sync(0xffffffffu, start, j);
        const uint32_t rx = __shfl_sync(0xffffffffu, t.x, j), ry = __shfl_sync(0xffffffffu, t.y, j);
        const uint32_t gj = __shfl_sync(0xffffffffu, g, j);
        if (o < span1) {
            const uint32_t x0 = rx & 0xFFFFu, y0 = rx >> 16, w = (ry & 0xFFFFu) - x0;
            const uint32_t dy = k / w;
            tile_out[o] = (y0 + dy) * grid_x + x0 + (k - dy * w);
            val_out[o] = gj;
        }
    }
}

// Coverage mask of one tile instance: bit w is set iff the Gaussian can blend a pixel of consumer warp w's
// rectangle in the blend kernels, pixel centres x0..x0+7 by y0..y0+3 with x0 = 16 tx + 8 (w & 1),
// y0 = 16 ty + 4 (w >> 1).  A bit needs both
//   (a) the projection kernel's box test {x +- hx, y +- hy} against the rectangle, in float -- so the mask is a subset
//       of the box hits and NaN geometry culls; hx = -1 (opacity below 1/255, alpha < 1/255 at every pixel) clears
//       the whole mask;
//   (b) the conic's quadratic form q(u, v) = a u^2 + 2 b u v + c v^2 of the centre offset (u, v) = (x - px, y - py)
//       being at most the threshold somewhere on the continuous rectangle of pixel-centre offsets.
// Threshold: project.cu sets hx >= 1.0001 sqrt(2 tau c / dc) and hy >= 1.0001 sqrt(2 tau a / dc) (dc = ac - b^2, tau
// the slack-inflated ln(255 opacity)) so that every blended pixel has exact q <= 2 tau; hence c * 2 tau <= dc hx^2 /
// 1.00019 and a * 2 tau <= dc hy^2 / 1.00019 (the float rounding of hx, hy costs < 2.4e-7 of the 2e-4 factor).
// hx or hy = 1e30 marks a conic without that bound: (b) is skipped.
// If the origin is outside the rectangle, the minimum of the convex q over it lies on an edge that faces the origin
// (at most one edge v = const and one u = const).  On an edge v = const, a * min_u q = dist(-b v, [a u0, a u1])^2 +
// dc v^2 is compared with dc hy^2; on u = const, c * min_v q = dist(-b u, [c v0, c v1])^2 + dc u^2 with dc hx^2 --
// sums of non-negative terms, no division.  Evaluated in double: a c and b b are exact products of floats, so dc is
// the value project.cu derived hx, hy from, and dc >= 2^-49 a c; the rounding of the other operations then stays
// below 1e-7 relative, far inside the 1.9e-4 margin, so (b) never drops a pair whose exact q is at most 2 tau.  Every
// double operation is spelled out (no contraction), so tools/lane_packing_model.py reproduces the mask bit for bit.
__device__ __forceinline__ uint32_t cover_mask(const float4 ga, const float4 gb, uint32_t tx, uint32_t ty) {
    uint32_t box = 0u;
#pragma unroll
    for (int w = 0; w < 8; ++w) {
        const int x0 = (int)tx * kTile + (w & 1) * 8, y0 = (int)ty * kTile + (w >> 1) * 4;
        const float fx0 = (float)x0, fx1 = (float)(x0 + 7), fy0 = (float)y0, fy1 = (float)(y0 + 3);
        const bool hit = (ga.x + ga.z >= fx0) && (ga.x - ga.z <= fx1) && (ga.y + ga.w >= fy0) && (ga.y - ga.w <= fy1);
        box |= (hit ? 1u : 0u) << w;
    }
    if (!(ga.z > 0.f)) return 0u;
    if (box == 0u || ga.z >= 1e30f || ga.w >= 1e30f) return box;
    const double a = gb.x, b = gb.y, c = gb.z, hx = ga.z, hy = ga.w;
    const double dc = __dsub_rn(__dmul_rn(a, c), __dmul_rn(b, b));
    const double thr_x = __dmul_rn(dc, __dmul_rn(hx, hx)), thr_y = __dmul_rn(dc, __dmul_rn(hy, hy));
    uint32_t mask = 0u;
    while (box != 0u) {
        const int w = __ffs(box) - 1;
        box &= box - 1u;
        const double x0 = (double)((int)tx * kTile + (w & 1) * 8), y0 = (double)((int)ty * kTile + (w >> 1) * 4);
        const double u0 = __dsub_rn((double)ga.x, x0 + 7.0), u1 = __dsub_rn((double)ga.x, x0);
        const double v0 = __dsub_rn((double)ga.y, y0 + 3.0), v1 = __dsub_rn((double)ga.y, y0);
        bool in = u0 <= 0.0 && u1 >= 0.0 && v0 <= 0.0 && v1 >= 0.0;
        if (v0 > 0.0 || v1 < 0.0) {
            const double v = v0 > 0.0 ? v0 : v1, bv = __dmul_rn(b, v);
            const double d = fmax(fmax(__dadd_rn(__dmul_rn(a, u0), bv), -__dadd_rn(__dmul_rn(a, u1), bv)), 0.0);
            in = in || __dadd_rn(__dmul_rn(d, d), __dmul_rn(__dmul_rn(dc, v), v)) <= thr_y;
        }
        if (u0 > 0.0 || u1 < 0.0) {
            const double u = u0 > 0.0 ? u0 : u1, bu = __dmul_rn(b, u);
            const double d = fmax(fmax(__dadd_rn(__dmul_rn(c, v0), bu), -__dadd_rn(__dmul_rn(c, v1), bu)), 0.0);
            in = in || __dadd_rn(__dmul_rn(d, d), __dmul_rn(__dmul_rn(dc, u), u)) <= thr_x;
        }
        mask |= (in ? 1u : 0u) << w;
    }
    return mask;
}

// One thread per sorted instance: tile range boundaries (identifyTileRanges) fused with the gather
// of the instance's splat record into the sorted SoA arrays the blend kernels stage by TMA, and the
// instance's coverage mask (recA.z).
__global__ void __launch_bounds__(256)
ranges_and_records_kernel(int R_host, const int32_t* __restrict__ count_dev, const uint32_t* __restrict__ tile_sorted,
                          const uint32_t* __restrict__ point_list, uint32_t grid_x,
                          const float4* __restrict__ geom, const float* __restrict__ colors, const float* __restrict__ colors2,
                          uint2* __restrict__ ranges, float4* __restrict__ recA, float4* __restrict__ recB,
                          float4* __restrict__ recC, float4* __restrict__ recD) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const int R = count_dev ? min(*count_dev, R_host) : R_host;   // sync-free mode: R_host is the capacity
    if (i >= R) return;
    const uint32_t tile = tile_sorted[i];
    if (i == 0) ranges[tile].x = 0u;
    else {
        const uint32_t prev = tile_sorted[i - 1];
        if (prev != tile) { ranges[prev].y = (uint32_t)i; ranges[tile].x = (uint32_t)i; }
    }
    if (i == R - 1) ranges[tile].y = (uint32_t)R;
    const uint32_t g = __ldg(point_list + i);
    const float4 ga = __ldg(geom + 2 * (size_t)g), gb = __ldg(geom + 2 * (size_t)g + 1);   // one 32-B sector
    recA[i] = make_float4(ga.x, ga.y, __uint_as_float(cover_mask(ga, gb, tile % grid_x, tile / grid_x)), 0.f);
    recB[i] = gb;
    const float* c = colors + 3 * (size_t)g;
    recC[i] = make_float4(__ldg(c), __ldg(c + 1), __ldg(c + 2), __uint_as_float(g));
    if (colors2 != nullptr) {
        const float* e = colors2 + 3 * (size_t)g;
        recD[i] = make_float4(__ldg(e), __ldg(e + 1), __ldg(e + 2), 0.f);
    }
}

}  // namespace

int launch_binning(const sb_settings& s, int P, int R, const float* colors, const float* colors2,
                   const GeometryWs& g, const BinningWs& b, const ImageWs& img, const int32_t* count_dev,
                   cudaStream_t st) {
    const int gx = (s.image_width + kTile - 1) / kTile, gy = (s.image_height + kTile - 1) / kTile;
    const int tiles = gx * gy;
    SB_CUDA_CHECK(cudaMemsetAsync(img.ranges, 0, sizeof(uint2) * (size_t)tiles, st));  // rasterizer_impl.cu:311
    if (R <= 0) return SB_OK;
    const int bits = (int)higher_msb((uint32_t)tiles);  // same bit count as the reference sort uses
    { ScopedStage _p(kStEmit, st);
      emit_instances_kernel<<<(P + 255) / 256, 256, 0, st>>>(P, g.sorted_idx, g.offsets, g.rect, (uint32_t)gx,
                                                             count_dev ? (uint32_t)R : 0xFFFFFFFFu,
                                                             b.tile_unsorted, b.val_unsorted); }
    SB_LAUNCH_CHECK("emit_instances_kernel");
    { ScopedStage _p(kStTileSort, st);
      // sync-free mode: the pair count is read on the device (count_dev), so only the live instances are sorted --
      // no sentinel padding of the unused capacity, no extra key bits
      const int rc = radix_sort_pairs(b.tile_unsorted, b.val_unsorted, b.tile_sorted, b.point_list, R, count_dev, 0, bits,
                                      b.sort_temp, b.sort_temp_bytes, st);
      if (rc != SB_OK) return rc; }
    ScopedStage _p(kStRecords, st);
    ranges_and_records_kernel<<<(R + 255) / 256, 256, 0, st>>>(R, count_dev, b.tile_sorted, b.point_list,
                                                               (uint32_t)gx, g.geom, colors, colors2,
                                                               img.ranges, b.recA, b.recB, b.recC, b.recD);
    SB_LAUNCH_CHECK("ranges_and_records_kernel");
    return SB_OK;
}

}  // namespace sb
