// common.cuh -- shared device helpers, workspace layouts and error plumbing for the
// splatam_b200 rasterizer (sm_90a, H100).  See DESIGN.md for the HBM layout.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stddef.h>
#include "../../include/splatam_b200.h"

namespace sb {

constexpr int kTile = SB_TILE;          // 16x16 pixel tiles (key contract)
constexpr int kAlign = 256;             // every workspace chunk is 256-B aligned (TMA needs 16)
constexpr uint32_t kCulledKey = 0xFFFFFFFFu;  // depth key of a Gaussian that emits nothing

// ---- error plumbing -------------------------------------------------------------------
void set_cuda_error(cudaError_t e, const char* where);
#define SB_CUDA_CHECK(expr)                                                       \
    do {                                                                          \
        cudaError_t _e = (expr);                                                  \
        if (_e != cudaSuccess) { ::sb::set_cuda_error(_e, #expr); return SB_ERR_CUDA; } \
    } while (0)
#define SB_LAUNCH_CHECK(name)                                                     \
    do {                                                                          \
        cudaError_t _e = cudaGetLastError();                                      \
        if (_e != cudaSuccess) { ::sb::set_cuda_error(_e, name); return SB_ERR_CUDA; } \
    } while (0)

// ---- optional per-stage device timing (sb_profile_begin/end; used by bench.py's roofline pass) ----
enum Stage { kStProject = 0, kStDepthSort, kStDepthScan, kStEmit, kStTileSort, kStRecords, kStBlendFwd,
             kStAccumZero, kStBlendBwd, kStGeomBwd, kNumStages };
struct ScopedStage {
    int slot; cudaStream_t st;
    ScopedStage(int stage, cudaStream_t s);
    ~ScopedStage();
};

// ---- bump allocator over a caller-owned workspace --------------------------------------
struct Carver {
    char* base; size_t off;
    __host__ explicit Carver(void* p) : base(static_cast<char*>(p)), off(0) {}
    template <typename T> __host__ T* take(size_t n) {
        off = (off + kAlign - 1) / kAlign * kAlign;
        T* r = base ? reinterpret_cast<T*>(base + off) : nullptr;
        off += n * sizeof(T);
        return r;
    }
    __host__ size_t used() const { return (off + kAlign - 1) / kAlign * kAlign; }
};

// ---- per-Gaussian state written by the projection kernel --------------------------------
// geomA = {pixel x, pixel y, conservative half-extent hx, hy of the contributing ellipse}
// geomB = {conic.x, conic.y, conic.z, opacity}
// rect  = {xmin | ymin<<16, xmax | ymax<<16} tile rectangle (getRect, auxiliary.h:46-56)
struct GeometryWs {
    int32_t*  header;        // [0]=num_rendered  [1]=num_visible  [2]=capacity overflow flag of the sync-free mode (device)
    uint32_t* depth_key;     // [P] float bits of view-space z, kCulledKey if it emits nothing
    uint32_t* tiles_touched; // [P]
    float4*   geomA;         // [P]
    float4*   geomB;         // [P]
    uint2*    rect;          // [P]
    uint32_t* sorted_key;    // [P] depth keys ascending
    uint32_t* sorted_idx;    // [P] Gaussian index in (depth, index) order
    uint32_t* offsets;       // [P] inclusive scan of tiles_touched in that order
    void*     sort_temp;     // radix_sort.cu scratch (histograms, look-back status, ping-pong pairs)
    size_t    sort_temp_bytes;
    void*     scan_temp;     // CUB inclusive-scan scratch
    size_t    scan_temp_bytes;
};
size_t geometry_scan_temp_bytes(int P);
GeometryWs carve_geometry(void* ws, int P, size_t* total);

// ---- per-instance state (R = num_rendered tile instances) -------------------------------
// Sorted SoA splat records staged by TMA into shared memory, 16 B each per array:
// recA = geomA of the instance's Gaussian, recB = geomB, recC = {r, g, b, bits(index)}.
struct BinningWs {
    uint32_t* tile_unsorted; // [R] tile id per instance, (depth,index) order
    uint32_t* val_unsorted;  // [R] Gaussian index per instance
    uint32_t* tile_sorted;   // [R]
    uint32_t* point_list;    // [R] Gaussian index, (tile, depth, index) order == reference point_list
    float4*   recA;          // [R]
    float4*   recB;          // [R]
    float4*   recC;          // [R]
    float4*   recD;          // [R] second colour set {e0, e1, e2, -} (fused two-set render only)
    void*     sort_temp;     // radix_sort.cu scratch
    size_t    sort_temp_bytes;
};
BinningWs carve_binning(void* ws, int R, int tiles, int color_sets, size_t* total);

struct ImageWs {
    uint2*    ranges;     // [tiles] [start,end) into the sorted instance list
    float*    final_T;    // [H*W]
    uint32_t* n_contrib;  // [H*W]
};
ImageWs carve_image(void* ws, int W, int H, size_t* total);

// Accumulator written by the backward blend with vector reductions, one 48-B row per Gaussian:
// {dmean2D.x, dmean2D.y, dconic.xx, dconic.xy, dconic.yy, dopacity, dcolor.r, .g, .b, pad x3}
constexpr int kAccumStride = 12;
// fused two-set render: 64-B rows {.. 9 as above .., dcolor2.rgb, dmean2D.xy from the FIRST colour set only, pad x2}
constexpr int kAccumStride2 = 16;

// ---- reference tile-id bit width (getHigherMsb, X/cuda_rasterizer/rasterizer_impl.cu:35-50) ----
inline uint32_t higher_msb(uint32_t n) {
    uint32_t msb = sizeof(n) * 4, step = msb;
    while (step > 1) { step /= 2; if (n >> msb) msb += step; else msb -= step; }
    if (n >> msb) msb++;
    return msb;
}

// ---- stage launchers (defined in the .cu files) ------------------------------------------
int launch_project(const sb_settings& s, int P, const float* means3D, const float* opacities,
                   const float* scales, const float* rotations, const float* cov3D_precomp,
                   int32_t* radii, const GeometryWs& g, cudaStream_t st);
int launch_depth_order(int P, const GeometryWs& g, cudaStream_t st);
// colors2 / out_color2 / dL2 / dL_dcolors2 == nullptr selects the plain 3-channel path
// count_dev != nullptr selects the sync-free mode: R is then the CAPACITY of the instance arrays and the true
// instance count is read on the device from *count_dev
int launch_binning(const sb_settings& s, int P, int R, const float* colors, const float* colors2,
                   const GeometryWs& g, const BinningWs& b, const ImageWs& img, const int32_t* count_dev,
                   cudaStream_t st);
int launch_finalize_count(int P, const GeometryWs& g, int capacity, cudaStream_t st);
// overflow_flag != nullptr (sync-free mode): device int that is non-zero when the instance lists were truncated; the
// images are then written as NaN
int launch_blend_forward(const sb_settings& s, int R, const GeometryWs& g, const BinningWs& b,
                         const ImageWs& img, float* out_color, float* out_color2, float* out_depth,
                         const int32_t* overflow_flag, cudaStream_t st);
int launch_blend_backward(const sb_settings& s, int R, const BinningWs& b, const ImageWs& img,
                          const float* dL_dout_color, const float* dL_dout_color2, float* accum,
                          cudaStream_t st);
int launch_geometry_backward(const sb_settings& s, int P, const float* means3D, const float* colors,
                             const float* scales, const float* rotations, const float* cov3D_precomp,
                             const int32_t* radii, const float* accum, int accum_stride,
                             float* dL_dmeans3D, float* dL_dmeans2D, float* dL_dcolors, float* dL_dcolors2,
                             float* dL_dopacity, float* dL_dscales, float* dL_drotations,
                             float* dL_dcov3D, cudaStream_t st);
int launch_mark_visible(int P, const float* means3D, const float* viewmatrix, uint8_t* present,
                        cudaStream_t st);

// ---- device helpers ------------------------------------------------------------------------
// Sum of one double per thread over a block of NT threads, in a fixed order (deterministic); `red` holds NT / 32
// doubles of shared memory.  The result is valid in thread tid == 0 only.
template <int NT>
__device__ __forceinline__ double block_sum(double v, double* red, int tid) {
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
    const int lane = tid & 31, warp = tid >> 5;
    __syncthreads();                      // red may still be read by the previous call
    if (lane == 0) red[warp] = v;
    __syncthreads();
    double s = 0.0;
    if (tid == 0)
        for (int w = 0; w < NT / 32; ++w) s += red[w];
    return s;
}

// Row k of a reference 4x4 matrix applied to a point, with the exact operation order nvcc emits
// for `m[k]*p.x + m[k+4]*p.y + m[k+8]*p.z + m[k+12]` (auxiliary.h:58-77):
//   fadd(fma(p.z, m[k+8], fma(p.x, m[k], fmul(p.y, m[k+4]))), m[k+12])
__device__ __forceinline__ float xform_row(const float* __restrict__ m, int k, float px, float py, float pz) {
    return __fadd_rn(__fmaf_rn(pz, m[k + 8], __fmaf_rn(px, m[k], __fmul_rn(py, m[k + 4]))), m[k + 12]);
}

}  // namespace sb
