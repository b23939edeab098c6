// mesh.cu -- a coloured triangle mesh from depth frames: TSDF fusion into a dense volume and marching cubes
// (splatam_b200/mesh.py).
//
//   sb_tsdf_integrate   B depth/colour frames -> the volume's tsdf, weight [nz,ny,nx] and color [nz,ny,nx,3]
//   sb_mc_count         pass 1: per sample, its vertices and its cell's triangles; one scan; the totals (V, F)
//   sb_mc_emit          pass 2: vertices in ascending edge id, faces in ascending cell then table order
//
// Rules (float32, each operation rounded as written, no contraction; oracle/mesh_numpy.py restates them):
//   * Integration: one thread owns one voxel, applies the B frames in order in registers and writes the state back
//     once, only if a frame changed it (a voxel no frame touches costs its coordinates only).  Per frame:
//     p = o + v * float(idx) per axis; (x, y, z) = ((r0 px + r1 py) + r2 pz) + t per row of w2c; z > 0;
//     u = ((fx x) / z) + cx, v likewise; pixel (floor(u + 0.5), floor(v + 0.5)) in the image; its depth d > 0 and
//     d <= depth_max; sdf = d - z >= -trunc; f = min(1, sdf / trunc); W' = W + 1, T' = (T W + f) / W',
//     C' = (C W + rgb) / W'.
//   * Marching cubes: a cell is live iff its 8 samples have W >= min_weight; a sample is inside iff T < 0.  Edge
//     (s, axis), id 3 s + axis, carries a vertex iff it is crossed and touches a live cell; the vertex sits at
//     p_s + t * voxel along the axis, t = T_a / (T_a - T_b), colour C_a + t * (C_b - C_a).  Triangles of a live cell
//     come from the generated table (mc_table.h) and face increasing T.
#include <cmath>

#include <cub/cub.cuh>

#include "common.cuh"
#include "mc_table.h"

namespace sb {

namespace {

constexpr int kMeshThreads = 256;

inline unsigned int blocks_for(long long n) { return (unsigned int)((n + kMeshThreads - 1) / kMeshThreads); }

__global__ void __launch_bounds__(kMeshThreads)
tsdf_integrate_kernel(int nx, int ny, int nz, float ox, float oy, float oz, float voxel, float trunc, int B, int H,
                      int W, const float* __restrict__ depth, const float* __restrict__ rgb,
                      const float* __restrict__ w2c, float fx, float fy, float cx, float cy, float depth_max,
                      float* __restrict__ tsdf, float* __restrict__ weight, float* __restrict__ color) {
    const long long s = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    const long long n = (long long)nx * ny * nz;
    if (s >= n) return;
    const int i = (int)(s % nx);
    const long long r = s / nx;
    const int j = (int)(r % ny), k = (int)(r / ny);
    const float px = __fadd_rn(ox, __fmul_rn(voxel, (float)i));
    const float py = __fadd_rn(oy, __fmul_rn(voxel, (float)j));
    const float pz = __fadd_rn(oz, __fmul_rn(voxel, (float)k));
    const size_t hw = (size_t)H * W;
    float T = 0.f, Wt = 0.f, c0 = 0.f, c1 = 0.f, c2 = 0.f;
    bool loaded = false;
    for (int b = 0; b < B; ++b) {
        const float* m = w2c + 16 * b;
        const float z = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(__ldg(m + 8), px), __fmul_rn(__ldg(m + 9), py)),
                                            __fmul_rn(__ldg(m + 10), pz)), __ldg(m + 11));
        if (!(z > 0.f)) continue;
        const float x = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(__ldg(m + 0), px), __fmul_rn(__ldg(m + 1), py)),
                                            __fmul_rn(__ldg(m + 2), pz)), __ldg(m + 3));
        const float y = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(__ldg(m + 4), px), __fmul_rn(__ldg(m + 5), py)),
                                            __fmul_rn(__ldg(m + 6), pz)), __ldg(m + 7));
        const float u = __fadd_rn(__fdiv_rn(__fmul_rn(fx, x), z), cx);
        const float v = __fadd_rn(__fdiv_rn(__fmul_rn(fy, y), z), cy);
        const float col = floorf(__fadd_rn(u, 0.5f)), row = floorf(__fadd_rn(v, 0.5f));
        if (!(col >= 0.f && col < (float)W && row >= 0.f && row < (float)H)) continue;
        const size_t q = (size_t)row * W + (size_t)col;
        const float d = __ldg(depth + b * hw + q);
        if (!(d > 0.f && d <= depth_max)) continue;
        const float sdf = __fsub_rn(d, z);
        if (sdf < -trunc) continue;
        const float f = fminf(1.f, __fdiv_rn(sdf, trunc));
        if (!loaded) {
            T = tsdf[s]; Wt = weight[s];
            c0 = color[3 * s]; c1 = color[3 * s + 1]; c2 = color[3 * s + 2];
            loaded = true;
        }
        const float w1 = __fadd_rn(Wt, 1.f);
        const float* im = rgb + 3 * b * hw + q;
        T = __fdiv_rn(__fadd_rn(__fmul_rn(T, Wt), f), w1);
        c0 = __fdiv_rn(__fadd_rn(__fmul_rn(c0, Wt), __ldg(im)), w1);
        c1 = __fdiv_rn(__fadd_rn(__fmul_rn(c1, Wt), __ldg(im + hw)), w1);
        c2 = __fdiv_rn(__fadd_rn(__fmul_rn(c2, Wt), __ldg(im + 2 * hw)), w1);
        Wt = w1;
    }
    if (loaded) {
        tsdf[s] = T; weight[s] = Wt;
        color[3 * s] = c0; color[3 * s + 1] = c1; color[3 * s + 2] = c2;
    }
}

struct Grid {
    int nx, ny, nz;
    __device__ long long stride(int axis) const { return axis == 0 ? 1 : axis == 1 ? nx : (long long)nx * ny; }
    __device__ int dim(int axis) const { return axis == 0 ? nx : axis == 1 ? ny : nz; }
};

__device__ __forceinline__ long long corner_offset(Grid g, int c) {
    return (c & 1) + (c >> 1 & 1) * g.stride(1) + (c >> 2 & 1) * g.stride(2);
}

__device__ __forceinline__ int cell_case(Grid g, long long s, const float* __restrict__ tsdf) {
    int cs = 0;
#pragma unroll
    for (int c = 0; c < 8; ++c) cs |= (tsdf[s + corner_offset(g, c)] < 0.f) << c;
    return cs;
}

constexpr uint8_t kLiveBit = 8;   // flags bit 3: the cell whose lowest sample is s is live; bits 0-2: edge vertices

// pass 1a: flags[s] = kLiveBit iff the cell at sample s exists and its 8 samples have W >= min_weight
__global__ void __launch_bounds__(kMeshThreads)
mc_live_kernel(Grid g, const float* __restrict__ weight, float min_weight, uint8_t* __restrict__ flags) {
    const long long s = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (s >= (long long)g.nx * g.ny * g.nz) return;
    const int i = (int)(s % g.nx), j = (int)((s / g.nx) % g.ny), k = (int)(s / ((long long)g.nx * g.ny));
    bool live = i < g.nx - 1 && j < g.ny - 1 && k < g.nz - 1;
#pragma unroll
    for (int c = 0; c < 8; ++c) live = live && weight[s + corner_offset(g, c)] >= min_weight;
    flags[s] = live ? kLiveBit : 0;
}

// pass 1b: counts[s] = (triangles of cell s) << 32 | (vertices on the edges of sample s); edge bits into flags[s]
__global__ void __launch_bounds__(kMeshThreads)
mc_count_kernel(Grid g, const float* __restrict__ tsdf, unsigned long long* __restrict__ counts,
                uint8_t* __restrict__ flags) {
    const long long n = (long long)g.nx * g.ny * g.nz;
    const long long s = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (s > n) return;
    if (s == n) { counts[n] = 0ull; return; }
    const int i = (int)(s % g.nx), j = (int)((s / g.nx) % g.ny), k = (int)(s / ((long long)g.nx * g.ny));
    const unsigned int own = flags[s];
    const unsigned int ntri = own & kLiveBit ? kMcTriCount[cell_case(g, s, tsdf)] : 0u;
    const bool in = tsdf[s] < 0.f;
    unsigned int f = 0;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        if ((a == 0 ? i : a == 1 ? j : k) >= g.dim(a) - 1 || in == (tsdf[s + g.stride(a)] < 0.f)) continue;
        // the up to four cells around the edge: one step down on either or both of the other two axes
        const int b0 = (a + 1) % 3, b1 = (a + 2) % 3;
        const bool d0 = (b0 == 0 ? i : b0 == 1 ? j : k) > 0, d1 = (b1 == 0 ? i : b1 == 1 ? j : k) > 0;
        bool adj = own & kLiveBit;
        adj = adj || (d0 && (flags[s - g.stride(b0)] & kLiveBit));
        adj = adj || (d1 && (flags[s - g.stride(b1)] & kLiveBit));
        adj = adj || (d0 && d1 && (flags[s - g.stride(b0) - g.stride(b1)] & kLiveBit));
        if (adj) f |= 1u << a;
    }
    counts[s] = ((unsigned long long)ntri << 32) | (unsigned int)__popc(f);
    // written after every neighbour read the live bits: the other threads read only kLiveBit, which this keeps
    flags[s] = (uint8_t)(own | f);
}

__global__ void mc_totals_kernel(const unsigned long long* __restrict__ offs, long long n, int* __restrict__ totals) {
    const unsigned long long t = offs[n];
    const unsigned long long nv = t & 0xffffffffull, nf = t >> 32;
    // 3 indices per face and 3 floats per vertex are addressed with int32 offsets in the callers
    totals[0] = nv < (1ull << 31) / 3 ? (int)nv : -1;
    totals[1] = nf < (1ull << 31) / 3 ? (int)nf : -1;
}

__global__ void __launch_bounds__(kMeshThreads)
mc_emit_kernel(Grid g, float ox, float oy, float oz, float voxel, const float* __restrict__ tsdf,
               const float* __restrict__ color, const unsigned long long* __restrict__ offs,
               const uint8_t* __restrict__ flags, float* __restrict__ verts, float* __restrict__ vcols,
               int* __restrict__ faces) {
    const long long n = (long long)g.nx * g.ny * g.nz;
    const long long s = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (s >= n) return;
    const unsigned long long o = offs[s], o1 = offs[s + 1];
    if (o == o1) return;
    const int idx[3] = {(int)(s % g.nx), (int)((s / g.nx) % g.ny), (int)(s / ((long long)g.nx * g.ny))};
    const unsigned int f = flags[s] & 7u;
    unsigned int r = (unsigned int)(o & 0xffffffffull);
    if (f) {
        const float p[3] = {__fadd_rn(ox, __fmul_rn(voxel, (float)idx[0])),
                            __fadd_rn(oy, __fmul_rn(voxel, (float)idx[1])),
                            __fadd_rn(oz, __fmul_rn(voxel, (float)idx[2]))};
        const float ta = tsdf[s];
        for (int a = 0; a < 3; ++a) {
            if (!(f >> a & 1)) continue;
            const long long sb = s + g.stride(a);
            const float t = __fdiv_rn(ta, __fsub_rn(ta, tsdf[sb]));
            float q[3] = {p[0], p[1], p[2]};
            q[a] = __fadd_rn(p[a], __fmul_rn(t, voxel));
            for (int c = 0; c < 3; ++c) {
                const float ca = color[3 * s + c], cb = color[3 * sb + c];
                verts[3 * (size_t)r + c] = q[c];
                vcols[3 * (size_t)r + c] = __fadd_rn(ca, __fmul_rn(t, __fsub_rn(cb, ca)));
            }
            ++r;
        }
    }
    const unsigned int t0 = (unsigned int)(o >> 32), nt = (unsigned int)(o1 >> 32) - t0;
    if (nt == 0) return;
    const int cs = cell_case(g, s, tsdf);
    for (unsigned int m = 0; m < nt; ++m) {
        for (int q = 0; q < 3; ++q) {
            const int e = kMcTriEdges[cs][3 * m + q];
            const int c = kMcEdgeCorner[e], a = kMcEdgeAxis[e];
            const long long se = s + corner_offset(g, c);
            const unsigned int v = (unsigned int)(offs[se] & 0xffffffffull) + __popc(flags[se] & ((1u << a) - 1u));
            faces[3 * (size_t)(t0 + m) + q] = (int)v;
        }
    }
}

struct McWs {
    unsigned long long* offs;   // [N + 1] counts, scanned in place into offsets
    uint8_t* flags;             // [N]
    void* scan_temp;
    size_t scan_bytes;
};

bool valid_grid(int nx, int ny, int nz) {
    return nx >= 1 && ny >= 1 && nz >= 1 && (long long)nx * ny * nz < (1LL << 31) - 1;
}

// the packed count holds up to 3 vertices per sample in its low 32 bits and up to kMcMaxTriangles triangles per cell
// in its high 32 bits: neither scanned total may wrap
bool valid_mc_grid(int nx, int ny, int nz) {
    static_assert(kMcMaxTriangles >= 3, "the triangle bound also bounds the vertex total");
    return valid_grid(nx, ny, nz) && kMcMaxTriangles * (long long)nx * ny * nz < (1LL << 32);
}

McWs carve_mc(void* ws, long long n) {
    Carver cv(ws);
    McWs w;
    w.offs = cv.take<unsigned long long>(n + 1);
    w.flags = cv.take<uint8_t>(n);
    w.scan_bytes = 0;
    cub::DeviceScan::ExclusiveSum(nullptr, w.scan_bytes, (unsigned long long*)nullptr, (unsigned long long*)nullptr,
                                  (int)(n + 1));
    w.scan_temp = cv.take<char>(w.scan_bytes);
    w.scan_bytes = cv.used() - (size_t)((char*)w.scan_temp - (char*)ws);
    return w;
}

size_t mc_bytes(long long n) {
    Carver cv(nullptr);
    cv.take<unsigned long long>(n + 1);
    cv.take<uint8_t>(n);
    size_t scan = 0;
    cub::DeviceScan::ExclusiveSum(nullptr, scan, (unsigned long long*)nullptr, (unsigned long long*)nullptr,
                                  (int)(n + 1));
    cv.take<char>(scan);
    return cv.used();
}

}  // namespace

}  // namespace sb

using namespace sb;

extern "C" {

SB_API int sb_tsdf_integrate(int nx, int ny, int nz, float ox, float oy, float oz, float voxel, float trunc, int B,
                             int height, int width, const float* depth, const float* rgb, const float* w2c, float fx,
                             float fy, float cx, float cy, float depth_max, float* tsdf, float* weight, float* color,
                             void* stream) {
    if (!valid_grid(nx, ny, nz) || !std::isfinite(ox) || !std::isfinite(oy) || !std::isfinite(oz) || !(voxel > 0.f) ||
        !std::isfinite(voxel) || !(trunc > 0.f) || !std::isfinite(trunc) || B < 0 || height < 1 || width < 1 ||
        (long long)height * width >= (1LL << 31) || !std::isfinite(fx) || !std::isfinite(fy) || !std::isfinite(cx) ||
        !std::isfinite(cy) || !(depth_max > 0.f) || !tsdf || !weight || !color ||
        (B > 0 && (!depth || !rgb || !w2c)))
        return SB_ERR_BAD_ARG;
    if (B == 0) return SB_OK;
    const long long n = (long long)nx * ny * nz;
    tsdf_integrate_kernel<<<blocks_for(n), kMeshThreads, 0, static_cast<cudaStream_t>(stream)>>>(
        nx, ny, nz, ox, oy, oz, voxel, trunc, B, height, width, depth, rgb, w2c, fx, fy, cx, cy, depth_max, tsdf,
        weight, color);
    SB_LAUNCH_CHECK("tsdf_integrate_kernel");
    return SB_OK;
}

SB_API int sb_mc_workspace_bytes(int nx, int ny, int nz, size_t* bytes) {
    if (!valid_mc_grid(nx, ny, nz) || !bytes) return SB_ERR_BAD_ARG;
    *bytes = mc_bytes((long long)nx * ny * nz);
    return SB_OK;
}

SB_API int sb_mc_count(int nx, int ny, int nz, const float* tsdf, const float* weight, float min_weight,
                       void* workspace, size_t workspace_bytes, int* totals, void* stream) {
    if (!valid_mc_grid(nx, ny, nz) || !tsdf || !weight || !workspace || !totals || !std::isfinite(min_weight))
        return SB_ERR_BAD_ARG;
    const long long n = (long long)nx * ny * nz;
    if (workspace_bytes < mc_bytes(n)) return SB_ERR_WORKSPACE;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    McWs w = carve_mc(workspace, n);
    mc_live_kernel<<<blocks_for(n), kMeshThreads, 0, st>>>(Grid{nx, ny, nz}, weight, min_weight, w.flags);
    SB_LAUNCH_CHECK("mc_live_kernel");
    mc_count_kernel<<<blocks_for(n + 1), kMeshThreads, 0, st>>>(Grid{nx, ny, nz}, tsdf, w.offs, w.flags);
    SB_LAUNCH_CHECK("mc_count_kernel");
    SB_CUDA_CHECK(cub::DeviceScan::ExclusiveSum(w.scan_temp, w.scan_bytes, w.offs, w.offs, (int)(n + 1), st));
    mc_totals_kernel<<<1, 1, 0, st>>>(w.offs, n, totals);
    SB_LAUNCH_CHECK("mc_totals_kernel");
    return SB_OK;
}

SB_API int sb_mc_emit(int nx, int ny, int nz, float ox, float oy, float oz, float voxel, const float* tsdf,
                      const float* color, void* workspace, size_t workspace_bytes, float* vertices, float* colors,
                      int* faces, void* stream) {
    if (!valid_mc_grid(nx, ny, nz) || !std::isfinite(ox) || !std::isfinite(oy) || !std::isfinite(oz) ||
        !(voxel > 0.f) || !std::isfinite(voxel) || !tsdf || !color || !workspace)
        return SB_ERR_BAD_ARG;
    const long long n = (long long)nx * ny * nz;
    if (workspace_bytes < mc_bytes(n)) return SB_ERR_WORKSPACE;
    McWs w = carve_mc(workspace, n);
    mc_emit_kernel<<<blocks_for(n), kMeshThreads, 0, static_cast<cudaStream_t>(stream)>>>(
        Grid{nx, ny, nz}, ox, oy, oz, voxel, tsdf, color, w.offs, w.flags, vertices, colors, faces);
    SB_LAUNCH_CHECK("mc_emit_kernel");
    return SB_OK;
}

}  // extern "C"
