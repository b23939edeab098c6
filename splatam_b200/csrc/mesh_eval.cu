// mesh_eval.cu -- the two hot parts of scoring a mesh against a ground-truth mesh (splatam_b200/mesh_eval.py):
// which points a sequence of depth frames observed, and exact nearest-neighbour distances between point sets.
//
//   sb_points_visible           points [N,3] x B frames -> mask[i] |= some frame sees point i
//   sb_nn_grid_workspace_bytes  the grid of N reference points over gx x gy x gz cells
//   sb_nn_grid_build            one u32 cell key per point, (key, index) sorted by sb::radix_sort_pairs, per-cell start
//                               offsets and the coordinates gathered into cell order
//   sb_nn_query                 per query, the minimum squared distance to the reference points
//
// Rules (float32, each operation rounded as written, no contraction; oracle/mesh_eval_numpy.py restates them):
//   * Visibility: per frame, (x, y, z) = ((r0 px + r1 py) + r2 pz) + t per row of w2c; z > 0; pixel
//     (floor(((fx x) / z) + cx + 0.5), floor(((fy y) / z) + cy + 0.5)) inside the image -- sb_tsdf_integrate's
//     projection -- and its depth d > 0 with z <= d + occlusion_eps.  A non-finite pose fails z > 0 and marks nothing.
//   * Distance: dx = qx - px, ...; d2 = (dx dx + dy dy) + dz dz.  The query returns the minimum of d2 over all
//     reference points, so it is bit-equal to a brute-force minimum whatever order cells are searched in.
//   * Search: rings of cells of growing Chebyshev radius around the query's cell (clamped into the grid).  After ring
//     r it stops when the best d2 is no larger than a lower bound on d2 for every cell outside the ring: for some axis
//     that cell lies past the ring, and on the other two axes the point lies in the grid box.  The bound is shrunk by
//     a tolerance far above the rounding of the binning and of the bound itself, so it never stops early.
#include <cmath>

#include "common.cuh"
#include "radix_sort.cuh"

namespace sb {

namespace {

constexpr int kEvalThreads = 256;
constexpr long long kMaxGridCells = 1LL << 28;

inline unsigned int eval_blocks(long long n) { return (unsigned int)((n + kEvalThreads - 1) / kEvalThreads); }

__global__ void __launch_bounds__(kEvalThreads)
points_visible_kernel(int n, const float* __restrict__ pts, int B, int H, int W, const float* __restrict__ depth,
                      const float* __restrict__ w2c, float fx, float fy, float cx, float cy, float eps,
                      uint8_t* __restrict__ mask) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint8_t was = mask[i];
    if (was) return;
    const float px = pts[3 * (size_t)i], py = pts[3 * (size_t)i + 1], pz = pts[3 * (size_t)i + 2];
    const size_t hw = (size_t)H * W;
    bool seen = false;
    for (int b = 0; b < B && !seen; ++b) {
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
        const float d = __ldg(depth + b * hw + (size_t)row * W + (size_t)col);
        seen = d > 0.f && z <= __fadd_rn(d, eps);
    }
    if (seen) mask[i] = 1;
}

struct NNGrid {
    float o[3];
    float cell;
    int g[3];
};

__device__ __forceinline__ int cell_of(const NNGrid& G, int a, float p) {
    const float t = floorf(__fdiv_rn(__fsub_rn(p, G.o[a]), G.cell));
    return (int)fminf(fmaxf(t, 0.f), (float)(G.g[a] - 1));     // fmaxf turns NaN into cell 0
}

__global__ void __launch_bounds__(kEvalThreads)
nn_key_kernel(int n, const float* __restrict__ pts, NNGrid G, uint32_t* __restrict__ keys) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int c0 = cell_of(G, 0, pts[3 * (size_t)i]), c1 = cell_of(G, 1, pts[3 * (size_t)i + 1]),
              c2 = cell_of(G, 2, pts[3 * (size_t)i + 2]);
    keys[i] = ((uint32_t)c2 * (uint32_t)G.g[1] + (uint32_t)c1) * (uint32_t)G.g[0] + (uint32_t)c0;
}

// start[c] = the first sorted position whose key is >= c, for c in [0, cells]
__global__ void __launch_bounds__(kEvalThreads)
nn_starts_kernel(int n, long long cells, const uint32_t* __restrict__ keys, uint32_t* __restrict__ start) {
    const long long c = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (c > cells) return;
    int lo = 0, hi = n;
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if ((long long)keys[mid] < c) lo = mid + 1;
        else hi = mid;
    }
    start[c] = (uint32_t)lo;
}

__global__ void __launch_bounds__(kEvalThreads)
nn_gather_kernel(int n, const float* __restrict__ pts, const uint32_t* __restrict__ idx, float4* __restrict__ out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const size_t j = idx[i];
    out[i] = make_float4(pts[3 * j], pts[3 * j + 1], pts[3 * j + 2], 0.f);
}

// distance from q to the interval [o + c0 cell, o + (c1 + 1) cell], shrunk by tol and clamped at 0
__device__ __forceinline__ float span_gap(const NNGrid& G, int a, float q, int c0, int c1, float tol) {
    const float lo = G.o[a] + (float)c0 * G.cell, hi = G.o[a] + (float)(c1 + 1) * G.cell;
    return fmaxf(fmaxf(lo - q, q - hi) - tol, 0.f);
}

struct Query {
    float q[3];
    float tol[3];
    float box2[3];   // squared distance to the grid box per axis, shrunk by tol
    int c[3];
    float best;
};

// the points of cells (x0..x1, y, z), contiguous in cell order, unless their box is farther than the best so far
__device__ __forceinline__ void scan_run(const NNGrid& G, Query& Q, int x0, int x1, int y, int z, float yz2,
                                         const uint32_t* __restrict__ start, const float4* __restrict__ pts) {
    const float gx = span_gap(G, 0, Q.q[0], x0, x1, Q.tol[0]);
    if (__fmul_rn(__fadd_rn(yz2, gx * gx), 0.999999f) > Q.best) return;
    const uint32_t row = ((uint32_t)z * (uint32_t)G.g[1] + (uint32_t)y) * (uint32_t)G.g[0];
    const uint32_t s = __ldg(start + row + x0), e = __ldg(start + row + x1 + 1);
    float best = Q.best;
    for (uint32_t k = s; k < e; ++k) {
        const float4 p = __ldg(pts + k);
        const float dx = __fsub_rn(Q.q[0], p.x), dy = __fsub_rn(Q.q[1], p.y), dz = __fsub_rn(Q.q[2], p.z);
        best = fminf(best, __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz)));
    }
    Q.best = best;
}

// lower bound on d2 for every point in a cell outside ring r
__device__ __forceinline__ float outside_bound(const NNGrid& G, const Query& Q, int r) {
    float lb = INFINITY;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        float rest = 0.f;
#pragma unroll
        for (int b = 0; b < 3; ++b)
            if (b != a) rest += Q.box2[b];
        if (Q.c[a] + r + 1 <= G.g[a] - 1) {
            const float gap = fmaxf(G.o[a] + (float)(Q.c[a] + r + 1) * G.cell - Q.q[a] - Q.tol[a], 0.f);
            lb = fminf(lb, rest + gap * gap);
        }
        if (Q.c[a] - r - 1 >= 0) {
            const float gap = fmaxf(Q.q[a] - (G.o[a] + (float)(Q.c[a] - r) * G.cell) - Q.tol[a], 0.f);
            lb = fminf(lb, rest + gap * gap);
        }
    }
    return lb * 0.999999f;
}

__global__ void __launch_bounds__(kEvalThreads)
nn_query_kernel(int m, const float* __restrict__ queries, NNGrid G, const uint32_t* __restrict__ start,
                const float4* __restrict__ pts, float* __restrict__ out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= m) return;
    Query Q;
    int rmax = 0;
    bool finite = true;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        const float q = queries[3 * (size_t)i + a];
        finite = finite && isfinite(q);
        Q.q[a] = q;
        const float hi = G.o[a] + (float)G.g[a] * G.cell;
        Q.tol[a] = 1e-5f * (fabsf(G.o[a]) + fabsf(hi) + fabsf(q) + G.cell);
        const float bg = fmaxf(fmaxf(G.o[a] - q, q - hi) - Q.tol[a], 0.f);
        Q.box2[a] = bg * bg;
        Q.c[a] = cell_of(G, a, q);
        rmax = max(rmax, max(Q.c[a], G.g[a] - 1 - Q.c[a]));
    }
    if (!finite) { out[i] = NAN; return; }
    Q.best = INFINITY;
    for (int r = 0;; ++r) {
        const int z0 = max(Q.c[2] - r, 0), z1 = min(Q.c[2] + r, G.g[2] - 1);
        const int y0 = max(Q.c[1] - r, 0), y1 = min(Q.c[1] + r, G.g[1] - 1);
        const int x0 = max(Q.c[0] - r, 0), x1 = min(Q.c[0] + r, G.g[0] - 1);
        for (int z = z0; z <= z1; ++z) {
            const float gz = span_gap(G, 2, Q.q[2], z, z, Q.tol[2]);
            const float z2 = gz * gz;
            if (__fmul_rn(z2, 0.999999f) > Q.best) continue;
            const bool zface = z == Q.c[2] - r || z == Q.c[2] + r;
            for (int y = y0; y <= y1; ++y) {
                const float gy = span_gap(G, 1, Q.q[1], y, y, Q.tol[1]);
                const float yz2 = z2 + gy * gy;
                if (__fmul_rn(yz2, 0.999999f) > Q.best) continue;
                if (zface || y == Q.c[1] - r || y == Q.c[1] + r) {
                    scan_run(G, Q, x0, x1, y, z, yz2, start, pts);
                } else {
                    if (Q.c[0] - r >= 0) scan_run(G, Q, Q.c[0] - r, Q.c[0] - r, y, z, yz2, start, pts);
                    if (r > 0 && Q.c[0] + r < G.g[0]) scan_run(G, Q, Q.c[0] + r, Q.c[0] + r, y, z, yz2, start, pts);
                }
            }
        }
        if (r >= rmax || Q.best <= outside_bound(G, Q, r)) break;
    }
    out[i] = Q.best;
}

struct NNWs {
    uint32_t* start;    // [cells + 1]
    float4* pts;        // [n] coordinates in cell order
    uint32_t* keys;     // [n] unsorted cell keys
    uint32_t* skeys;    // [n] sorted cell keys
    uint32_t* sidx;     // [n] point index in cell order
    void* sort_temp;
    size_t sort_bytes;
};

int key_bits(long long cells) {
    int b = 1;
    while ((1LL << b) < cells) ++b;
    return b;
}

NNWs carve_nn(void* ws, int n, long long cells, size_t* total) {
    Carver cv(ws);
    NNWs w;
    w.start = cv.take<uint32_t>((size_t)cells + 1);
    w.pts = cv.take<float4>(n);
    w.keys = cv.take<uint32_t>(n);
    w.skeys = cv.take<uint32_t>(n);
    w.sidx = cv.take<uint32_t>(n);
    w.sort_bytes = radix_temp_bytes(n, key_bits(cells));
    w.sort_temp = cv.take<char>(w.sort_bytes);
    *total = cv.used();
    return w;
}

bool valid_nn_grid(int n, float ox, float oy, float oz, float cell, int gx, int gy, int gz) {
    return n >= 1 && n < (1 << 30) && std::isfinite(ox) && std::isfinite(oy) && std::isfinite(oz) &&
           std::isfinite(cell) && cell > 0.f && gx >= 1 && gy >= 1 && gz >= 1 &&
           (long long)gx * gy * gz <= kMaxGridCells;
}

NNGrid make_grid(float ox, float oy, float oz, float cell, int gx, int gy, int gz) {
    NNGrid G;
    G.o[0] = ox; G.o[1] = oy; G.o[2] = oz;
    G.cell = cell;
    G.g[0] = gx; G.g[1] = gy; G.g[2] = gz;
    return G;
}

}  // namespace

}  // namespace sb

using namespace sb;

extern "C" {

SB_API int sb_points_visible(int n, const float* points, int B, int height, int width, const float* depth,
                             const float* w2c, float fx, float fy, float cx, float cy, float occlusion_eps,
                             uint8_t* mask, void* stream) {
    if (n < 0 || B < 0 || height < 1 || width < 1 || (long long)height * width >= (1LL << 31) ||
        !std::isfinite(fx) || !std::isfinite(fy) || !std::isfinite(cx) || !std::isfinite(cy) ||
        !std::isfinite(occlusion_eps) || occlusion_eps < 0.f || (n > 0 && (!points || !mask)) ||
        (n > 0 && B > 0 && (!depth || !w2c)))
        return SB_ERR_BAD_ARG;
    if (n == 0 || B == 0) return SB_OK;
    points_visible_kernel<<<eval_blocks(n), kEvalThreads, 0, static_cast<cudaStream_t>(stream)>>>(
        n, points, B, height, width, depth, w2c, fx, fy, cx, cy, occlusion_eps, mask);
    SB_LAUNCH_CHECK("points_visible_kernel");
    return SB_OK;
}

SB_API int sb_nn_grid_workspace_bytes(int n, int gx, int gy, int gz, size_t* bytes) {
    if (!valid_nn_grid(n, 0.f, 0.f, 0.f, 1.f, gx, gy, gz) || !bytes) return SB_ERR_BAD_ARG;
    carve_nn(nullptr, n, (long long)gx * gy * gz, bytes);
    return SB_OK;
}

SB_API int sb_nn_grid_build(int n, const float* points, float ox, float oy, float oz, float cell, int gx, int gy,
                            int gz, void* workspace, size_t workspace_bytes, void* stream) {
    if (!valid_nn_grid(n, ox, oy, oz, cell, gx, gy, gz) || !points || !workspace) return SB_ERR_BAD_ARG;
    const long long cells = (long long)gx * gy * gz;
    size_t need = 0;
    carve_nn(nullptr, n, cells, &need);
    if (workspace_bytes < need) return SB_ERR_WORKSPACE;
    NNWs w = carve_nn(workspace, n, cells, &need);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const NNGrid G = make_grid(ox, oy, oz, cell, gx, gy, gz);
    nn_key_kernel<<<eval_blocks(n), kEvalThreads, 0, st>>>(n, points, G, w.keys);
    SB_LAUNCH_CHECK("nn_key_kernel");
    const int rc = radix_sort_pairs(w.keys, nullptr, w.skeys, w.sidx, n, nullptr, 0, key_bits(cells), w.sort_temp,
                                    w.sort_bytes, st);
    if (rc != SB_OK) return rc;
    nn_starts_kernel<<<eval_blocks(cells + 1), kEvalThreads, 0, st>>>(n, cells, w.skeys, w.start);
    SB_LAUNCH_CHECK("nn_starts_kernel");
    nn_gather_kernel<<<eval_blocks(n), kEvalThreads, 0, st>>>(n, points, w.sidx, w.pts);
    SB_LAUNCH_CHECK("nn_gather_kernel");
    return SB_OK;
}

SB_API int sb_nn_query(int m, const float* queries, int n, float ox, float oy, float oz, float cell, int gx, int gy,
                       int gz, const void* workspace, size_t workspace_bytes, float* d2, void* stream) {
    if (m < 0 || !valid_nn_grid(n, ox, oy, oz, cell, gx, gy, gz) || !workspace || (m > 0 && (!queries || !d2)))
        return SB_ERR_BAD_ARG;
    const long long cells = (long long)gx * gy * gz;
    size_t need = 0;
    carve_nn(nullptr, n, cells, &need);
    if (workspace_bytes < need) return SB_ERR_WORKSPACE;
    if (m == 0) return SB_OK;
    NNWs w = carve_nn(const_cast<void*>(workspace), n, cells, &need);
    nn_query_kernel<<<eval_blocks(m), kEvalThreads, 0, static_cast<cudaStream_t>(stream)>>>(
        m, queries, make_grid(ox, oy, oz, cell, gx, gy, gz), w.start, w.pts, d2);
    SB_LAUNCH_CHECK("nn_query_kernel");
    return SB_OK;
}

}  // extern "C"
