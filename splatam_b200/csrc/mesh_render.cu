// mesh_render.cu -- depth maps of a triangle mesh from B cameras, for scoring a mesh by its rendered depth
// (splatam_b200/mesh_eval.py: MeshDepth, depth_l1).
//
//   sb_mesh_depth_workspace_bytes  the z-buffer keys [B,H,W] u64, one pixel count per (view, face) u64 and cub's scan
//   sb_mesh_depth                  depth [B,H,W] float32 and face_id [B,H,W] int32
//
// Rule (float32, each operation rounded as written, no contraction; oracle/mesh_render_numpy.py restates it; the
// header states it in full): per (view, face) the vertices go to camera coordinates with sb_tsdf_integrate's
// transform, the face is clipped against z = near (Sutherland-Hodgman in vertex order, new points parametrised from
// the inside vertex, z = near exactly) into a polygon of 3 or 4 vertices fanned from its first vertex, and each
// piece is projected and tested at the pixel centres of its bounding box with three edge functions evaluated in a
// canonical endpoint order.  A covered pixel's perspective-correct z goes into a 64-bit atomicMin key
// (bits(z) << 32 | face), so the result does not depend on the order of the writes.
//
// Load balance: triangles range from below a pixel to the whole image, so pixels, not faces, are the unit of work.
//   1. mesh_count_kernel, one thread per (view, face): transform, clip, project, and write the bounding-box pixel
//      count of its pieces (0, 1 or 2 of them).
//   2. cub::DeviceScan::ExclusiveSum over the B F + 1 counts, in place (sb_mc_count's scan); the last is the total.
//   3. mesh_raster_kernel, a grid sized to fill the GPU: each thread walks the pixel slots [0, total) with a grid
//      stride, finds its (view, face) by binary search in the scanned offsets, recomputes that face's pieces with the
//      same function as pass 1, and tests one pixel.  Neighbouring slots are neighbouring pixels of one piece, so a
//      large face spreads over the whole grid and its z-buffer writes coalesce.  The total is read on the device: the
//      host reads nothing.
//   4. mesh_resolve_kernel: keys -> depth (0 where nothing drew) and face_id (-1).
#include <cmath>
#include <cub/cub.cuh>

#include "common.cuh"

namespace sb {

namespace {

constexpr int kRenderThreads = 256;
constexpr unsigned long long kEmptyKey = ~0ull;

inline unsigned int render_blocks(long long n) {
    return (unsigned int)((n + kRenderThreads - 1) / kRenderThreads);
}

struct Cam {
    float fx, fy, cx, cy, near;
    int H, W;
};

struct V3 {
    float x, y, z;
};

// up to two projected triangles (u, v, z) and their clamped bounding boxes
struct Pieces {
    int n;
    float u[2][3], v[2][3], z[2][3];
    int c0[2], r0[2], nc[2], nr[2];
};

__device__ __forceinline__ float row_dot(const float* __restrict__ m, float px, float py, float pz) {
    return __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(__ldg(m), px), __fmul_rn(__ldg(m + 1), py)),
                               __fmul_rn(__ldg(m + 2), pz)), __ldg(m + 3));
}

// the point on P -> Q at z = near, P inside (z >= near) and Q outside
__device__ __forceinline__ V3 cross_near(V3 P, V3 Q, float near) {
    const float s = __fdiv_rn(__fsub_rn(near, P.z), __fsub_rn(Q.z, P.z));
    return V3{__fadd_rn(P.x, __fmul_rn(s, __fsub_rn(Q.x, P.x))), __fadd_rn(P.y, __fmul_rn(s, __fsub_rn(Q.y, P.y))),
              near};
}

// transform, drop, clip, fan, project and box face f of view b
__device__ __forceinline__ void face_pieces(int V, const float* __restrict__ verts, const int* __restrict__ faces,
                                            const float* __restrict__ m, int f, const Cam& C, Pieces& out) {
    out.n = 0;
#pragma unroll
    for (int t = 0; t < 2; ++t) out.c0[t] = out.r0[t] = out.nc[t] = out.nr[t] = 0;   // a dropped face counts 0
    V3 p[3];
    bool finite = true;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const int i = __ldg(faces + 3 * (size_t)f + k);
        if (i < 0 || i >= V) return;
        const float px = __ldg(verts + 3 * (size_t)i), py = __ldg(verts + 3 * (size_t)i + 1),
                    pz = __ldg(verts + 3 * (size_t)i + 2);
        p[k] = V3{row_dot(m, px, py, pz), row_dot(m + 4, px, py, pz), row_dot(m + 8, px, py, pz)};
        finite = finite && isfinite(p[k].x) && isfinite(p[k].y) && isfinite(p[k].z);
    }
    if (!finite) return;
    V3 poly[4];
    int np = 0;
    // put() selects the slot with constant indices, so poly stays in registers
    auto put = [&](const V3& q) {
        if (np == 0) poly[0] = q;
        else if (np == 1) poly[1] = q;
        else if (np == 2) poly[2] = q;
        else poly[3] = q;
        ++np;
    };
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const V3 P = p[k], Q = p[(k + 1) % 3];
        const bool inP = P.z >= C.near, inQ = Q.z >= C.near;
        if (inP) put(P);
        if (inP && !inQ) put(cross_near(P, Q, C.near));
        if (!inP && inQ) put(cross_near(Q, P, C.near));
    }
    if (np < 3) return;
    float pu[4], pv[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        if (k < np) {
            pu[k] = __fadd_rn(__fdiv_rn(__fmul_rn(C.fx, poly[k].x), poly[k].z), C.cx);
            pv[k] = __fadd_rn(__fdiv_rn(__fmul_rn(C.fy, poly[k].y), poly[k].z), C.cy);
        }
    }
    out.n = np - 2;
#pragma unroll
    for (int t = 0; t < 2; ++t) {
        if (t < out.n) {
            const int idx[3] = {0, t + 1, t + 2};
            float umin = INFINITY, umax = -INFINITY, vmin = INFINITY, vmax = -INFINITY;
#pragma unroll
            for (int k = 0; k < 3; ++k) {
                out.u[t][k] = pu[idx[k]];
                out.v[t][k] = pv[idx[k]];
                out.z[t][k] = poly[idx[k]].z;
                umin = fminf(umin, out.u[t][k]); umax = fmaxf(umax, out.u[t][k]);
                vmin = fminf(vmin, out.v[t][k]); vmax = fmaxf(vmax, out.v[t][k]);
            }
            const float c0 = fmaxf(ceilf(umin), 0.f), c1 = fminf(floorf(umax), (float)(C.W - 1));
            const float r0 = fmaxf(ceilf(vmin), 0.f), r1 = fminf(floorf(vmax), (float)(C.H - 1));
            const bool any = c0 <= c1 && r0 <= r1;
            out.c0[t] = any ? (int)c0 : 0;
            out.r0[t] = any ? (int)r0 : 0;
            out.nc[t] = any ? (int)c1 - (int)c0 + 1 : 0;
            out.nr[t] = any ? (int)r1 - (int)r0 + 1 : 0;
        }
    }
}

// the edge function of P -> Q at pixel (c, r), from the endpoints in lexicographic (u, v) order, negated if swapped
__device__ __forceinline__ float edge(float uP, float vP, float uQ, float vQ, float c, float r) {
    const bool swap = uQ < uP || (uQ == uP && vQ < vP);
    const float u0 = swap ? uQ : uP, v0 = swap ? vQ : vP, u1 = swap ? uP : uQ, v1 = swap ? vP : vQ;
    const float e = __fsub_rn(__fmul_rn(__fsub_rn(u1, u0), __fsub_rn(r, v0)),
                              __fmul_rn(__fsub_rn(v1, v0), __fsub_rn(c, u0)));
    return swap ? -e : e;
}

__global__ void __launch_bounds__(kRenderThreads)
mesh_count_kernel(int V, const float* __restrict__ verts, int F, const int* __restrict__ faces, int B,
                  const float* __restrict__ w2c, Cam C, unsigned long long* __restrict__ counts) {
    const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    const long long n = (long long)B * F;
    if (i > n) return;
    if (i == n) { counts[n] = 0; return; }
    const int b = (int)(i / F), f = (int)(i - (long long)b * F);
    Pieces P;
    face_pieces(V, verts, faces, w2c + 16 * b, f, C, P);
    counts[i] = (unsigned long long)P.nc[0] * P.nr[0] + (unsigned long long)P.nc[1] * P.nr[1];
}

__global__ void __launch_bounds__(kRenderThreads, 2)   // room for the two pieces without spilling
mesh_raster_kernel(int V, const float* __restrict__ verts, int F, const int* __restrict__ faces, int B,
                   const float* __restrict__ w2c, Cam C, const unsigned long long* __restrict__ offs,
                   unsigned long long* __restrict__ keys) {
    const long long n = (long long)B * F;
    const unsigned long long total = offs[n];
    const unsigned long long stride = (unsigned long long)gridDim.x * blockDim.x;
    for (unsigned long long j = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x; j < total; j += stride) {
        long long lo = 0, hi = n;     // the last i with offs[i] <= j; offs[0] = 0 <= j < offs[n]
        while (hi - lo > 1) {
            const long long mid = (lo + hi) >> 1;
            if (__ldg(offs + mid) <= j) lo = mid;
            else hi = mid;
        }
        const int b = (int)(lo / F), f = (int)(lo - (long long)b * F);
        Pieces P;
        face_pieces(V, verts, faces, w2c + 16 * b, f, C, P);
        unsigned int k = (unsigned int)(j - __ldg(offs + lo));
        const unsigned int n0 = (unsigned int)P.nc[0] * (unsigned int)P.nr[0];
        const int t = k < n0 ? 0 : 1;
        if (t) k -= n0;
        const int ncol = t ? P.nc[1] : P.nc[0];
        const float c = (float)((t ? P.c0[1] : P.c0[0]) + (int)(k % (unsigned int)ncol));
        const float r = (float)((t ? P.r0[1] : P.r0[0]) + (int)(k / (unsigned int)ncol));
        float u[3], v[3], z[3];
#pragma unroll
        for (int q = 0; q < 3; ++q) {
            u[q] = t ? P.u[1][q] : P.u[0][q];
            v[q] = t ? P.v[1][q] : P.v[0][q];
            z[q] = t ? P.z[1][q] : P.z[0][q];
        }
        const float ea = edge(u[1], v[1], u[2], v[2], c, r);     // opposite vertex a: b -> c
        const float eb = edge(u[2], v[2], u[0], v[0], c, r);     // opposite vertex b: c -> a
        const float ec = edge(u[0], v[0], u[1], v[1], c, r);     // opposite vertex c: a -> b
        const bool inside = (ea >= 0.f && eb >= 0.f && ec >= 0.f) || (ea <= 0.f && eb <= 0.f && ec <= 0.f);
        const float s = __fadd_rn(__fadd_rn(ea, eb), ec);
        if (!inside || s == 0.f) continue;
        const float iz = __fdiv_rn(__fadd_rn(__fadd_rn(__fdiv_rn(ea, z[0]), __fdiv_rn(eb, z[1])), __fdiv_rn(ec, z[2])),
                                   s);
        const float zz = __fdiv_rn(1.f, iz);
        if (!(isfinite(zz) && zz > 0.f)) continue;
        const unsigned long long key = ((unsigned long long)__float_as_uint(zz) << 32) | (unsigned int)f;
        atomicMin(keys + ((size_t)b * C.H + (size_t)r) * C.W + (size_t)c, key);
    }
}

__global__ void __launch_bounds__(kRenderThreads)
mesh_resolve_kernel(long long n, const unsigned long long* __restrict__ keys, float* __restrict__ depth,
                    int* __restrict__ face_id) {
    const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (i >= n) return;
    const unsigned long long k = keys[i];
    const bool hit = k != kEmptyKey;
    depth[i] = hit ? __uint_as_float((unsigned int)(k >> 32)) : 0.f;
    face_id[i] = hit ? (int)(unsigned int)k : -1;
}

struct RenderWs {
    unsigned long long* keys;   // [B H W]
    unsigned long long* offs;   // [B F + 1] counts, scanned in place
    void* scan_temp;
    size_t scan_bytes;
};

RenderWs carve_render(void* ws, int F, int B, int H, int W, size_t* total) {
    Carver cv(ws);
    RenderWs w;
    const long long n = (long long)B * F;
    w.keys = cv.take<unsigned long long>((size_t)B * H * W);
    w.offs = cv.take<unsigned long long>(n + 1);
    w.scan_bytes = 0;
    cub::DeviceScan::ExclusiveSum(nullptr, w.scan_bytes, (unsigned long long*)nullptr, (unsigned long long*)nullptr,
                                  (int)(n + 1));
    w.scan_temp = cv.take<char>(w.scan_bytes);
    *total = cv.used();
    return w;
}

bool valid_render_sizes(int F, int B, int H, int W) {
    return F >= 1 && B >= 1 && H >= 1 && W >= 1 && (long long)B * H * W < (1LL << 31) &&
           (long long)B * F < (1LL << 31) - 1;
}

}  // namespace

}  // namespace sb

using namespace sb;

extern "C" {

SB_API int sb_mesh_depth_workspace_bytes(int f, int B, int height, int width, size_t* bytes) {
    if (!valid_render_sizes(f, B, height, width) || !bytes) return SB_ERR_BAD_ARG;
    carve_render(nullptr, f, B, height, width, bytes);
    return SB_OK;
}

SB_API int sb_mesh_depth(int v, const float* vertices, int f, const int* faces, int B, int height, int width,
                         const float* w2c, float fx, float fy, float cx, float cy, float near, void* workspace,
                         size_t workspace_bytes, float* depth, int* face_id, void* stream) {
    if (v < 1 || !valid_render_sizes(f, B, height, width) || !vertices || !faces || !w2c || !workspace || !depth ||
        !face_id || !(std::isfinite(fx) && fx > 0.f) || !(std::isfinite(fy) && fy > 0.f) || !std::isfinite(cx) ||
        !std::isfinite(cy) || !(std::isfinite(near) && near > 0.f))
        return SB_ERR_BAD_ARG;
    size_t need = 0;
    carve_render(nullptr, f, B, height, width, &need);
    if (workspace_bytes < need) return SB_ERR_WORKSPACE;
    RenderWs w = carve_render(workspace, f, B, height, width, &need);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const long long pixels = (long long)B * height * width, n = (long long)B * f;
    const Cam C{fx, fy, cx, cy, near, height, width};
    int dev = 0, sms = 0;
    SB_CUDA_CHECK(cudaGetDevice(&dev));
    SB_CUDA_CHECK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    SB_CUDA_CHECK(cudaMemsetAsync(w.keys, 0xFF, (size_t)pixels * sizeof(unsigned long long), st));
    mesh_count_kernel<<<render_blocks(n + 1), kRenderThreads, 0, st>>>(v, vertices, f, faces, B, w2c, C, w.offs);
    SB_LAUNCH_CHECK("mesh_count_kernel");
    SB_CUDA_CHECK(cub::DeviceScan::ExclusiveSum(w.scan_temp, w.scan_bytes, w.offs, w.offs, (int)(n + 1), st));
    mesh_raster_kernel<<<sms * (2048 / kRenderThreads), kRenderThreads, 0, st>>>(v, vertices, f, faces, B, w2c, C,
                                                                                 w.offs, w.keys);
    SB_LAUNCH_CHECK("mesh_raster_kernel");
    mesh_resolve_kernel<<<render_blocks(pixels), kRenderThreads, 0, st>>>(pixels, w.keys, depth, face_id);
    SB_LAUNCH_CHECK("mesh_resolve_kernel");
    return SB_OK;
}

}  // extern "C"
