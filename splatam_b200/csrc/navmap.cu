// navmap.cu -- navigation maps from a TSDF volume (splatam_b200/navmap.py): occupancy labels, an exact Euclidean
// signed distance field and trilinear distance queries.
//
//   sb_nav_labels     tsdf, weight -> labels uint8 (0 unknown, 1 free, 2 occupied)
//   sb_esdf           labels -> sd2 int32 (signed squared lattice distance) and esdf float32 (metres)
//   sb_esdf_query     esdf, points [N,3] -> dist [N], grad [N,3]
//
// The rules are stated in include/splatam_b200.h and restated in oracle/navmap_numpy.py.
//
// The distance transform is separable (Felzenszwalb & Huttenlocher, "Distance Transforms of Sampled Functions"):
// d(s) = min over sites of |s - o|^2 is three 1D lower envelopes of parabolas, along x, then y, then z.  Both signs run
// at once: sign 0 measures the distance to the obstacle set O (buffer A), sign 1 the distance to its complement
// (buffer B).  Pass x starts from the mask (f = 0 on a site, no parabola elsewhere); passes y and z take the previous
// pass's squared distances.  One thread owns one line of one sign; neighbouring threads own neighbouring lines, which
// for passes y and z are neighbouring x, so their strided reads coalesce.  The envelope stack of a line, (site,
// f(site)) pairs, lives in the workspace at [entry][line], so it coalesces too; its second phase reads only the stack,
// so passes y and z write their line in place.  Every envelope comparison is an int64 cross-multiplication: no
// rounding anywhere before the final square root.  After pass z a sample of O has A = 0 and B >= 1, any other sample
// B = 0 and A >= 1, so sign 0 writes sd2 = +A where A > 0 and sign 1 writes sd2 = -B where B > 0.
#include <cmath>

#include "common.cuh"

namespace sb {

namespace {

constexpr int kNavThreads = 256;
constexpr int kEdtThreads = 128;
constexpr int kEdtChunk = 8;            // samples of a line loaded ahead of the envelope update
constexpr int kNoSite = 0x7fffffff;     // f of a sample that is no site: the line has no obstacle (yet) in reach
constexpr int kMaxDim = 8192;

inline unsigned int blocks_of(long long n, int t) { return (unsigned int)((n + t - 1) / t); }

__global__ void __launch_bounds__(kNavThreads)
nav_labels_kernel(long long n, const float* __restrict__ tsdf, const float* __restrict__ weight, float trunc,
                  float min_weight, float occ_dist, uint8_t* __restrict__ labels) {
    const long long s = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (s >= n) return;
    const float w = weight[s];
    uint8_t l = 0;
    if (!(w < min_weight)) l = __fmul_rn(tsdf[s], trunc) <= occ_dist ? 2 : 1;
    labels[s] = l;
}

struct Line {
    long long base, stride;
    int n;
};

// line `line` of `axis`: lines of x are indexed by (j, k), of y by (i, k), of z by (i, j), i fastest
__device__ __forceinline__ Line line_of(int axis, int nx, int ny, int nz, long long line) {
    if (axis == 0) return Line{line * nx, 1, nx};
    if (axis == 1) {
        const long long i = line % nx, k = line / nx;
        return Line{k * nx * (long long)ny + i, nx, ny};
    }
    return Line{line, (long long)nx * ny, nz};
}

// One pass of the exact 1D transform d(q) = min over sites v of (q - v)^2 + f(v) along `axis`, for both signs
// (blockIdx.y).  AXIS 0 reads the labels; AXIS 1 and 2 read buf (A for sign 0, B for sign 1).  AXIS 0 and 1 write buf;
// AXIS 2 writes the signed results.
template <int AXIS>
__global__ void __launch_bounds__(kEdtThreads)
edt_pass_kernel(int nx, int ny, int nz, long long nlines, const uint8_t* __restrict__ labels, int unknown_is_obstacle,
                int* __restrict__ bufA, int* __restrict__ bufB, int2* __restrict__ stacks, float voxel,
                int* __restrict__ sd2, float* __restrict__ esdf) {
    const long long line = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (line >= nlines) return;
    const int sign = blockIdx.y;
    const long long n_all = (long long)nx * ny * nz;
    int* __restrict__ buf = sign ? bufB : bufA;
    int2* __restrict__ stack = stacks + sign * n_all + line;     // entry k at stack[k * nlines]
    const Line L = line_of(AXIS, nx, ny, nz, line);

    // phase 1: the lower envelope.  The top entry (vk, fk) and the one below it (vp, fp) stay in registers; the
    // boundary z[k] between them is num_k / den_k with num_k = (fk + vk^2) - (fp + vp^2), den_k = 2 (vk - vp).
    int k = -1;
    int vk = 0, fk = 0, vp = 0, fp = 0;
    for (int q0 = 0; q0 < L.n; q0 += kEdtChunk) {
        // the chunk's loads are issued together, so a thread keeps kEdtChunk of them in flight
        int fc[kEdtChunk];
#pragma unroll
        for (int c = 0; c < kEdtChunk; ++c) {
            const int q = q0 + c;
            if (q >= L.n) {
                fc[c] = kNoSite;
            } else if (AXIS == 0) {
                const uint8_t l = labels[L.base + q * L.stride];
                const bool in_o = l == 2 || (unknown_is_obstacle && l == 0);
                fc[c] = in_o != (sign != 0) ? 0 : kNoSite;
            } else {
                fc[c] = buf[L.base + q * L.stride];
            }
        }
#pragma unroll
        for (int c = 0; c < kEdtChunk; ++c) {
            const int q = q0 + c, fq = fc[c];
            if (fq == kNoSite) continue;
            const long long cq = fq + (long long)q * q;
            while (k > 0) {
                // s = ((fq + q^2) - (fk + vk^2)) / (2 (q - vk)); pop the top while s <= z[k]
                const long long num = cq - (fk + (long long)vk * vk), den = 2LL * (q - vk);
                const long long numk = (fk + (long long)vk * vk) - (fp + (long long)vp * vp), denk = 2LL * (vk - vp);
                if (num * denk > numk * den) break;
                --k;
                vk = vp; fk = fp;
                if (k > 0) {
                    const int2 e = stack[(long long)(k - 1) * nlines];
                    vp = e.x; fp = e.y;
                }
            }
            ++k;
            stack[(long long)k * nlines] = make_int2(q, fq);
            vp = vk; fp = fk;
            vk = q; fk = fq;
        }
    }

    // phase 2: walk the envelope; entry j + 1 takes over from entry j once q passes their boundary.  Entry j + 2 is
    // loaded one advance ahead, so the walk does not wait on the stack.
    int j = 0;
    int2 cur = make_int2(0, kNoSite), nxt = make_int2(0, 0), nxt2 = make_int2(0, 0);
    if (k >= 0) cur = stack[0];
    if (k >= 1) nxt = stack[nlines];
    if (k >= 2) nxt2 = stack[2 * nlines];
    for (int q = 0; q < L.n; ++q) {
        int d = kNoSite;
        if (k >= 0) {
            while (j < k) {
                // boundary of cur and nxt: num / den < q  <=>  num < q den (den > 0)
                const long long num = (nxt.y + (long long)nxt.x * nxt.x) - (cur.y + (long long)cur.x * cur.x);
                const long long den = 2LL * (nxt.x - cur.x);
                if (num >= q * den) break;
                ++j;
                cur = nxt;
                nxt = nxt2;
                if (j + 2 <= k) nxt2 = stack[(long long)(j + 2) * nlines];
            }
            d = (q - cur.x) * (q - cur.x) + cur.y;
        }
        const long long s = L.base + q * L.stride;
        if (AXIS < 2) {
            buf[s] = d;
        } else if (d > 0) {
            // d == kNoSite: this sign's set is empty, the sentinel +-INT32_MAX / +-inf
            sd2[s] = sign ? -d : d;
            const float m = d == kNoSite ? INFINITY : __fmul_rn(voxel, __fsqrt_rn(__int2float_rn(d)));
            esdf[s] = sign ? -m : m;
        }
    }
}

__device__ __forceinline__ float lerp_rn(float a, float b, float t) { return __fadd_rn(a, __fmul_rn(t, __fsub_rn(b, a))); }

__global__ void __launch_bounds__(kNavThreads)
esdf_query_kernel(int nx, int ny, int nz, float ox, float oy, float oz, float voxel, const float* __restrict__ esdf,
                  int N, const float* __restrict__ points, float* __restrict__ dist, float* __restrict__ grad) {
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= N) return;
    const int dims[3] = {nx, ny, nz};
    const float org[3] = {ox, oy, oz};
    int idx[3];
    float t[3];
    bool inside = true;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        const float u = __fdiv_rn(__fsub_rn(points[3 * (long long)p + a], org[a]), voxel);
        inside = inside && isfinite(u) && u >= 0.f && u <= (float)(dims[a] - 1);
        const int i = inside ? min((int)floorf(u), dims[a] - 2) : 0;
        idx[a] = i;
        t[a] = __fsub_rn(u, (float)i);
    }
    if (!inside) {
        dist[p] = NAN;
        grad[3 * (long long)p] = NAN; grad[3 * (long long)p + 1] = NAN; grad[3 * (long long)p + 2] = NAN;
        return;
    }
    const long long sy = nx, sz = (long long)nx * ny;
    const long long s0 = idx[2] * sz + idx[1] * sy + idx[0];
    float c[8];    // c[dz * 4 + dy * 2 + dx]
#pragma unroll
    for (int q = 0; q < 8; ++q) c[q] = esdf[s0 + (q >> 2) * sz + (q >> 1 & 1) * sy + (q & 1)];
    float inf = 0.f;
#pragma unroll
    for (int q = 7; q >= 0; --q)
        if (isinf(c[q])) inf = c[q];                      // the first infinite corner in corner order
    float d, gx, gy, gz;
    if (inf != 0.f) {
        d = inf; gx = gy = gz = 0.f;
    } else {
        const float e00 = lerp_rn(c[0], c[1], t[0]), e01 = lerp_rn(c[2], c[3], t[0]);
        const float e10 = lerp_rn(c[4], c[5], t[0]), e11 = lerp_rn(c[6], c[7], t[0]);
        const float f0 = lerp_rn(e00, e01, t[1]), f1 = lerp_rn(e10, e11, t[1]);
        d = lerp_rn(f0, f1, t[2]);
        const float ax = lerp_rn(lerp_rn(__fsub_rn(c[1], c[0]), __fsub_rn(c[3], c[2]), t[1]),
                                 lerp_rn(__fsub_rn(c[5], c[4]), __fsub_rn(c[7], c[6]), t[1]), t[2]);
        const float ay = lerp_rn(__fsub_rn(e01, e00), __fsub_rn(e11, e10), t[2]);
        const float az = __fsub_rn(f1, f0);
        gx = __fdiv_rn(ax, voxel); gy = __fdiv_rn(ay, voxel); gz = __fdiv_rn(az, voxel);
    }
    dist[p] = d;
    grad[3 * (long long)p] = gx; grad[3 * (long long)p + 1] = gy; grad[3 * (long long)p + 2] = gz;
}

bool valid_nav_grid(int nx, int ny, int nz) {
    return nx >= 1 && ny >= 1 && nz >= 1 && nx <= kMaxDim && ny <= kMaxDim && nz <= kMaxDim &&
           (long long)nx * ny * nz < (1LL << 31);
}

struct EdtWs {
    int* A;        // [N] squared distance to O
    int* B;        // [N] squared distance to the complement of O
    int2* stacks;  // [2][N] envelope entries, line-fastest
};

EdtWs carve_edt(void* ws, long long n, size_t* total) {
    Carver cv(ws);
    EdtWs w;
    w.A = cv.take<int>(n);
    w.B = cv.take<int>(n);
    w.stacks = cv.take<int2>(2 * n);
    *total = cv.used();
    return w;
}

}  // namespace

}  // namespace sb

using namespace sb;

extern "C" {

SB_API int sb_nav_labels(int nx, int ny, int nz, const float* tsdf, const float* weight, float trunc, float min_weight,
                         float occ_dist, uint8_t* labels, void* stream) {
    if (!valid_nav_grid(nx, ny, nz) || !tsdf || !weight || !labels || !std::isfinite(trunc) || !(trunc > 0.f) ||
        !std::isfinite(min_weight) || !std::isfinite(occ_dist))
        return SB_ERR_BAD_ARG;
    const long long n = (long long)nx * ny * nz;
    nav_labels_kernel<<<blocks_of(n, kNavThreads), kNavThreads, 0, static_cast<cudaStream_t>(stream)>>>(
        n, tsdf, weight, trunc, min_weight, occ_dist, labels);
    SB_LAUNCH_CHECK("nav_labels_kernel");
    return SB_OK;
}

SB_API int sb_esdf_workspace_bytes(int nx, int ny, int nz, size_t* bytes) {
    if (!valid_nav_grid(nx, ny, nz) || !bytes) return SB_ERR_BAD_ARG;
    carve_edt(nullptr, (long long)nx * ny * nz, bytes);
    return SB_OK;
}

SB_API int sb_esdf(int nx, int ny, int nz, const uint8_t* labels, float voxel, int unknown_is_obstacle,
                   void* workspace, size_t workspace_bytes, int* sd2, float* esdf, void* stream) {
    if (!valid_nav_grid(nx, ny, nz) || !labels || !workspace || !sd2 || !esdf || !std::isfinite(voxel) ||
        !(voxel > 0.f) || (unknown_is_obstacle != 0 && unknown_is_obstacle != 1))
        return SB_ERR_BAD_ARG;
    const long long n = (long long)nx * ny * nz;
    size_t need = 0;
    carve_edt(nullptr, n, &need);
    if (workspace_bytes < need) return SB_ERR_WORKSPACE;
    EdtWs w = carve_edt(workspace, n, &need);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const long long lx = n / nx, ly = n / ny, lz = n / nz;
    edt_pass_kernel<0><<<dim3(blocks_of(lx, kEdtThreads), 2), kEdtThreads, 0, st>>>(
        nx, ny, nz, lx, labels, unknown_is_obstacle, w.A, w.B, w.stacks, voxel, sd2, esdf);
    SB_LAUNCH_CHECK("edt_pass_kernel<x>");
    edt_pass_kernel<1><<<dim3(blocks_of(ly, kEdtThreads), 2), kEdtThreads, 0, st>>>(
        nx, ny, nz, ly, labels, unknown_is_obstacle, w.A, w.B, w.stacks, voxel, sd2, esdf);
    SB_LAUNCH_CHECK("edt_pass_kernel<y>");
    edt_pass_kernel<2><<<dim3(blocks_of(lz, kEdtThreads), 2), kEdtThreads, 0, st>>>(
        nx, ny, nz, lz, labels, unknown_is_obstacle, w.A, w.B, w.stacks, voxel, sd2, esdf);
    SB_LAUNCH_CHECK("edt_pass_kernel<z>");
    return SB_OK;
}

SB_API int sb_esdf_query(int nx, int ny, int nz, float ox, float oy, float oz, float voxel, const float* esdf, int N,
                         const float* points, float* dist, float* grad, void* stream) {
    if (!valid_nav_grid(nx, ny, nz) || nx < 2 || ny < 2 || nz < 2 || !std::isfinite(ox) || !std::isfinite(oy) ||
        !std::isfinite(oz) || !std::isfinite(voxel) || !(voxel > 0.f) || N < 0 || !esdf ||
        (N > 0 && (!points || !dist || !grad)))
        return SB_ERR_BAD_ARG;
    if (N == 0) return SB_OK;
    esdf_query_kernel<<<blocks_of(N, kNavThreads), kNavThreads, 0, static_cast<cudaStream_t>(stream)>>>(
        nx, ny, nz, ox, oy, oz, voxel, esdf, N, points, dist, grad);
    SB_LAUNCH_CHECK("esdf_query_kernel");
    return SB_OK;
}

}  // extern "C"
