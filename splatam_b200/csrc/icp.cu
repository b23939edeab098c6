// icp.cu -- frame-to-model projective point-to-plane ICP, coarse to fine (splatam_b200/icp.py: align; the rule is
// restated in oracle/icp_numpy.py and stated in full in include/splatam_b200.h).
//
//   sb_icp_workspace_bytes  the three-level depth / vertex / normal pyramids, association codes, per-block partials
//                           and the pose state
//   sb_icp_align            every level, every iteration, on one stream; no host synchronisation (capturable)
//   sb_icp_export           copies one level's maps out of a workspace, for inspection
//
// Per-pixel maths is float32 with each operation rounded as written (__f*_rn: no contraction), so the maps and the
// association codes equal the numpy restatement bit for bit.  The normal equations are summed in double in a fixed
// order: each of kBlocks blocks reduces its grid-stride share of the pixels (thread registers, then warp shuffles,
// then warps in order), and the solve kernel sums the kBlocks partials of each term in block order.  The solve itself
// (Cholesky, exp map) runs in one thread in double.
#include <cmath>

#include "common.cuh"

namespace sb {

namespace {

constexpr int kLevels = SB_ICP_LEVELS;
constexpr int kStats = SB_ICP_STATS;
constexpr int kThreads = 256;
constexpr int kBlocks = 128;           // fixed, so the summation order does not depend on the device
constexpr int kTerms = 30;             // 21 JtJ (upper triangle, row-major), 6 Jtr, sum r^2, inliers, valid pixels
constexpr float kSilThres = 0.99f;     // model depth = depth_acc / sil where sil > kSilThres (mesh extraction's rule)
constexpr float kPyrBand = 0.05f;      // pyramid: samples within this depth [m] of the block minimum are averaged
constexpr float kNormalSlant = 5.f;    // a normal needs |dz| fx <= kNormalSlant z to each of its 4 neighbours: a
                                       // surface seen at up to 79 degrees from the view ray, the same at each level
constexpr float kDist0 = 0.1f;         // association distance [m] at level 0, doubling per level
constexpr double kMinCount = 32.0;     // fewer associated pixels: the update is skipped
constexpr double kMinInlierFrac = 0.4; // acceptance: inliers / valid data pixels of the last iteration
constexpr double kMaxRms = 0.03;       // acceptance: RMS point-to-plane residual [m] of the last iteration
constexpr double kMinPivotRatio = 1e-5;// acceptance: smallest / largest Cholesky pivot of the last system
constexpr int kRgbdStats = SB_RGBD_ICP_STATS;
constexpr int kPhotoTerms = 29;        // 21 JtJ_I, 6 Jtr_I, sum r_I^2, photometric pairs
constexpr float kMaxPhotoRes = SB_RGBD_ICP_MAX_RESIDUAL;      // |I_model - I_data| gate of a photometric pair
constexpr double kMaxPhotoRms = SB_RGBD_ICP_MAX_RMS;          // acceptance with weight > 0: photometric RMS
constexpr double kMinPhotoPairs = SB_RGBD_ICP_MIN_PAIRS;      // ... and at least this many photometric pairs

inline unsigned int blocks_for(long long n) { return (unsigned int)((n + kThreads - 1) / kThreads); }

struct Level {
    int H, W;
    float fx, fy, cx, cy;
    float* model_depth;   // [H W], 0 = invalid
    float* data_depth;    // [H W], 0 = invalid
    float* model_vertex;  // [3, H, W] planes x, y, z; 0 where invalid
    float* model_normal;  // [3, H, W]; 0 where invalid
    float* data_vertex;   // [3, H, W]
    uint8_t* assoc;       // [H W] 0 no data, 1 data not associated, 2 associated (latest iteration at this level)
};

struct IcpWs {
    Level lv[kLevels];
    double* partials;     // [kBlocks, kTerms]
    double* T;            // [12] row-major 3x4, camera t -> camera t-1
};

IcpWs carve_icp(Carver& c, int H, int W) {
    IcpWs w;
    for (int l = 0; l < kLevels; ++l) {
        Level& L = w.lv[l];
        L.H = H >> l;
        L.W = W >> l;
        const size_t n = (size_t)L.H * L.W;
        L.model_depth = c.take<float>(n);
        L.data_depth = c.take<float>(n);
        L.model_vertex = c.take<float>(3 * n);
        L.model_normal = c.take<float>(3 * n);
        L.data_vertex = c.take<float>(3 * n);
        L.assoc = c.take<uint8_t>(n);
    }
    w.partials = c.take<double>((size_t)kBlocks * kTerms);
    w.T = c.take<double>(12);
    return w;
}

IcpWs carve_icp(void* ws, int H, int W, size_t* total) {
    Carver c(ws);
    IcpWs w = carve_icp(c, H, W);
    if (total) *total = c.used();
    return w;
}

struct GreyLevel {
    float* model_grey;    // [H W], NaN where invalid (the model depth is invalid)
    float* data_grey;     // [H W], NaN where the data depth is invalid
    float* model_grad;    // [2, H, W] dI/du, dI/dv; NaN where invalid (the model normal is invalid)
    uint8_t* photo;       // [H W] 0 no geometric pair, 1 no photometric pair, 2 paired (latest iteration)
};

// sb_icp_align's workspace first (sb_icp_export reads it), then the grey pyramid and the photometric partials
struct RgbdWs {
    IcpWs g;
    GreyLevel lv[kLevels];
    double* photo_partials;   // [kBlocks, kPhotoTerms]
};

RgbdWs carve_rgbd(void* ws, int H, int W, size_t* total) {
    Carver c(ws);
    RgbdWs w;
    w.g = carve_icp(c, H, W);
    for (int l = 0; l < kLevels; ++l) {
        const size_t n = (size_t)(H >> l) * (W >> l);
        w.lv[l].model_grey = c.take<float>(n);
        w.lv[l].data_grey = c.take<float>(n);
        w.lv[l].model_grad = c.take<float>(2 * n);
        w.lv[l].photo = c.take<uint8_t>(n);
    }
    w.photo_partials = c.take<double>((size_t)kBlocks * kPhotoTerms);
    if (total) *total = c.used();
    return w;
}

bool valid_sizes(int H, int W) {
    return H >= (1 << (kLevels - 1)) && W >= (1 << (kLevels - 1)) && (long long)H * W < (1LL << 31);
}

__global__ void __launch_bounds__(kThreads)
icp_level0_kernel(int n, const float* __restrict__ depth_sil, const float* __restrict__ data,
                  float* __restrict__ model_depth, float* __restrict__ data_depth) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float sil = depth_sil[n + i];
    const float m = __fdiv_rn(depth_sil[i], sil);
    model_depth[i] = (sil > kSilThres && isfinite(m) && m > 0.f) ? m : 0.f;
    const float d = data[i];
    data_depth[i] = (isfinite(d) && d > 0.f) ? d : 0.f;
}

// 2x2 reduction of a level into the next: the mean, in sample order, of the block's valid samples within kPyrBand of
// the block's smallest valid depth.  kGrey: the mean of `grey` over exactly those samples instead (NaN if none)
template <bool kGrey>
__device__ __forceinline__ float reduce_block(const float* __restrict__ src, int Ws, int x, int y,
                                              const float* __restrict__ grey) {
    const float s[4] = {src[(size_t)(2 * y) * Ws + 2 * x], src[(size_t)(2 * y) * Ws + 2 * x + 1],
                        src[(size_t)(2 * y + 1) * Ws + 2 * x], src[(size_t)(2 * y + 1) * Ws + 2 * x + 1]};
    float m = INFINITY;
#pragma unroll
    for (int k = 0; k < 4; ++k)
        if (s[k] > 0.f) m = fminf(m, s[k]);
    float sum = 0.f;
    int cnt = 0;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const bool use = s[k] > 0.f && __fsub_rn(s[k], m) <= kPyrBand;
        if constexpr (kGrey)
            sum = __fadd_rn(sum, use ? grey[(size_t)(2 * y + (k >> 1)) * Ws + 2 * x + (k & 1)] : 0.f);
        else
            sum = __fadd_rn(sum, use ? s[k] : 0.f);
        cnt += use;
    }
    if constexpr (kGrey) return cnt ? __fdiv_rn(sum, (float)cnt) : NAN;
    return cnt ? __fdiv_rn(sum, (float)cnt) : 0.f;
}

__global__ void __launch_bounds__(kThreads)
icp_downsample_kernel(int Hd, int Wd, int Ws, const float* __restrict__ model_src, const float* __restrict__ data_src,
                      float* __restrict__ model_dst, float* __restrict__ data_dst) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= Hd * Wd) return;
    const int x = i % Wd, y = i / Wd;
    model_dst[i] = reduce_block<false>(model_src, Ws, x, y, nullptr);
    data_dst[i] = reduce_block<false>(data_src, Ws, x, y, nullptr);
}

__device__ __forceinline__ float3 backproject(float z, int u, int v, float fx, float fy, float cx, float cy) {
    if (!(z > 0.f)) return make_float3(0.f, 0.f, 0.f);
    return make_float3(__fmul_rn(__fdiv_rn(__fsub_rn((float)u, cx), fx), z),
                       __fmul_rn(__fdiv_rn(__fsub_rn((float)v, cy), fy), z), z);
}

__device__ __forceinline__ float3 sub3(float3 a, float3 b) {
    return make_float3(__fsub_rn(a.x, b.x), __fsub_rn(a.y, b.y), __fsub_rn(a.z, b.z));
}

__device__ __forceinline__ float3 cross3(float3 a, float3 b) {
    return make_float3(__fsub_rn(__fmul_rn(a.y, b.z), __fmul_rn(a.z, b.y)),
                       __fsub_rn(__fmul_rn(a.z, b.x), __fmul_rn(a.x, b.z)),
                       __fsub_rn(__fmul_rn(a.x, b.y), __fmul_rn(a.y, b.x)));
}

__device__ __forceinline__ float dot3(float3 a, float3 b) {
    return __fadd_rn(__fadd_rn(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)), __fmul_rn(a.z, b.z));
}

// model vertex and normal maps and the data vertex map of one level
__global__ void __launch_bounds__(kThreads)
icp_maps_kernel(Level L) {
    const int n = L.H * L.W;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int u = i % L.W, v = i / L.W;
    const float3 dv = backproject(L.data_depth[i], u, v, L.fx, L.fy, L.cx, L.cy);
    L.data_vertex[i] = dv.x; L.data_vertex[n + i] = dv.y; L.data_vertex[2 * n + i] = dv.z;
    const float z = L.model_depth[i];
    const float3 mv = backproject(z, u, v, L.fx, L.fy, L.cx, L.cy);
    L.model_vertex[i] = mv.x; L.model_vertex[n + i] = mv.y; L.model_vertex[2 * n + i] = mv.z;
    float3 nrm = make_float3(0.f, 0.f, 0.f);
    if (z > 0.f && u >= 1 && u + 1 < L.W && v >= 1 && v + 1 < L.H) {
        const float zl = L.model_depth[i - 1], zr = L.model_depth[i + 1];
        const float zu = L.model_depth[i - L.W], zd = L.model_depth[i + L.W];
        const float lim = __fmul_rn(kNormalSlant, z);
        const bool ok = zl > 0.f && zr > 0.f && zu > 0.f && zd > 0.f &&
                        __fmul_rn(fabsf(__fsub_rn(zl, z)), L.fx) <= lim &&
                        __fmul_rn(fabsf(__fsub_rn(zr, z)), L.fx) <= lim &&
                        __fmul_rn(fabsf(__fsub_rn(zu, z)), L.fx) <= lim &&
                        __fmul_rn(fabsf(__fsub_rn(zd, z)), L.fx) <= lim;
        if (ok) {
            const float3 dx = sub3(backproject(zr, u + 1, v, L.fx, L.fy, L.cx, L.cy),
                                   backproject(zl, u - 1, v, L.fx, L.fy, L.cx, L.cy));
            const float3 dy = sub3(backproject(zd, u, v + 1, L.fx, L.fy, L.cx, L.cy),
                                   backproject(zu, u, v - 1, L.fx, L.fy, L.cx, L.cy));
            const float3 c = cross3(dx, dy);
            const float len = __fsqrt_rn(dot3(c, c));
            if (len > 0.f && isfinite(len))
                nrm = make_float3(__fdiv_rn(c.x, len), __fdiv_rn(c.y, len), __fdiv_rn(c.z, len));
        }
    }
    L.model_normal[i] = nrm.x; L.model_normal[n + i] = nrm.y; L.model_normal[2 * n + i] = nrm.z;
}

// 3x4 rigid transforms in double, row-major [R | t]
__device__ void rigid_inverse(const double* a, double* o) {
    for (int r = 0; r < 3; ++r) {
        for (int c = 0; c < 3; ++c) o[4 * r + c] = a[4 * c + r];
        o[4 * r + 3] = -(a[r] * a[3] + a[4 + r] * a[7] + a[8 + r] * a[11]);
    }
}

__device__ void compose(const double* a, const double* b, double* o) {   // o = a b
    for (int r = 0; r < 3; ++r) {
        for (int c = 0; c < 4; ++c) {
            double s = a[4 * r] * b[c] + a[4 * r + 1] * b[4 + c] + a[4 * r + 2] * b[8 + c];
            o[4 * r + c] = c == 3 ? s + a[4 * r + 3] : s;
        }
    }
}

// T = w2c_prev inv(w2c_init); the stats record starts at zero
__global__ void icp_init_kernel(const float* __restrict__ w2c_prev, const float* __restrict__ w2c_init,
                                double* __restrict__ T, double* __restrict__ stats) {
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    double a[12], b[12], bi[12];
    for (int k = 0; k < 12; ++k) { a[k] = (double)w2c_prev[k]; b[k] = (double)w2c_init[k]; }
    rigid_inverse(b, bi);
    compose(a, bi, T);
    for (int k = 0; k < kStats; ++k) stats[k] = 0.0;
}

// the geometric pair of a valid data vertex v (rule 4 of the header): true if paired, with p = R v + t, the model
// normal nm at the pair and d = p - q
__device__ __forceinline__ bool geo_pair(const Level L, const float (&R)[12], float dist2, float3 v, int n, float3& p,
                                         float3& nm, float3& d) {
    p = make_float3(__fadd_rn(dot3(make_float3(R[0], R[1], R[2]), v), R[3]),
                    __fadd_rn(dot3(make_float3(R[4], R[5], R[6]), v), R[7]),
                    __fadd_rn(dot3(make_float3(R[8], R[9], R[10]), v), R[11]));
    if (p.z > 0.f) {
        const float uf = floorf(__fadd_rn(__fadd_rn(__fdiv_rn(__fmul_rn(L.fx, p.x), p.z), L.cx), 0.5f));
        const float vf = floorf(__fadd_rn(__fadd_rn(__fdiv_rn(__fmul_rn(L.fy, p.y), p.z), L.cy), 0.5f));
        if (uf >= 0.f && uf < (float)L.W && vf >= 0.f && vf < (float)L.H) {
            const int j = (int)vf * L.W + (int)uf;
            const float3 q = make_float3(L.model_vertex[j], L.model_vertex[n + j], L.model_vertex[2 * n + j]);
            nm = make_float3(L.model_normal[j], L.model_normal[n + j], L.model_normal[2 * n + j]);
            d = sub3(p, q);
            if (q.z > 0.f && (nm.x != 0.f || nm.y != 0.f || nm.z != 0.f) && dot3(d, d) <= dist2) return true;
        }
    }
    return false;
}

// a paired pixel's point-to-plane terms: r = n.(p - q), J = [p x n, n] into acc[0..29) (kTerms' layout)
__device__ __forceinline__ void geo_accumulate(double* acc, float3 p, float3 nm, float3 d) {
    const float r = dot3(nm, d);
    const float3 pn = cross3(p, nm);
    const double J[6] = {pn.x, pn.y, pn.z, nm.x, nm.y, nm.z};
    int k = 0;
#pragma unroll
    for (int a = 0; a < 6; ++a)
#pragma unroll
        for (int b = a; b < 6; ++b) acc[k++] += J[a] * J[b];
#pragma unroll
    for (int a = 0; a < 6; ++a) acc[21 + a] += J[a] * (double)r;
    acc[27] += (double)r * (double)r;
    acc[28] += 1.0;
}

__global__ void __launch_bounds__(kThreads)
icp_associate_kernel(Level L, float dist2, const double* __restrict__ T, double* __restrict__ partials) {
    __shared__ double red[kThreads / 32][kTerms];
    float R[12];
#pragma unroll
    for (int k = 0; k < 12; ++k) R[k] = __double2float_rn(T[k]);
    const int n = L.H * L.W;
    double acc[kTerms];
#pragma unroll
    for (int k = 0; k < kTerms; ++k) acc[k] = 0.0;
    for (int i = blockIdx.x * kThreads + threadIdx.x; i < n; i += kBlocks * kThreads) {
        const float3 v = make_float3(L.data_vertex[i], L.data_vertex[n + i], L.data_vertex[2 * n + i]);
        uint8_t code = 0;
        if (v.z > 0.f) {
            code = 1;
            acc[29] += 1.0;
            float3 p, nm, d;
            if (geo_pair(L, R, dist2, v, n, p, nm, d)) {
                code = 2;
                geo_accumulate(acc, p, nm, d);
            }
        }
        L.assoc[i] = code;
    }
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int k = 0; k < kTerms; ++k) {
        double s = acc[k];
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) s += __shfl_xor_sync(0xffffffffu, s, off);
        if (lane == 0) red[warp][k] = s;
    }
    __syncthreads();
    if (threadIdx.x < kTerms) {
        double s = 0.0;
        for (int w = 0; w < kThreads / 32; ++w) s += red[w][threadIdx.x];
        partials[(size_t)blockIdx.x * kTerms + threadIdx.x] = s;
    }
}

// sum the partials (thread k: term k, blocks in order), then thread 0 solves JtJ xi = -Jtr by Cholesky and applies
// T <- exp(xi) T; the latest system goes to the stats record.  kJoint (sb_rgbd_icp_align): threads 32.. also sum the
// photometric partials, which go to stats[36..66), and the system solved is JtJ + lam2 JtJ_I, Jtr + lam2 Jtr_I
template <bool kJoint>
__global__ void icp_solve_kernel(const double* __restrict__ partials, double* __restrict__ T,
                                 double* __restrict__ stats, const double* __restrict__ photo_partials, double lam2) {
    __shared__ double s[kJoint ? 32 + kPhotoTerms : kTerms];
    if (threadIdx.x < kTerms) {
        double a = 0.0;
        for (int b = 0; b < kBlocks; ++b) a += partials[(size_t)b * kTerms + threadIdx.x];
        s[threadIdx.x] = a;
    }
    if constexpr (kJoint) {
        if (threadIdx.x >= 32 && threadIdx.x < 32 + kPhotoTerms) {
            double a = 0.0;
            for (int b = 0; b < kBlocks; ++b) a += photo_partials[(size_t)b * kPhotoTerms + threadIdx.x - 32];
            s[threadIdx.x] = a;
        }
    }
    __syncthreads();
    if (threadIdx.x != 0) return;
    if constexpr (kJoint) {
        const double* ph = s + 32;               // 21 JtJ_I, 6 Jtr_I, sum r_I^2, photometric pairs
        stats[36] = ph[28];
        stats[37] = ph[28] > 0.0 ? sqrt(ph[27] / ph[28]) : INFINITY;
        for (int k = 0; k < 28; ++k) stats[38 + k] = ph[k];
        for (int k = 0; k < 27; ++k) s[k] += lam2 * ph[k];
    }
    double A[6][6], L[6][6], y[6], xi[6];
    int k = 0;
    for (int a = 0; a < 6; ++a)
        for (int b = a; b < 6; ++b) { A[a][b] = A[b][a] = s[k]; stats[8 + k] = s[k]; ++k; }
    for (int a = 0; a < 6; ++a) stats[29 + a] = s[21 + a];
    stats[35] = s[27];
    stats[3] = s[28];
    stats[4] = s[29];
    bool ok = s[28] >= kMinCount;
    double pmin = INFINITY, pmax = 0.0;
    for (int j = 0; j < 6 && ok; ++j) {
        double d = A[j][j];
        for (int q = 0; q < j; ++q) d -= L[j][q] * L[j][q];
        if (!(d > 0.0) || !isfinite(d)) { ok = false; break; }
        pmin = fmin(pmin, d);
        pmax = fmax(pmax, d);
        L[j][j] = sqrt(d);
        for (int i = j + 1; i < 6; ++i) {
            double e = A[i][j];
            for (int q = 0; q < j; ++q) e -= L[i][q] * L[j][q];
            L[i][j] = e / L[j][j];
        }
    }
    stats[5] = ok ? pmin / pmax : 0.0;
    if (ok) {
        for (int i = 0; i < 6; ++i) {            // L y = -g
            double e = -s[21 + i];
            for (int q = 0; q < i; ++q) e -= L[i][q] * y[q];
            y[i] = e / L[i][i];
        }
        for (int i = 5; i >= 0; --i) {           // L^T xi = y
            double e = y[i];
            for (int q = i + 1; q < 6; ++q) e -= L[q][i] * xi[q];
            xi[i] = e / L[i][i];
        }
        for (int i = 0; i < 6; ++i) ok = ok && isfinite(xi[i]);
    }
    if (!ok) {
        stats[6] = 1.0;                          // some update was skipped
        stats[7] = 1.0;                          // ... the latest one
        return;
    }
    stats[7] = 0.0;
    // exp map of xi = (w, v): R = I + A W + B W^2, V = I + B W + C W^2, t = V v
    const double w0 = xi[0], w1 = xi[1], w2 = xi[2];
    const double th2 = w0 * w0 + w1 * w1 + w2 * w2, th = sqrt(th2);
    double cA, cB, cC;
    if (th < 1e-6) {
        cA = 1.0 - th2 / 6.0; cB = 0.5 - th2 / 24.0; cC = 1.0 / 6.0 - th2 / 120.0;
    } else {
        cA = sin(th) / th; cB = (1.0 - cos(th)) / th2; cC = (th - sin(th)) / (th2 * th);
    }
    const double W[3][3] = {{0.0, -w2, w1}, {w2, 0.0, -w0}, {-w1, w0, 0.0}};
    double W2[3][3];
    for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c) W2[r][c] = W[r][0] * W[0][c] + W[r][1] * W[1][c] + W[r][2] * W[2][c];
    double E[12];
    for (int r = 0; r < 3; ++r) {
        double tv = 0.0;
        for (int c = 0; c < 3; ++c) {
            const double I = r == c ? 1.0 : 0.0;
            E[4 * r + c] = I + cA * W[r][c] + cB * W2[r][c];
            tv += (I + cB * W[r][c] + cC * W2[r][c]) * xi[3 + c];
        }
        E[4 * r + 3] = tv;
    }
    double Tn[12];
    compose(E, T, Tn);
    for (int q = 0; q < 12; ++q) T[q] = Tn[q];
}

// acceptance (rule 5, and `extra`) and the chosen pose: w2c_out = inv(T) w2c_prev if accepted, else w2c_init
__device__ __forceinline__ void select_pose(const double* __restrict__ T, const float* __restrict__ w2c_prev,
                                            const float* __restrict__ w2c_init, float* __restrict__ w2c_out,
                                            double* __restrict__ stats, bool extra) {
    const double inl = stats[3], valid = stats[4];
    const double frac = valid > 0.0 ? inl / valid : 0.0;
    const double rms = inl > 0.0 ? sqrt(stats[35] / inl) : INFINITY;
    const bool acc = valid > 0.0 && frac >= kMinInlierFrac && rms <= kMaxRms && stats[5] >= kMinPivotRatio &&
                     stats[7] == 0.0 && extra;
    stats[0] = acc ? 1.0 : 0.0;
    stats[1] = frac;
    stats[2] = rms;
    if (!acc) {
        for (int k = 0; k < 16; ++k) w2c_out[k] = w2c_init[k];
        return;
    }
    double Ti[12], P[12], O[12];
    rigid_inverse(T, Ti);
    for (int k = 0; k < 12; ++k) P[k] = (double)w2c_prev[k];
    compose(Ti, P, O);
    for (int k = 0; k < 12; ++k) w2c_out[k] = (float)O[k];
    w2c_out[12] = 0.f; w2c_out[13] = 0.f; w2c_out[14] = 0.f; w2c_out[15] = 1.f;
}

__global__ void icp_select_kernel(const double* __restrict__ T, const float* __restrict__ w2c_prev,
                                  const float* __restrict__ w2c_init, float* __restrict__ w2c_out,
                                  double* __restrict__ stats) {
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    select_pose(T, w2c_prev, w2c_init, w2c_out, stats, true);
}

// ---- RGB-D ICP (sb_rgbd_icp_align): the grey pyramid, the model gradient and the fused association ----------------

// level 0 grey where the level-0 depth is valid (rule a), NaN elsewhere
__global__ void __launch_bounds__(kThreads)
rgbd_grey0_kernel(int n, const float* __restrict__ model_rgb, const float* __restrict__ data_rgb,
                  const float* __restrict__ model_depth, const float* __restrict__ data_depth,
                  float* __restrict__ model_grey, float* __restrict__ data_grey) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    model_grey[i] = model_depth[i] > 0.f ? grey_of(model_rgb, n, i) : NAN;
    data_grey[i] = data_depth[i] > 0.f ? grey_of(data_rgb, n, i) : NAN;
}

__global__ void __launch_bounds__(kThreads)
rgbd_grey_downsample_kernel(int Hd, int Wd, int Ws, const float* __restrict__ model_depth,
                            const float* __restrict__ data_depth, const float* __restrict__ model_src,
                            const float* __restrict__ data_src, float* __restrict__ model_dst,
                            float* __restrict__ data_dst) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= Hd * Wd) return;
    const int x = i % Wd, y = i / Wd;
    model_dst[i] = reduce_block<true>(model_depth, Ws, x, y, model_src);
    data_dst[i] = reduce_block<true>(data_depth, Ws, x, y, data_src);
}

// central differences of the model grey where the model normal is valid (rule c)
__global__ void __launch_bounds__(kThreads)
rgbd_gradient_kernel(Level L, GreyLevel G) {
    const int n = L.H * L.W;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    float gu = NAN, gv = NAN;
    if (L.model_normal[i] != 0.f || L.model_normal[n + i] != 0.f || L.model_normal[2 * n + i] != 0.f) {
        gu = __fmul_rn(__fsub_rn(G.model_grey[i + 1], G.model_grey[i - 1]), 0.5f);
        gv = __fmul_rn(__fsub_rn(G.model_grey[i + L.W], G.model_grey[i - L.W]), 0.5f);
    }
    G.model_grad[i] = gu;
    G.model_grad[n + i] = gv;
}

// the photometric pair of a data pixel whose geometric pair is p (rule d): true with r_I and J_I
__device__ __forceinline__ bool photo_pair(const Level& L, const GreyLevel& G, int n, float3 p, float data_grey,
                                           float& r, float (&J)[6]) {
    const float uc = __fadd_rn(__fdiv_rn(__fmul_rn(L.fx, p.x), p.z), L.cx);
    const float vc = __fadd_rn(__fdiv_rn(__fmul_rn(L.fy, p.y), p.z), L.cy);
    const float u0 = floorf(uc), v0 = floorf(vc);
    if (!(u0 >= 0.f && __fadd_rn(u0, 1.f) < (float)L.W && v0 >= 0.f && __fadd_rn(v0, 1.f) < (float)L.H)) return false;
    const float a = __fsub_rn(uc, u0), b = __fsub_rn(vc, v0);
    const float a1 = __fsub_rn(1.f, a), b1 = __fsub_rn(1.f, b);
    const float w[4] = {__fmul_rn(a1, b1), __fmul_rn(a, b1), __fmul_rn(a1, b), __fmul_rn(a, b)};
    const int j0 = (int)v0 * L.W + (int)u0;
    const int tap[4] = {j0, j0 + 1, j0 + L.W, j0 + L.W + 1};
    float I = 0.f, gu = 0.f, gv = 0.f;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const float ik = G.model_grey[tap[k]], uk = G.model_grad[tap[k]], vk = G.model_grad[n + tap[k]];
        if (!(isfinite(ik) && isfinite(uk) && isfinite(vk))) return false;
        I = __fadd_rn(I, __fmul_rn(w[k], ik));
        gu = __fadd_rn(gu, __fmul_rn(w[k], uk));
        gv = __fadd_rn(gv, __fmul_rn(w[k], vk));
    }
    r = __fsub_rn(I, data_grey);
    if (!(fabsf(r) <= kMaxPhotoRes)) return false;
    const float g0 = __fdiv_rn(__fmul_rn(gu, L.fx), p.z), g1 = __fdiv_rn(__fmul_rn(gv, L.fy), p.z);
    const float g2 = -__fdiv_rn(__fadd_rn(__fmul_rn(g0, p.x), __fmul_rn(g1, p.y)), p.z);
    const float3 g = make_float3(g0, g1, g2);
    const float3 pg = cross3(p, g);
    J[0] = pg.x; J[1] = pg.y; J[2] = pg.z; J[3] = g0; J[4] = g1; J[5] = g2;
    bool ok = true;
#pragma unroll
    for (int k = 0; k < 6; ++k) ok = ok && isfinite(J[k]);
    return ok;
}

// icp_associate_kernel's geometric pass with the photometric term fused in: the geometric partials in kTerms' layout
// (summed exactly as icp_associate_kernel sums them), the photometric ones in kPhotoTerms' layout
__global__ void __launch_bounds__(kThreads)
rgbd_associate_kernel(Level L, GreyLevel G, float dist2, const double* __restrict__ T, double* __restrict__ partials,
                      double* __restrict__ photo_partials) {
    constexpr int kAll = kTerms + kPhotoTerms;
    __shared__ double red[kThreads / 32][kAll];
    float R[12];
#pragma unroll
    for (int k = 0; k < 12; ++k) R[k] = __double2float_rn(T[k]);
    const int n = L.H * L.W;
    double acc[kAll];
#pragma unroll
    for (int k = 0; k < kAll; ++k) acc[k] = 0.0;
    for (int i = blockIdx.x * kThreads + threadIdx.x; i < n; i += kBlocks * kThreads) {
        const float3 v = make_float3(L.data_vertex[i], L.data_vertex[n + i], L.data_vertex[2 * n + i]);
        uint8_t code = 0, photo = 0;
        if (v.z > 0.f) {
            code = 1;
            acc[29] += 1.0;
            float3 p, nm, d;
            if (geo_pair(L, R, dist2, v, n, p, nm, d)) {
                code = 2;
                photo = 1;
                geo_accumulate(acc, p, nm, d);
                float r, J[6];
                if (photo_pair(L, G, n, p, G.data_grey[i], r, J)) {
                    photo = 2;
                    double* ph = acc + kTerms;
                    int k = 0;
#pragma unroll
                    for (int a = 0; a < 6; ++a)
#pragma unroll
                        for (int b = a; b < 6; ++b) ph[k++] += (double)J[a] * (double)J[b];
#pragma unroll
                    for (int a = 0; a < 6; ++a) ph[21 + a] += (double)J[a] * (double)r;
                    ph[27] += (double)r * (double)r;
                    ph[28] += 1.0;
                }
            }
        }
        L.assoc[i] = code;
        G.photo[i] = photo;
    }
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int k = 0; k < kAll; ++k) {
        double s = acc[k];
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) s += __shfl_xor_sync(0xffffffffu, s, off);
        if (lane == 0) red[warp][k] = s;
    }
    __syncthreads();
    if (threadIdx.x < kAll) {
        double s = 0.0;
        for (int w = 0; w < kThreads / 32; ++w) s += red[w][threadIdx.x];
        if (threadIdx.x < kTerms)
            partials[(size_t)blockIdx.x * kTerms + threadIdx.x] = s;
        else
            photo_partials[(size_t)blockIdx.x * kPhotoTerms + threadIdx.x - kTerms] = s;
    }
}

// rule f on top of rule 5
__global__ void rgbd_select_kernel(const double* __restrict__ T, const float* __restrict__ w2c_prev,
                                   const float* __restrict__ w2c_init, float* __restrict__ w2c_out,
                                   double* __restrict__ stats, float weight) {
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    const bool photo_ok = weight == 0.f || (stats[36] >= kMinPhotoPairs && stats[37] <= kMaxPhotoRms);
    select_pose(T, w2c_prev, w2c_init, w2c_out, stats, photo_ok);
}

void level_intrinsics(IcpWs& w, float fx, float fy, float cx, float cy) {
    for (int l = 0; l < kLevels; ++l) {
        Level& L = w.lv[l];
        L.fx = fx; L.fy = fy; L.cx = cx; L.cy = cy;
        // a coarse pixel's centre is the mean of its block's centres: u_{l+1} = (u_l - 0.5) / 2
        fx = fx * 0.5f; fy = fy * 0.5f; cx = (cx - 0.5f) * 0.5f; cy = (cy - 0.5f) * 0.5f;
    }
}

bool valid_camera(float fx, float fy, float cx, float cy) {
    return std::isfinite(fx) && fx > 0.f && std::isfinite(fy) && fy > 0.f && std::isfinite(cx) && std::isfinite(cy);
}

bool valid_iters(const int* iters) {
    for (int l = 0; l < kLevels; ++l)
        if (iters[l] < 0 || iters[l] > 1000) return false;
    return true;
}

// steps 1-3 of sb_icp_align: the depth pyramid and the vertex and normal maps of every level
int launch_maps(IcpWs& w, int height, int width, const float* model_depth_sil, const float* data_depth,
                cudaStream_t st) {
    const int n0 = height * width;
    icp_level0_kernel<<<blocks_for(n0), kThreads, 0, st>>>(n0, model_depth_sil, data_depth, w.lv[0].model_depth,
                                                           w.lv[0].data_depth);
    SB_LAUNCH_CHECK("icp_level0_kernel");
    for (int l = 1; l < kLevels; ++l) {
        const Level &S = w.lv[l - 1], &D = w.lv[l];
        icp_downsample_kernel<<<blocks_for((long long)D.H * D.W), kThreads, 0, st>>>(
            D.H, D.W, S.W, S.model_depth, S.data_depth, D.model_depth, D.data_depth);
        SB_LAUNCH_CHECK("icp_downsample_kernel");
    }
    for (int l = 0; l < kLevels; ++l) {
        icp_maps_kernel<<<blocks_for((long long)w.lv[l].H * w.lv[l].W), kThreads, 0, st>>>(w.lv[l]);
        SB_LAUNCH_CHECK("icp_maps_kernel");
    }
    return SB_OK;
}

}  // namespace

}  // namespace sb

using namespace sb;

extern "C" {

SB_API int sb_icp_workspace_bytes(int height, int width, size_t* bytes) {
    if (!valid_sizes(height, width) || !bytes) return SB_ERR_BAD_ARG;
    carve_icp(nullptr, height, width, bytes);
    return SB_OK;
}

SB_API int sb_icp_align(int height, int width, const float* model_depth_sil, const float* data_depth, float fx,
                        float fy, float cx, float cy, const float* w2c_prev, const float* w2c_init, const int* iters,
                        void* workspace, size_t workspace_bytes, float* w2c_out, double* stats, void* stream) {
    if (!valid_sizes(height, width) || !model_depth_sil || !data_depth || !w2c_prev || !w2c_init || !iters ||
        !workspace || !w2c_out || !stats || !valid_camera(fx, fy, cx, cy) || !valid_iters(iters))
        return SB_ERR_BAD_ARG;
    size_t need = 0;
    carve_icp(nullptr, height, width, &need);
    if (workspace_bytes < need) return SB_ERR_WORKSPACE;
    IcpWs w = carve_icp(workspace, height, width, &need);
    level_intrinsics(w, fx, fy, cx, cy);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int rc = launch_maps(w, height, width, model_depth_sil, data_depth, st);
    if (rc != SB_OK) return rc;
    icp_init_kernel<<<1, 1, 0, st>>>(w2c_prev, w2c_init, w.T, stats);
    SB_LAUNCH_CHECK("icp_init_kernel");
    for (int l = kLevels - 1; l >= 0; --l) {
        const float d = kDist0 * (float)(1 << l);
        for (int it = 0; it < iters[l]; ++it) {
            icp_associate_kernel<<<kBlocks, kThreads, 0, st>>>(w.lv[l], d * d, w.T, w.partials);
            SB_LAUNCH_CHECK("icp_associate_kernel");
            icp_solve_kernel<false><<<1, 32, 0, st>>>(w.partials, w.T, stats, nullptr, 0.0);
            SB_LAUNCH_CHECK("icp_solve_kernel");
        }
    }
    icp_select_kernel<<<1, 1, 0, st>>>(w.T, w2c_prev, w2c_init, w2c_out, stats);
    SB_LAUNCH_CHECK("icp_select_kernel");
    return SB_OK;
}

SB_API int sb_rgbd_icp_workspace_bytes(int height, int width, size_t* bytes) {
    if (!valid_sizes(height, width) || !bytes) return SB_ERR_BAD_ARG;
    carve_rgbd(nullptr, height, width, bytes);
    return SB_OK;
}

SB_API int sb_rgbd_icp_align(int height, int width, const float* model_depth_sil, const float* model_rgb,
                             const float* data_depth, const float* data_rgb, float fx, float fy, float cx, float cy,
                             const float* w2c_prev, const float* w2c_init, const int* iters, float weight,
                             void* workspace, size_t workspace_bytes, float* w2c_out, double* stats, void* stream) {
    if (!valid_sizes(height, width) || !model_depth_sil || !model_rgb || !data_depth || !data_rgb || !w2c_prev ||
        !w2c_init || !iters || !workspace || !w2c_out || !stats || !valid_camera(fx, fy, cx, cy) ||
        !valid_iters(iters) || !(std::isfinite(weight) && weight >= 0.f))
        return SB_ERR_BAD_ARG;
    size_t need = 0;
    carve_rgbd(nullptr, height, width, &need);
    if (workspace_bytes < need) return SB_ERR_WORKSPACE;
    RgbdWs w = carve_rgbd(workspace, height, width, &need);
    level_intrinsics(w.g, fx, fy, cx, cy);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int rc = launch_maps(w.g, height, width, model_depth_sil, data_depth, st);
    if (rc != SB_OK) return rc;
    const int n0 = height * width;
    rgbd_grey0_kernel<<<blocks_for(n0), kThreads, 0, st>>>(n0, model_rgb, data_rgb, w.g.lv[0].model_depth,
                                                           w.g.lv[0].data_depth, w.lv[0].model_grey,
                                                           w.lv[0].data_grey);
    SB_LAUNCH_CHECK("rgbd_grey0_kernel");
    for (int l = 1; l < kLevels; ++l) {
        const Level &S = w.g.lv[l - 1], &D = w.g.lv[l];
        rgbd_grey_downsample_kernel<<<blocks_for((long long)D.H * D.W), kThreads, 0, st>>>(
            D.H, D.W, S.W, S.model_depth, S.data_depth, w.lv[l - 1].model_grey, w.lv[l - 1].data_grey,
            w.lv[l].model_grey, w.lv[l].data_grey);
        SB_LAUNCH_CHECK("rgbd_grey_downsample_kernel");
    }
    for (int l = 0; l < kLevels; ++l) {
        rgbd_gradient_kernel<<<blocks_for((long long)w.g.lv[l].H * w.g.lv[l].W), kThreads, 0, st>>>(w.g.lv[l],
                                                                                                     w.lv[l]);
        SB_LAUNCH_CHECK("rgbd_gradient_kernel");
    }
    icp_init_kernel<<<1, 1, 0, st>>>(w2c_prev, w2c_init, w.g.T, stats);
    SB_LAUNCH_CHECK("icp_init_kernel");
    SB_CUDA_CHECK(cudaMemsetAsync(stats + kStats, 0, (kRgbdStats - kStats) * sizeof(double), st));
    const double lam2 = (double)weight * (double)weight;
    for (int l = kLevels - 1; l >= 0; --l) {
        const float d = kDist0 * (float)(1 << l);
        for (int it = 0; it < iters[l]; ++it) {
            rgbd_associate_kernel<<<kBlocks, kThreads, 0, st>>>(w.g.lv[l], w.lv[l], d * d, w.g.T, w.g.partials,
                                                                w.photo_partials);
            SB_LAUNCH_CHECK("rgbd_associate_kernel");
            icp_solve_kernel<true><<<1, 64, 0, st>>>(w.g.partials, w.g.T, stats, w.photo_partials, lam2);
            SB_LAUNCH_CHECK("icp_solve_kernel");
        }
    }
    rgbd_select_kernel<<<1, 1, 0, st>>>(w.g.T, w2c_prev, w2c_init, w2c_out, stats, weight);
    SB_LAUNCH_CHECK("rgbd_select_kernel");
    return SB_OK;
}

SB_API int sb_rgbd_icp_export(int height, int width, const void* workspace, size_t workspace_bytes, int level,
                              float* model_grey, float* data_grey, float* model_grad, uint8_t* photo, void* stream) {
    if (!valid_sizes(height, width) || !workspace || level < 0 || level >= kLevels || !model_grey || !data_grey ||
        !model_grad || !photo)
        return SB_ERR_BAD_ARG;
    size_t need = 0;
    carve_rgbd(nullptr, height, width, &need);
    if (workspace_bytes < need) return SB_ERR_WORKSPACE;
    RgbdWs w = carve_rgbd(const_cast<void*>(workspace), height, width, &need);
    const GreyLevel& G = w.lv[level];
    const size_t n = (size_t)(height >> level) * (width >> level);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const cudaMemcpyKind k = cudaMemcpyDeviceToDevice;
    SB_CUDA_CHECK(cudaMemcpyAsync(model_grey, G.model_grey, n * sizeof(float), k, st));
    SB_CUDA_CHECK(cudaMemcpyAsync(data_grey, G.data_grey, n * sizeof(float), k, st));
    SB_CUDA_CHECK(cudaMemcpyAsync(model_grad, G.model_grad, 2 * n * sizeof(float), k, st));
    SB_CUDA_CHECK(cudaMemcpyAsync(photo, G.photo, n, k, st));
    return SB_OK;
}

SB_API int sb_icp_export(int height, int width, const void* workspace, size_t workspace_bytes, int level,
                         float* model_depth, float* data_depth, float* model_vertex, float* model_normal,
                         float* data_vertex, uint8_t* assoc, void* stream) {
    if (!valid_sizes(height, width) || !workspace || level < 0 || level >= kLevels || !model_depth || !data_depth ||
        !model_vertex || !model_normal || !data_vertex || !assoc)
        return SB_ERR_BAD_ARG;
    size_t need = 0;
    carve_icp(nullptr, height, width, &need);
    if (workspace_bytes < need) return SB_ERR_WORKSPACE;
    IcpWs w = carve_icp(const_cast<void*>(workspace), height, width, &need);
    const Level& L = w.lv[level];
    const size_t n = (size_t)L.H * L.W;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const cudaMemcpyKind k = cudaMemcpyDeviceToDevice;
    SB_CUDA_CHECK(cudaMemcpyAsync(model_depth, L.model_depth, n * sizeof(float), k, st));
    SB_CUDA_CHECK(cudaMemcpyAsync(data_depth, L.data_depth, n * sizeof(float), k, st));
    SB_CUDA_CHECK(cudaMemcpyAsync(model_vertex, L.model_vertex, 3 * n * sizeof(float), k, st));
    SB_CUDA_CHECK(cudaMemcpyAsync(model_normal, L.model_normal, 3 * n * sizeof(float), k, st));
    SB_CUDA_CHECK(cudaMemcpyAsync(data_vertex, L.data_vertex, 3 * n * sizeof(float), k, st));
    SB_CUDA_CHECK(cudaMemcpyAsync(assoc, L.assoc, n, k, st));
    return SB_OK;
}

}  // extern "C"
