// loop.cu -- loop closure: map deformation and the keyframe pose graph (splatam_b200/loop.py; the rules are stated in
// include/splatam_b200.h and restated in oracle/loop_numpy.py).
//
//   sb_deform_gaussians              one thread per Gaussian: mean and unnormalised quaternion moved by the correction
//                                    of the Gaussian's creation frame, float32 with every operation rounded as written
//   sb_pose_graph_normal_equations   per-edge residuals and 6x6 Jacobian blocks (one thread per edge), then the dense
//                                    H and b assembled by one block in edge order (the same bits on every call)
//   sb_pose_graph_update             one block: T <- exp(xi) T for every free node, the residual test of every edge,
//                                    the per-frame correction table and the accept flag
//
// Poses are w2c rigid transforms stored as double [12], row-major 3x4.  A tangent vector is (phi, rho): rotation
// first, as in csrc/icp.cu.
#include <cmath>

#include "common.cuh"

namespace sb {

namespace {

constexpr int kThreads = 256;

inline unsigned int blocks_for(long long n) { return (unsigned int)((n + kThreads - 1) / kThreads); }

// sin and cos through sincospi: its argument reduction is exact and needs no local memory, unlike sin / cos of an
// argument the compiler cannot bound
__device__ __forceinline__ void sin_cos(double th, double* s, double* c) { sincospi(th * (1.0 / M_PI), s, c); }

// ---- map deformation (float32, each operation rounded as written) ---------------------------------------------------

// quaternion (w, x, y, z) of the rotation R (row-major 3x3): the candidate row of the largest of
// 4w^2, 4x^2, 4y^2, 4z^2 (the first one on ties), divided by 2 sqrt(max(that, 0))
__device__ __forceinline__ float4 quat_of_rotation(const float* c) {
    const float r00 = c[0], r01 = c[1], r02 = c[2], r10 = c[4], r11 = c[5], r12 = c[6], r20 = c[8], r21 = c[9],
                r22 = c[10];
    const float f0 = __fadd_rn(__fadd_rn(__fadd_rn(1.f, r00), r11), r22);
    const float f1 = __fsub_rn(__fsub_rn(__fadd_rn(1.f, r00), r11), r22);
    const float f2 = __fsub_rn(__fadd_rn(__fsub_rn(1.f, r00), r11), r22);
    const float f3 = __fadd_rn(__fsub_rn(__fsub_rn(1.f, r00), r11), r22);
    int k = 0;
    float m = f0;
    if (f1 > m) { k = 1; m = f1; }
    if (f2 > m) { k = 2; m = f2; }
    if (f3 > m) { k = 3; m = f3; }
    const float den = __fmul_rn(2.f, __fsqrt_rn(fmaxf(m, 0.f)));
    float4 q;
    if (k == 0)      q = make_float4(f0, __fsub_rn(r21, r12), __fsub_rn(r02, r20), __fsub_rn(r10, r01));
    else if (k == 1) q = make_float4(__fsub_rn(r21, r12), f1, __fadd_rn(r10, r01), __fadd_rn(r02, r20));
    else if (k == 2) q = make_float4(__fsub_rn(r02, r20), __fadd_rn(r10, r01), f2, __fadd_rn(r12, r21));
    else             q = make_float4(__fsub_rn(r10, r01), __fadd_rn(r02, r20), __fadd_rn(r12, r21), f3);
    return make_float4(__fdiv_rn(q.x, den), __fdiv_rn(q.y, den), __fdiv_rn(q.z, den), __fdiv_rn(q.w, den));
}

__global__ void __launch_bounds__(kThreads)
deform_gaussians_kernel(int P, float* __restrict__ means, float* __restrict__ rots, const float* __restrict__ timestep,
                        int T, const float* __restrict__ table, const int* __restrict__ apply_flag) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P || *apply_flag == 0) return;
    const float ts = timestep[i];
    if (!(ts >= 0.f && ts < (float)T)) return;
    const float* c = table + 12 * (size_t)(int)ts;
    bool identity = true;
#pragma unroll
    for (int k = 0; k < 12; ++k) identity = identity && c[k] == ((k == 0 || k == 5 || k == 10) ? 1.f : 0.f);
    if (identity) return;
    const float x = means[3 * (size_t)i], y = means[3 * (size_t)i + 1], z = means[3 * (size_t)i + 2];
#pragma unroll
    for (int r = 0; r < 3; ++r) {
        const float* row = c + 4 * r;
        means[3 * (size_t)i + r] =
            __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(row[0], x), __fmul_rn(row[1], y)), __fmul_rn(row[2], z)), row[3]);
    }
    const float4 a = quat_of_rotation(c);
    float* q = rots + 4 * (size_t)i;           // no float4 access: the view of a flat buffer is only 4-byte aligned
    const float4 b = make_float4(q[0], q[1], q[2], q[3]);
    // Hamilton product a b, (w, x, y, z)
    float4 o;
    o.x = __fsub_rn(__fsub_rn(__fsub_rn(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)), __fmul_rn(a.z, b.z)),
                    __fmul_rn(a.w, b.w));
    o.y = __fsub_rn(__fadd_rn(__fadd_rn(__fmul_rn(a.x, b.y), __fmul_rn(a.y, b.x)), __fmul_rn(a.z, b.w)),
                    __fmul_rn(a.w, b.z));
    o.z = __fadd_rn(__fadd_rn(__fsub_rn(__fmul_rn(a.x, b.z), __fmul_rn(a.y, b.w)), __fmul_rn(a.z, b.x)),
                    __fmul_rn(a.w, b.y));
    o.w = __fadd_rn(__fsub_rn(__fadd_rn(__fmul_rn(a.x, b.w), __fmul_rn(a.y, b.z)), __fmul_rn(a.z, b.y)),
                    __fmul_rn(a.w, b.x));
    q[0] = o.x; q[1] = o.y; q[2] = o.z; q[3] = o.w;
}

// ---- SE(3) in double -------------------------------------------------------------------------------------------------

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

__device__ void skew(const double* w, double (*W)[3]) {
    W[0][0] = 0.0;   W[0][1] = -w[2]; W[0][2] = w[1];
    W[1][0] = w[2];  W[1][1] = 0.0;   W[1][2] = -w[0];
    W[2][0] = -w[1]; W[2][1] = w[0];  W[2][2] = 0.0;
}

// exp of xi = (phi, rho): R = I + A W + B W^2, V = I + B W + C W^2, t = V rho
__device__ void exp_se3(const double* xi, double* E) {
    const double th2 = xi[0] * xi[0] + xi[1] * xi[1] + xi[2] * xi[2], th = sqrt(th2);
    double cA, cB, cC;
    if (th < 1e-6) {
        cA = 1.0 - th2 / 6.0; cB = 0.5 - th2 / 24.0; cC = 1.0 / 6.0 - th2 / 120.0;
    } else {
        double sn, cs;
        sin_cos(th, &sn, &cs);
        cA = sn / th; cB = (1.0 - cs) / th2; cC = (th - sn) / (th2 * th);
    }
    double W[3][3], W2[3][3];
    skew(xi, W);
    for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c) W2[r][c] = W[r][0] * W[0][c] + W[r][1] * W[1][c] + W[r][2] * W[2][c];
    for (int r = 0; r < 3; ++r) {
        double tv = 0.0;
        for (int c = 0; c < 3; ++c) {
            const double I = r == c ? 1.0 : 0.0;
            E[4 * r + c] = I + cA * W[r][c] + cB * W2[r][c];
            tv += (I + cB * W[r][c] + cC * W2[r][c]) * xi[3 + c];
        }
        E[4 * r + 3] = tv;
    }
}

// rotation angle of a (nearly orthonormal) rotation: atan2(|vee(R - R^T)| / 2, (tr R - 1) / 2), which a symmetric
// departure from orthonormality does not disturb, unlike acos of the trace alone
__device__ double rotation_angle(const double* E) {
    const double a = 0.5 * (E[9] - E[6]), b = 0.5 * (E[2] - E[8]), c = 0.5 * (E[4] - E[1]);
    return atan2(sqrt(a * a + b * b + c * c), 0.5 * (E[0] + E[5] + E[10] - 1.0));
}

// log of a rigid transform whose rotation angle is below pi: phi = theta / sin theta vee(R - R^T) / 2,
// rho = V^-1 t with V^-1 = I - W/2 + (1 - theta sin theta / (2 (1 - cos theta))) / theta^2 W^2
__device__ void log_se3(const double* E, double* xi) {
    const double th = rotation_angle(E);
    double sn, cs;
    sin_cos(th, &sn, &cs);
    const double s = th < 1e-6 ? 1.0 + th * th / 6.0 : th / sn;
    xi[0] = 0.5 * s * (E[9] - E[6]);
    xi[1] = 0.5 * s * (E[2] - E[8]);
    xi[2] = 0.5 * s * (E[4] - E[1]);
    const double th2 = th * th;
    const double g = th < 1e-4 ? 1.0 / 12.0 + th2 / 720.0 : (1.0 - th * sn / (2.0 * (1.0 - cs))) / th2;
    double W[3][3];
    skew(xi, W);
    const double t[3] = {E[3], E[7], E[11]};
    for (int r = 0; r < 3; ++r) {
        double v = t[r];
        for (int c = 0; c < 3; ++c) {
            const double w2 = W[r][0] * W[0][c] + W[r][1] * W[1][c] + W[r][2] * W[2][c];
            v += (-0.5 * W[r][c] + g * w2) * t[c];
        }
        xi[3 + r] = v;
    }
}

// adjoint of a rigid transform, (phi, rho) order: [[R, 0], [t^ R, R]]
__device__ void adjoint(const double* T, double (*A)[6]) {
    double tx[3][3];
    const double t[3] = {T[3], T[7], T[11]};
    skew(t, tx);
    for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c) {
            const double R = T[4 * r + c];
            double tR = 0.0;
            for (int k = 0; k < 3; ++k) tR += tx[r][k] * T[4 * k + c];
            A[r][c] = R; A[r][3 + c] = 0.0; A[3 + r][c] = tR; A[3 + r][3 + c] = R;
        }
}

// inverse left Jacobian of se(3) through the second order of its series: I - ad_e / 2 + ad_e^2 / 12
__device__ void jl_inverse(const double* e, double (*J)[6]) {
    double ad[6][6], P[3][3], Q[3][3];
    skew(e, P);
    skew(e + 3, Q);
    for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c) {
            ad[r][c] = P[r][c]; ad[r][3 + c] = 0.0; ad[3 + r][c] = Q[r][c]; ad[3 + r][3 + c] = P[r][c];
        }
    for (int r = 0; r < 6; ++r)
        for (int c = 0; c < 6; ++c) {
            double a2 = 0.0;
            for (int k = 0; k < 6; ++k) a2 += ad[r][k] * ad[k][c];
            J[r][c] = (r == c ? 1.0 : 0.0) - 0.5 * ad[r][c] + a2 / 12.0;
        }
}

__device__ __forceinline__ bool edge_ok(const int* edges, int e, int N) {
    const int i = edges[2 * e], j = edges[2 * e + 1];
    return i >= 0 && i < N && j >= 0 && j < N && i != j;
}

// E = Z T_i T_j^-1 of edge e
__device__ void edge_error(const double* poses, const int* edges, const double* Z, int e, double* E) {
    const int i = edges[2 * e], j = edges[2 * e + 1];
    double Tji[12], ZTi[12];
    rigid_inverse(poses + 12 * (size_t)j, Tji);
    compose(Z + 12 * (size_t)e, poses + 12 * (size_t)i, ZTi);
    compose(ZTi, Tji, E);
}

// per edge: r = log(E), d r / d xi_i = Jl^-1(r) Ad(Z), d r / d xi_j = -Jl^-1(r) Ad(E)
__global__ void __launch_bounds__(kThreads)
pose_graph_edges_kernel(int N, int E, const double* __restrict__ poses, const int* __restrict__ edges,
                        const double* __restrict__ Z, double* __restrict__ residuals, double* __restrict__ jac) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= E) return;
    double* r = residuals + 6 * (size_t)e;
    double* Ji = jac + 72 * (size_t)e;
    double* Jj = Ji + 36;
    if (!edge_ok(edges, e, N)) {
        for (int k = 0; k < 6; ++k) r[k] = NAN;
        for (int k = 0; k < 72; ++k) Ji[k] = 0.0;
        return;
    }
    double Er[12], Jinv[6][6], Az[6][6], Ae[6][6];
    edge_error(poses, edges, Z, e, Er);
    log_se3(Er, r);
    jl_inverse(r, Jinv);
    adjoint(Z + 12 * (size_t)e, Az);
    adjoint(Er, Ae);
    for (int a = 0; a < 6; ++a)
        for (int b = 0; b < 6; ++b) {
            double si = 0.0, sj = 0.0;
            for (int k = 0; k < 6; ++k) { si += Jinv[a][k] * Az[k][b]; sj += Jinv[a][k] * Ae[k][b]; }
            Ji[6 * a + b] = si;
            Jj[6 * a + b] = -sj;
        }
}

// H = sum_e A^T W A, b = sum_e A^T W r over the free nodes (node 0 is fixed), edge by edge in order: within an edge
// the four 6x6 blocks and the two 6-vectors are disjoint, one thread per entry
__global__ void __launch_bounds__(kThreads)
pose_graph_assemble_kernel(int N, int E, const int* __restrict__ edges, const double* __restrict__ weights,
                           const double* __restrict__ residuals, const double* __restrict__ jac,
                           double* __restrict__ H, double* __restrict__ b) {
    const size_t n = 6 * (size_t)(N - 1);
    const int tid = threadIdx.x;
    for (int e = 0; e < E; ++e) {
        if (edge_ok(edges, e, N)) {
            const int ni = edges[2 * e], nj = edges[2 * e + 1];
            const double* Ai = jac + 72 * (size_t)e;
            const double* r = residuals + 6 * (size_t)e;
            const double wr = weights[2 * e], wt = weights[2 * e + 1];
            if (tid < 144) {
                const int blk = tid / 36, rr = (tid % 36) / 6, cc = tid % 6;
                const int np = (blk >> 1) ? nj : ni, nq = (blk & 1) ? nj : ni;
                const double* Ap = Ai + ((blk >> 1) ? 36 : 0);
                const double* Aq = Ai + ((blk & 1) ? 36 : 0);
                if (np > 0 && nq > 0) {
                    double s = 0.0;
                    for (int k = 0; k < 6; ++k) s += Ap[6 * k + rr] * (k < 3 ? wr : wt) * Aq[6 * k + cc];
                    H[(6 * (size_t)(np - 1) + rr) * n + 6 * (size_t)(nq - 1) + cc] += s;
                }
            } else if (tid < 156) {
                const int p = (tid - 144) / 6, rr = (tid - 144) % 6;
                const int np = p ? nj : ni;
                const double* Ap = Ai + (p ? 36 : 0);
                if (np > 0) {
                    double s = 0.0;
                    for (int k = 0; k < 6; ++k) s += Ap[6 * k + rr] * (k < 3 ? wr : wt) * r[k];
                    b[6 * (size_t)(np - 1) + rr] += s;
                }
            }
        }
        __syncthreads();
    }
}

__device__ void rotation_angle_and_shift(const double* E, double* out) {
    out[0] = sqrt(E[3] * E[3] + E[7] * E[7] + E[11] * E[11]);
    out[1] = rotation_angle(E);
}

__global__ void __launch_bounds__(kThreads)
pose_graph_update_kernel(int N, int E, int T, double* __restrict__ poses, const double* __restrict__ poses_old,
                         const double* __restrict__ xi, const int* __restrict__ edges, const double* __restrict__ Z,
                         const int* __restrict__ frame_node, double max_m, double max_rad, float* __restrict__ table,
                         int* __restrict__ flag, double* __restrict__ edge_err) {
    __shared__ int ok;
    if (threadIdx.x == 0) ok = 1;
    for (int n = 1 + threadIdx.x; n < N; n += blockDim.x) {
        double Ex[12], Tn[12];
        exp_se3(xi + 6 * (size_t)(n - 1), Ex);
        compose(Ex, poses + 12 * (size_t)n, Tn);
        for (int k = 0; k < 12; ++k) poses[12 * (size_t)n + k] = Tn[k];
    }
    __syncthreads();
    for (int e = threadIdx.x; e < E; e += blockDim.x) {
        double err[2] = {NAN, NAN};
        if (edge_ok(edges, e, N)) {
            double Er[12];
            edge_error(poses, edges, Z, e, Er);
            rotation_angle_and_shift(Er, err);
        }
        edge_err[2 * e] = err[0];
        edge_err[2 * e + 1] = err[1];
        if (!(err[0] <= max_m && err[1] <= max_rad)) atomicAnd(&ok, 0);
    }
    for (int s = threadIdx.x; s < T; s += blockDim.x) {
        const int n = frame_node[s];
        float* c = table + 12 * (size_t)s;
        if (n < 0 || n >= N) {
            for (int k = 0; k < 12; ++k) c[k] = (k == 0 || k == 5 || k == 10) ? 1.f : 0.f;
            continue;
        }
        bool same = true;                       // an unmoved node: the identity, exactly
        for (int k = 0; k < 12; ++k) same = same && poses[12 * (size_t)n + k] == poses_old[12 * (size_t)n + k];
        if (same) {
            for (int k = 0; k < 12; ++k) c[k] = (k == 0 || k == 5 || k == 10) ? 1.f : 0.f;
            continue;
        }
        double inv[12], C[12];
        rigid_inverse(poses + 12 * (size_t)n, inv);
        compose(inv, poses_old + 12 * (size_t)n, C);
        for (int k = 0; k < 12; ++k) c[k] = (float)C[k];
    }
    __syncthreads();
    if (threadIdx.x == 0) *flag = ok;
}

}  // namespace

}  // namespace sb

using namespace sb;

extern "C" {

SB_API int sb_deform_gaussians(int P, float* means3D, float* unnorm_rotations, const float* timestep, int T,
                               const float* corrections, const int* apply_flag, void* stream) {
    if (P < 0 || T < 1 || !apply_flag || !corrections || (P > 0 && (!means3D || !unnorm_rotations || !timestep)))
        return SB_ERR_BAD_ARG;
    if (P == 0) return SB_OK;
    deform_gaussians_kernel<<<blocks_for(P), kThreads, 0, static_cast<cudaStream_t>(stream)>>>(
        P, means3D, unnorm_rotations, timestep, T, corrections, apply_flag);
    SB_LAUNCH_CHECK("deform_gaussians_kernel");
    return SB_OK;
}

SB_API int sb_pose_graph_normal_equations(int N, int E, const double* poses, const int* edges, const double* Z,
                                          const double* weights, double* residuals, double* jacobians, double* H,
                                          double* b, void* stream) {
    if (N < 2 || N > 20000 || E < 1 || !poses || !edges || !Z || !weights || !residuals || !jacobians || !H || !b)
        return SB_ERR_BAD_ARG;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const size_t n = 6 * (size_t)(N - 1);
    SB_CUDA_CHECK(cudaMemsetAsync(H, 0, n * n * sizeof(double), st));
    SB_CUDA_CHECK(cudaMemsetAsync(b, 0, n * sizeof(double), st));
    pose_graph_edges_kernel<<<blocks_for(E), kThreads, 0, st>>>(N, E, poses, edges, Z, residuals, jacobians);
    SB_LAUNCH_CHECK("pose_graph_edges_kernel");
    pose_graph_assemble_kernel<<<1, kThreads, 0, st>>>(N, E, edges, weights, residuals, jacobians, H, b);
    SB_LAUNCH_CHECK("pose_graph_assemble_kernel");
    return SB_OK;
}

SB_API int sb_pose_graph_update(int N, int E, int T, double* poses, const double* poses_old, const double* xi,
                                const int* edges, const double* Z, const int* frame_node, double max_residual_m,
                                double max_residual_rad, float* corrections, int* apply_flag, double* edge_err,
                                void* stream) {
    if (N < 2 || N > 20000 || E < 1 || T < 1 || !poses || !poses_old || !xi || !edges || !Z || !frame_node ||
        !corrections || !apply_flag || !edge_err || !(max_residual_m >= 0.0) || !(max_residual_rad >= 0.0))
        return SB_ERR_BAD_ARG;
    pose_graph_update_kernel<<<1, kThreads, 0, static_cast<cudaStream_t>(stream)>>>(
        N, E, T, poses, poses_old, xi, edges, Z, frame_node, max_residual_m, max_residual_rad, corrections, apply_flag,
        edge_err);
    SB_LAUNCH_CHECK("pose_graph_update_kernel");
    return SB_OK;
}

}  // extern "C"
