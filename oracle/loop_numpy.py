"""Loop closure restated in numpy (csrc/loop.cu; the rules are stated in include/splatam_b200.h): the map deformation in
float32 with every operation rounded as the kernel rounds it, and the keyframe pose graph -- residuals, Jacobians,
dense normal equations, the Gauss-Newton solve with node 0 fixed, the residual test and the per-frame correction
table -- in float64.  Poses are 4x4 w2c matrices; a tangent vector is (phi, rho), rotation first."""
import numpy as np

f32 = np.float32


def _identity12():
    return np.array([1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0], np.float32)


def quat_of_rotation(c):
    """(w, x, y, z) float32 of the rotation in correction c [12] (sb_deform_gaussians' rule)."""
    c = np.asarray(c, np.float32)
    r00, r01, r02, r10, r11, r12, r20, r21, r22 = c[0], c[1], c[2], c[4], c[5], c[6], c[8], c[9], c[10]
    one = f32(1.0)
    f = [((one + r00) + r11) + r22, ((one + r00) - r11) - r22, ((one - r00) + r11) - r22, ((one - r00) - r11) + r22]
    k = 0
    for i in (1, 2, 3):
        if f[i] > f[k]:
            k = i
    den = f32(2.0) * np.sqrt(np.maximum(f[k], f32(0.0)))
    rows = [[f[0], r21 - r12, r02 - r20, r10 - r01], [r21 - r12, f[1], r10 + r01, r02 + r20],
            [r02 - r20, r10 + r01, f[2], r12 + r21], [r10 - r01, r02 + r20, r12 + r21, f[3]]]
    return np.array([v / den for v in rows[k]], np.float32)


def deform(means, rots, timestep, table, apply_flag):
    """sb_deform_gaussians: new (means [P,3], rots [P,4]) float32."""
    means = np.array(means, np.float32)
    rots = np.array(rots, np.float32)
    table = np.asarray(table, np.float32)
    if not apply_flag:
        return means, rots
    T = table.shape[0]
    ts = np.asarray(timestep, np.float32)
    for s in np.unique(ts):
        if not (s >= 0 and s < T):
            continue
        c = table[int(s)]
        if np.array_equal(c, _identity12()):
            continue
        m = ts == s
        x, y, z = means[m, 0], means[m, 1], means[m, 2]
        out = np.empty((m.sum(), 3), np.float32)
        for r in range(3):
            out[:, r] = ((c[4 * r] * x + c[4 * r + 1] * y) + c[4 * r + 2] * z) + c[4 * r + 3]
        means[m] = out
        aw, ax, ay, az = quat_of_rotation(c)
        bw, bx, by, bz = rots[m, 0], rots[m, 1], rots[m, 2], rots[m, 3]
        rots[m] = np.stack([((aw * bw - ax * bx) - ay * by) - az * bz, ((aw * bx + ax * bw) + ay * bz) - az * by,
                            ((aw * by - ax * bz) + ay * bw) + az * bx, ((aw * bz + ax * by) - ay * bx) + az * bw], 1)
    return means, rots


# ---- SE(3), float64 ----------------------------------------------------------------------------------------------

def skew(w):
    return np.array([[0.0, -w[2], w[1]], [w[2], 0.0, -w[0]], [-w[1], w[0], 0.0]])


def exp_se3(xi):
    xi = np.asarray(xi, np.float64)
    th2 = float(xi[:3] @ xi[:3])
    th = np.sqrt(th2)
    if th < 1e-6:
        a, b, c = 1.0 - th2 / 6.0, 0.5 - th2 / 24.0, 1.0 / 6.0 - th2 / 120.0
    else:
        a, b, c = np.sin(th) / th, (1.0 - np.cos(th)) / th2, (th - np.sin(th)) / (th2 * th)
    W = skew(xi[:3])
    E = np.eye(4)
    E[:3, :3] = np.eye(3) + a * W + b * W @ W
    E[:3, 3] = (np.eye(3) + b * W + c * W @ W) @ xi[3:]
    return E


def rigid(axis, deg, t):
    """exp of a rotation of `deg` degrees about `axis` and the translation `t` (a 4x4 float64 transform)."""
    a = np.asarray(axis, np.float64)
    return exp_se3(np.concatenate([a / np.linalg.norm(a) * np.radians(deg), t]))


def random_graph(N, loops, seed):
    """A random pose graph: ground-truth poses (node 0 the identity), odometry between consecutive nodes and `loops`
    loop edges between random pairs, each measurement off the truth by ~0.2 degrees and 5 mm; the estimate chains the
    odometry.  Returns (estimated poses [N] 4x4, edges [(i, j)], measurements [E] 4x4)."""
    rng = np.random.default_rng(seed)
    gt = [np.eye(4)] + [rigid(rng.normal(size=3), rng.uniform(0, 40), rng.normal(size=3)) for _ in range(N - 1)]
    noise = lambda: exp_se3(np.concatenate([rng.normal(size=3) * 0.003, rng.normal(size=3) * 0.005]))
    edges = [(k - 1, k) for k in range(1, N)]
    Z = [noise() @ gt[k] @ inv(gt[k - 1]) for k in range(1, N)]
    for _ in range(loops):
        i, j = sorted(rng.choice(N, 2, replace=False))
        edges.append((int(i), int(j)))
        Z.append(noise() @ gt[j] @ inv(gt[i]))
    est = [gt[0]]
    for z in Z[:N - 1]:
        est.append(z @ est[-1])
    return est, edges, Z


def rotation_angle(E):
    """atan2(|vee(R - R^T)| / 2, (tr R - 1) / 2): robust to a symmetric departure from orthonormality."""
    v = 0.5 * np.array([E[2, 1] - E[1, 2], E[0, 2] - E[2, 0], E[1, 0] - E[0, 1]])
    return np.arctan2(np.linalg.norm(v), 0.5 * (E[0, 0] + E[1, 1] + E[2, 2] - 1.0))


def log_se3(E):
    th = rotation_angle(E)
    s = 1.0 + th * th / 6.0 if th < 1e-6 else th / np.sin(th)
    phi = 0.5 * s * np.array([E[2, 1] - E[1, 2], E[0, 2] - E[2, 0], E[1, 0] - E[0, 1]])
    th2 = th * th
    g = 1.0 / 12.0 + th2 / 720.0 if th < 1e-4 else (1.0 - th * np.sin(th) / (2.0 * (1.0 - np.cos(th)))) / th2
    W = skew(phi)
    return np.concatenate([phi, (np.eye(3) - 0.5 * W + g * W @ W) @ E[:3, 3]])


def inv(T):
    o = np.eye(4)
    o[:3, :3] = T[:3, :3].T
    o[:3, 3] = -T[:3, :3].T @ T[:3, 3]
    return o


def adjoint(T):
    A = np.zeros((6, 6))
    A[:3, :3] = A[3:, 3:] = T[:3, :3]
    A[3:, :3] = skew(T[:3, 3]) @ T[:3, :3]
    return A


def ad(e):
    A = np.zeros((6, 6))
    A[:3, :3] = A[3:, 3:] = skew(e[:3])
    A[3:, :3] = skew(e[3:])
    return A


def jl_inverse(e):
    a = ad(e)
    return np.eye(6) - 0.5 * a + a @ a / 12.0


def edge_error(Ti, Tj, Z):
    return Z @ Ti @ inv(Tj)


def edge_terms(Ti, Tj, Z):
    """(r = log(Z Ti Tj^-1), d r / d xi_i, d r / d xi_j) of one edge, left perturbation T <- exp(xi) T."""
    E = edge_error(Ti, Tj, Z)
    r = log_se3(E)
    J = jl_inverse(r)
    return r, J @ adjoint(Z), -J @ adjoint(E)


def normal_equations(poses, edges, Z, weights):
    """Dense (H [6(N-1)]^2, b [6(N-1)], residuals [E,6]) over nodes 1..N-1, node 0 fixed; poses [N,4,4]."""
    N = len(poses)
    n = 6 * (N - 1)
    H, b = np.zeros((n, n)), np.zeros(n)
    res = np.zeros((len(edges), 6))
    for e, (i, j) in enumerate(edges):
        r, Ai, Aj = edge_terms(poses[i], poses[j], Z[e])
        res[e] = r
        W = np.diag([weights[e][0]] * 3 + [weights[e][1]] * 3)
        for p, Ap in ((i, Ai), (j, Aj)):
            if p == 0:
                continue
            b[6 * (p - 1):6 * p] += Ap.T @ W @ r
            for q, Aq in ((i, Ai), (j, Aj)):
                if q > 0:
                    H[6 * (p - 1):6 * p, 6 * (q - 1):6 * q] += Ap.T @ W @ Aq
    return H, b, res


def edge_errors(poses, edges, Z):
    """[E,2]: (|t|, rotation angle) of Z Ti Tj^-1 per edge."""
    out = []
    for e, (i, j) in enumerate(edges):
        E = edge_error(poses[i], poses[j], Z[e])
        out.append((np.linalg.norm(E[:3, 3]), rotation_angle(E)))
    return np.array(out)


def solve(poses, edges, Z, weights, iters=10, tol=1e-10):
    """Gauss-Newton with node 0 fixed: a step with |xi| < tol is not applied and ends the solve.  Returns the new
    poses [N,4,4] and the number of steps applied."""
    poses = [np.array(p, np.float64) for p in poses]
    applied = 0
    for _ in range(iters):
        H, b, _ = normal_equations(poses, edges, Z, weights)
        L = np.linalg.cholesky(H)
        xi = -np.linalg.solve(L.T, np.linalg.solve(L, b))
        if np.linalg.norm(xi) < tol:
            break
        for n in range(1, len(poses)):
            poses[n] = exp_se3(xi[6 * (n - 1):6 * n]) @ poses[n]
        applied += 1
    return np.stack(poses), applied


def accept(poses, edges, Z, max_m, max_rad):
    err = edge_errors(poses, edges, Z)
    return bool(np.all(err[:, 0] <= max_m) and np.all(err[:, 1] <= max_rad))


def correction_table(poses_old, poses_new, frame_node):
    """float32 [T,12]: frame s takes C = T_new^-1 T_old of node frame_node[s]; the identity for an unmoved node or a
    node index < 0."""
    out = np.tile(_identity12(), (len(frame_node), 1))
    for s, n in enumerate(frame_node):
        if n < 0 or np.array_equal(poses_new[n], poses_old[n]):
            continue
        out[s] = (inv(poses_new[n]) @ poses_old[n])[:3].reshape(12).astype(np.float32)
    return out
