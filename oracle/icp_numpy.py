"""NumPy restatement of csrc/icp.cu (sb_icp_align), so the pyramid, the vertex and normal maps and the association codes
can be compared bit for bit and the normal equations and the pose to double rounding.  Every float32 operation below is
rounded on its own (numpy does not contract a * b + c), as the kernels' __fadd_rn / __fmul_rn / __fdiv_rn /
__fsqrt_rn are; the sums and the solve are float64.

    pyramid(depth_sil [2,H,W], data [H,W], K) -> [level dict(model_depth, data_depth, model_vertex, model_normal,
                                                              data_vertex, K)] for levels 0, 1, 2
    associate(level, T [3,4] float64, l) -> (assoc [H,W] uint8, terms [30] float64, J [N,6] float32, r [N] float32)
    align(depth_sil, data, K, w2c_prev, w2c_init, iters) -> (w2c [4,4] float32, stats [36] float64, levels)"""
import numpy as np

f32 = np.float32
LEVELS = 3
STATS = 36
SIL_THRES = f32(0.99)
PYR_BAND = f32(0.05)
NORMAL_SLANT = f32(5.0)
DIST0 = f32(0.1)
MIN_COUNT = 32.0
MIN_INLIER_FRAC = 0.4
MAX_RMS = 0.03
MIN_PIVOT_RATIO = 1e-5


def level0(depth_sil, data):
    d, sil = np.asarray(depth_sil[0], f32), np.asarray(depth_sil[1], f32)
    with np.errstate(all="ignore"):
        m = d / sil
    model = np.where((sil > SIL_THRES) & np.isfinite(m) & (m > 0), m, f32(0)).astype(f32)
    x = np.asarray(data, f32).reshape(d.shape)
    with np.errstate(invalid="ignore"):
        data_d = np.where(np.isfinite(x) & (x > 0), x, f32(0)).astype(f32)
    return model, data_d


def downsample(d):
    H, W = d.shape[0] >> 1, d.shape[1] >> 1
    s = [d[0:2 * H:2, 0:2 * W:2], d[0:2 * H:2, 1:2 * W:2], d[1:2 * H:2, 0:2 * W:2], d[1:2 * H:2, 1:2 * W:2]]
    m = np.full((H, W), np.inf, f32)
    for x in s:
        m = np.where(x > 0, np.fmin(m, x), m)
    total, cnt = np.zeros((H, W), f32), np.zeros((H, W), np.int32)
    for x in s:
        with np.errstate(invalid="ignore"):
            use = (x > 0) & ((x - m) <= PYR_BAND)
        total = total + np.where(use, x, f32(0))
        cnt += use
    with np.errstate(invalid="ignore", divide="ignore"):
        return np.where(cnt > 0, total / cnt.astype(f32), f32(0)).astype(f32)


def level_intrinsics(K):
    fx, fy, cx, cy = f32(K[0][0]), f32(K[1][1]), f32(K[0][2]), f32(K[1][2])
    out = []
    for _ in range(LEVELS):
        out.append((fx, fy, cx, cy))
        fx, fy, cx, cy = fx * f32(0.5), fy * f32(0.5), (cx - f32(0.5)) * f32(0.5), (cy - f32(0.5)) * f32(0.5)
    return out


def backproject(z, K):
    fx, fy, cx, cy = K
    H, W = z.shape
    u = np.arange(W, dtype=f32)[None, :]
    v = np.arange(H, dtype=f32)[:, None]
    ok = z > 0
    x = ((u - cx) / fx) * z
    y = ((v - cy) / fy) * z
    return np.where(ok[None], np.stack([x, y, z]), f32(0)).astype(f32)


def cross(a, b):
    return np.stack([a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0]])


def dot(a, b):
    return (a[0] * b[0] + a[1] * b[1]) + a[2] * b[2]


def normals(V, fx):
    """Model normals of a vertex map [3,H,W] (z = depth, 0 where invalid) at a level of focal length fx."""
    _, H, W = V.shape
    z = V[2]
    N = np.zeros_like(V)
    if H < 3 or W < 3:
        return N
    c = z[1:-1, 1:-1]
    zl, zr, zu, zd = z[1:-1, :-2], z[1:-1, 2:], z[:-2, 1:-1], z[2:, 1:-1]
    ok = (c > 0) & (zl > 0) & (zr > 0) & (zu > 0) & (zd > 0)
    for nb in (zl, zr, zu, zd):
        ok &= np.abs(nb - c) * fx <= NORMAL_SLANT * c
    dx = V[:, 1:-1, 2:] - V[:, 1:-1, :-2]
    dy = V[:, 2:, 1:-1] - V[:, :-2, 1:-1]
    cr = cross(dx, dy)
    ln = np.sqrt(dot(cr, cr))
    ok &= (ln > 0) & np.isfinite(ln)
    with np.errstate(invalid="ignore", divide="ignore"):
        n = cr / ln
    N[:, 1:-1, 1:-1] = np.where(ok[None], n, f32(0))
    return N


def pyramid(depth_sil, data, K):
    md, dd = level0(depth_sil, data)
    out = []
    for l, Kl in enumerate(level_intrinsics(K)):
        if l:
            md, dd = downsample(md), downsample(dd)
        mv = backproject(md, Kl)
        out.append(dict(model_depth=md, data_depth=dd, model_vertex=mv, model_normal=normals(mv, Kl[0]),
                        data_vertex=backproject(dd, Kl), K=Kl))
    return out


def associate(L, T, l):
    """One iteration's association and per-pixel terms at level dict L with T (3x4 float64) at level index l."""
    fx, fy, cx, cy = L["K"]
    R = np.asarray(T, np.float64).reshape(3, 4).astype(f32)
    V, MV, MN = L["data_vertex"], L["model_vertex"], L["model_normal"]
    _, H, W = V.shape
    valid = V[2] > 0
    p = np.stack([((R[r, 0] * V[0] + R[r, 1] * V[1]) + R[r, 2] * V[2]) + R[r, 3] for r in range(3)])
    with np.errstate(all="ignore"):
        uf = np.floor(((fx * p[0]) / p[2] + cx) + f32(0.5))
        vf = np.floor(((fy * p[1]) / p[2] + cy) + f32(0.5))
        inside = valid & (p[2] > 0) & (uf >= 0) & (uf < f32(W)) & (vf >= 0) & (vf < f32(H))
    ui = np.where(inside, uf, 0).astype(np.int64)
    vi = np.where(inside, vf, 0).astype(np.int64)
    q, n = MV[:, vi, ui], MN[:, vi, ui]
    d = p - q
    thr = DIST0 * f32(1 << l)
    with np.errstate(all="ignore"):
        pair = inside & (q[2] > 0) & ((n[0] != 0) | (n[1] != 0) | (n[2] != 0)) & (dot(d, d) <= thr * thr)
    assoc = np.where(pair, 2, np.where(valid, 1, 0)).astype(np.uint8)
    ps, ns, ds = p[:, pair], n[:, pair], d[:, pair]
    r = dot(ns, ds)
    J = np.concatenate([cross(ps, ns), ns]).T.astype(f32)             # [N, 6]
    J64, r64 = J.astype(np.float64), r.astype(np.float64)
    A = J64.T @ J64
    iu = np.triu_indices(6)
    terms = np.concatenate([A[iu], J64.T @ r64, [float(r64 @ r64), float(pair.sum()), float(valid.sum())]])
    return assoc, terms, J, r


def solve(terms):
    """(ok, xi [6], pivot ratio) of JtJ xi = -Jtr by Cholesky, as icp_solve_kernel."""
    A = np.zeros((6, 6))
    A[np.triu_indices(6)] = terms[:21]
    A = np.triu(A) + np.triu(A, 1).T
    g = terms[21:27]
    if not terms[28] >= MIN_COUNT:
        return False, None, 0.0
    L = np.zeros((6, 6))
    piv = []
    for j in range(6):
        d = A[j, j] - sum(L[j, q] * L[j, q] for q in range(j))
        if not (d > 0 and np.isfinite(d)):
            return False, None, 0.0
        piv.append(d)
        L[j, j] = np.sqrt(d)
        for i in range(j + 1, 6):
            L[i, j] = (A[i, j] - sum(L[i, q] * L[j, q] for q in range(j))) / L[j, j]
    y = np.zeros(6)
    for i in range(6):
        y[i] = (-g[i] - sum(L[i, q] * y[q] for q in range(i))) / L[i, i]
    xi = np.zeros(6)
    for i in range(5, -1, -1):
        xi[i] = (y[i] - sum(L[q, i] * xi[q] for q in range(i + 1, 6))) / L[i, i]
    if not np.all(np.isfinite(xi)):
        return False, None, 0.0
    return True, xi, min(piv) / max(piv)


def exp_se3(xi):
    """3x4 [R | t] of the twist xi = (w, v): R = I + A W + B W^2, t = (I + B W + C W^2) v."""
    w, v = np.asarray(xi[:3], np.float64), np.asarray(xi[3:], np.float64)
    th2 = float(w @ w)
    th = np.sqrt(th2)
    if th < 1e-6:
        a, b, c = 1.0 - th2 / 6.0, 0.5 - th2 / 24.0, 1.0 / 6.0 - th2 / 120.0
    else:
        a, b, c = np.sin(th) / th, (1.0 - np.cos(th)) / th2, (th - np.sin(th)) / (th2 * th)
    Wm = np.array([[0.0, -w[2], w[1]], [w[2], 0.0, -w[0]], [-w[1], w[0], 0.0]])
    W2 = Wm @ Wm
    I = np.eye(3)
    return np.concatenate([I + a * Wm + b * W2, ((I + b * Wm + c * W2) @ v)[:, None]], axis=1)


def _h(T):
    return np.concatenate([np.asarray(T, np.float64).reshape(3, 4), [[0.0, 0.0, 0.0, 1.0]]])


def rigid_inverse(T):
    T = np.asarray(T, np.float64).reshape(-1)[:12].reshape(3, 4)
    R, t = T[:, :3], T[:, 3]
    return np.concatenate([R.T, (-(R.T @ t))[:, None]], axis=1)


def align(depth_sil, data, K, w2c_prev, w2c_init, iters=(10, 5, 4)):
    levels = pyramid(depth_sil, data, K)
    prev = np.asarray(w2c_prev, f32).astype(np.float64)
    init = np.asarray(w2c_init, f32).astype(np.float64)
    T = (_h(prev[:3]) @ _h(rigid_inverse(init)))[:3]
    stats = np.zeros(STATS)
    for l in range(LEVELS - 1, -1, -1):
        for _ in range(int(iters[l])):
            _, terms, _, _ = associate(levels[l], T, l)
            stats[8:29], stats[29:35], stats[35] = terms[:21], terms[21:27], terms[27]
            stats[3], stats[4] = terms[28], terms[29]
            ok, xi, ratio = solve(terms)
            stats[5] = ratio if ok else 0.0
            if not ok:
                stats[6] = stats[7] = 1.0
                continue
            stats[7] = 0.0
            T = (_h(exp_se3(xi)) @ _h(T))[:3]
    inl, valid = stats[3], stats[4]
    frac = inl / valid if valid > 0 else 0.0
    rms = np.sqrt(stats[35] / inl) if inl > 0 else np.inf
    acc = valid > 0 and frac >= MIN_INLIER_FRAC and rms <= MAX_RMS and stats[5] >= MIN_PIVOT_RATIO and stats[7] == 0
    stats[0], stats[1], stats[2] = float(acc), frac, rms
    if not acc:
        return np.asarray(w2c_init, f32).copy(), stats, levels
    out = np.eye(4, dtype=f32)
    out[:3] = (_h(rigid_inverse(T)) @ _h(prev[:3]))[:3].astype(f32)
    return out, stats, levels
