"""NumPy restatement of sb_rgbd_icp_align's photometric additions (csrc/icp.cu) and of sb_track_health_rgb's colour
NCC (csrc/reloc.cu), on top of oracle/icp_numpy.py, which this module imports and leaves as it is.  Every float32
operation is rounded on its own, as the kernels' __f*_rn are, so the grey pyramid, the gradients and the photometric
codes compare bit for bit; the sums and the solve are float64.

    pyramid(depth_sil, model_rgb, data, data_rgb, K) -> icp_numpy.pyramid's levels, each with model_grey, data_grey
                                                        [H,W] and model_grad [2,H,W] added
    associate(level, T, l) -> (assoc, photo codes, geometric terms [30], photometric terms [29])
    align(depth_sil, model_rgb, data, data_rgb, K, w2c_prev, w2c_init, iters, weight) -> (w2c, stats [66], levels)
    health_ncc(depth_sil, frame_depth, map_rgb, frame_rgb, ...) -> sb_track_health_rgb's record [7] (colour NCC)"""
import numpy as np

from oracle import icp_numpy as G
from oracle import reloc_numpy as Rn

f32 = np.float32
STATS = 66
MAX_RESIDUAL = f32(0.3)
MAX_RMS = 0.1
MIN_PAIRS = 32.0
MIN_NCC_PAIRS = 64.0


def grey(rgb):
    """(0.299 r + 0.587 g) + 0.114 b of rgb [3,...] in float32, reloc_numpy's weights and order."""
    rgb = np.asarray(rgb, f32)
    with np.errstate(all="ignore"):
        return (rgb[0] * Rn._G[0] + rgb[1] * Rn._G[1]) + rgb[2] * Rn._G[2]


def downsample_grey(depth, g):
    """The mean of g over exactly the samples icp_numpy.downsample averages of `depth`; NaN where none."""
    H, W = depth.shape[0] >> 1, depth.shape[1] >> 1
    sl = [(slice(0, 2 * H, 2), slice(0, 2 * W, 2)), (slice(0, 2 * H, 2), slice(1, 2 * W, 2)),
          (slice(1, 2 * H, 2), slice(0, 2 * W, 2)), (slice(1, 2 * H, 2), slice(1, 2 * W, 2))]
    m = np.full((H, W), np.inf, f32)
    for s in sl:
        m = np.where(depth[s] > 0, np.fmin(m, depth[s]), m)
    total, cnt = np.zeros((H, W), f32), np.zeros((H, W), np.int32)
    for s in sl:
        with np.errstate(invalid="ignore"):
            use = (depth[s] > 0) & ((depth[s] - m) <= G.PYR_BAND)
            total = total + np.where(use, g[s], f32(0))
        cnt += use
    with np.errstate(all="ignore"):
        return np.where(cnt > 0, total / cnt.astype(f32), f32(np.nan)).astype(f32)


def gradient(g, normal):
    """Central differences of g where the model normal is valid, NaN elsewhere: [2,H,W]."""
    out = np.full((2,) + g.shape, np.nan, f32)
    ok = (normal[0] != 0) | (normal[1] != 0) | (normal[2] != 0)
    with np.errstate(all="ignore"):
        gu = (g[1:-1, 2:] - g[1:-1, :-2]) * f32(0.5)
        gv = (g[2:, 1:-1] - g[:-2, 1:-1]) * f32(0.5)
    inner = ok[1:-1, 1:-1]
    out[0, 1:-1, 1:-1] = np.where(inner, gu, f32(np.nan))
    out[1, 1:-1, 1:-1] = np.where(inner, gv, f32(np.nan))
    return out


def pyramid(depth_sil, model_rgb, data, data_rgb, K):
    levels = G.pyramid(depth_sil, data, K)
    gm, gd = grey(model_rgb), grey(data_rgb)
    for l, L in enumerate(levels):
        if l == 0:
            gm = np.where(L["model_depth"] > 0, gm, f32(np.nan)).astype(f32)
            gd = np.where(L["data_depth"] > 0, gd, f32(np.nan)).astype(f32)
        else:
            P = levels[l - 1]
            gm, gd = downsample_grey(P["model_depth"], gm), downsample_grey(P["data_depth"], gd)
        L.update(model_grey=gm, data_grey=gd, model_grad=gradient(gm, L["model_normal"]))
    return levels


def photometric_jacobian(p, grad, K):
    """J_I [N,6] = [p x g, g], g = (dpi/dp)^T grad, in the dtype of p (float32 rounded as the kernel, or float64)."""
    fx, fy = K[0], K[1]
    dt = p.dtype.type
    g0 = (grad[0] * dt(fx)) / p[2]
    g1 = (grad[1] * dt(fy)) / p[2]
    g2 = -((g0 * p[0] + g1 * p[1]) / p[2])
    g = np.stack([g0, g1, g2])
    return np.concatenate([G.cross(p, g), g]).T


def sample(L, p):
    """Bilinear model grey and gradient at the continuous projection of p [3,N] (float32): (ok, I, gu, gv)."""
    fx, fy, cx, cy = L["K"]
    H, W = L["model_grey"].shape
    with np.errstate(all="ignore"):
        uc = (fx * p[0]) / p[2] + cx
        vc = (fy * p[1]) / p[2] + cy
        u0, v0 = np.floor(uc), np.floor(vc)
        ok = (u0 >= 0) & (u0 + f32(1) < f32(W)) & (v0 >= 0) & (v0 + f32(1) < f32(H))
    ui, vi = np.where(ok, u0, 0).astype(np.int64), np.where(ok, v0, 0).astype(np.int64)
    a, b = (uc - u0).astype(f32), (vc - v0).astype(f32)
    a1, b1 = f32(1) - a, f32(1) - b
    w = [a1 * b1, a * b1, a1 * b, a * b]
    taps = [(vi, ui), (vi, ui + 1), (vi + 1, ui), (vi + 1, ui + 1)]
    out = []
    for m in (L["model_grey"], L["model_grad"][0], L["model_grad"][1]):
        acc = np.zeros(p.shape[1], f32)
        for wk, (y, x) in zip(w, taps):
            v = m[np.minimum(y, H - 1), np.minimum(x, W - 1)]
            ok &= np.isfinite(v)
            with np.errstate(all="ignore"):
                acc = acc + wk * v
        out.append(acc)
    return (ok, *out)


def associate(L, T, l):
    assoc, terms, _, _ = G.associate(L, T, l)
    R = np.asarray(T, np.float64).reshape(3, 4).astype(f32)
    V = L["data_vertex"]
    p = np.stack([((R[r, 0] * V[0] + R[r, 1] * V[1]) + R[r, 2] * V[2]) + R[r, 3] for r in range(3)])
    pair = assoc == 2
    ps, Id = p[:, pair], L["data_grey"][pair]
    ok, I, gu, gv = sample(L, ps)
    with np.errstate(all="ignore"):
        r = I - Id
        ok &= np.abs(r) <= MAX_RESIDUAL
        J = photometric_jacobian(ps, np.stack([gu, gv]), L["K"]).astype(f32)
    ok &= np.all(np.isfinite(J), axis=1)
    photo = np.zeros(assoc.shape, np.uint8)
    photo[pair] = np.where(ok, 2, 1)
    J64, r64 = J[ok].astype(np.float64), r[ok].astype(np.float64)
    A = J64.T @ J64
    pterms = np.concatenate([A[np.triu_indices(6)], J64.T @ r64, [float(r64 @ r64), float(ok.sum())]])
    return assoc, photo, terms, pterms


def align(depth_sil, model_rgb, data, data_rgb, K, w2c_prev, w2c_init, iters=(10, 5, 4), weight=0.0):
    levels = pyramid(depth_sil, model_rgb, data, data_rgb, K)
    prev = np.asarray(w2c_prev, f32).astype(np.float64)
    init = np.asarray(w2c_init, f32).astype(np.float64)
    T = (G._h(prev[:3]) @ G._h(G.rigid_inverse(init)))[:3]
    lam2 = float(np.float32(weight)) ** 2
    stats = np.zeros(STATS)
    for l in range(G.LEVELS - 1, -1, -1):
        for _ in range(int(iters[l])):
            _, _, terms, ph = associate(levels[l], T, l)
            joint = terms.copy()
            joint[:27] = terms[:27] + lam2 * ph[:27]
            stats[8:29], stats[29:35], stats[35] = joint[:21], joint[21:27], terms[27]
            stats[3], stats[4] = terms[28], terms[29]
            stats[36] = ph[28]
            stats[37] = np.sqrt(ph[27] / ph[28]) if ph[28] > 0 else np.inf
            stats[38:66] = ph[:28]
            ok, xi, ratio = G.solve(joint)
            stats[5] = ratio if ok else 0.0
            if not ok:
                stats[6] = stats[7] = 1.0
                continue
            stats[7] = 0.0
            T = (G._h(G.exp_se3(xi)) @ G._h(T))[:3]
    inl, valid = stats[3], stats[4]
    frac = inl / valid if valid > 0 else 0.0
    rms = np.sqrt(stats[35] / inl) if inl > 0 else np.inf
    photo_ok = weight == 0 or (stats[36] >= MIN_PAIRS and stats[37] <= MAX_RMS)
    acc = (valid > 0 and frac >= G.MIN_INLIER_FRAC and rms <= G.MAX_RMS and stats[5] >= G.MIN_PIVOT_RATIO
           and stats[7] == 0 and photo_ok)
    stats[0], stats[1], stats[2] = float(acc), frac, rms
    if not acc:
        return np.asarray(w2c_init, f32).copy(), stats, levels
    out = np.eye(4, dtype=f32)
    out[:3] = (G._h(G.rigid_inverse(T)) @ G._h(prev[:3]))[:3].astype(f32)
    return out, stats, levels


def health_ncc(depth_sil, frame_depth, map_rgb, frame_rgb, tau_abs, tau_rel, min_coverage, min_inliers, min_ncc):
    """sb_track_health_rgb's record [valid, covered, inliers, rms, healthy, ncc pairs, ncc] (float64): the colour NCC
    (each channel centred on its own mean, the sums pooled over the channels) over the inliers whose six colour values
    are finite."""
    st = Rn.health(depth_sil, frame_depth, tau_abs, tau_rel, min_coverage, min_inliers)
    acc, sil = np.asarray(depth_sil[0], f32), np.asarray(depth_sil[1], f32)
    df = np.asarray(frame_depth, f32).reshape(acc.shape)
    m, f = np.asarray(map_rgb, f32).reshape(3, *acc.shape), np.asarray(frame_rgb, f32).reshape(3, *acc.shape)
    with np.errstate(all="ignore"):
        r = ((acc / sil).astype(f32) - df).astype(f32)
        lim = np.maximum(f32(tau_abs), f32(tau_rel) * df)
        inl = np.isfinite(df) & (df > 0) & (sil > Rn.SIL_THRES) & (np.abs(r) < lim)
    use = inl & np.isfinite(m).all(0) & np.isfinite(f).all(0)
    n = float(use.sum())
    ncc = 0.0
    if n > 0:
        a, b = m[:, use].astype(np.float64), f[:, use].astype(np.float64)
        ea, eb = a - a.sum(1, keepdims=True) / n, b - b.sum(1, keepdims=True) / n
        va, vb = (ea * ea).sum(), (eb * eb).sum()
        ncc = float((ea * eb).sum() / np.sqrt(va * vb)) if va > 0 and vb > 0 else 0.0
    ok = bool(st[4]) and n >= MIN_NCC_PAIRS and ncc >= min_ncc
    return np.array([st[0], st[1], st[2], st[3], 1.0 if ok else 0.0, n, ncc])
