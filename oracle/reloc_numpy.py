"""NumPy restatement of csrc/reloc.cu (the rules in include/splatam_b200.h, "relocalisation"): thumbnail descriptors
(float32, each operation rounded as written, sums in the kernel's order, so the result is bit-equal), their scores
(double; the kernel's order of summation differs, so agreement is to rounding), top-k and the tracking health
record."""
import numpy as np

THUMB_ROWS = 48
MAX_K = 8
SIL_THRES = np.float32(0.99)
_G = (np.float32(0.299), np.float32(0.587), np.float32(0.114))


def thumbnail_size(H, W):
    s = max(1, H // THUMB_ROWS)
    return H // s, W // s, s


def _block_means(rgb, depth, sil):
    """rgb [3,H,W], depth [H,W], sil [H,W] or None (float32) -> [2,h,w] before the blur."""
    H, W = depth.shape
    h, w, s = thumbnail_size(H, W)
    f32 = np.float32
    with np.errstate(all="ignore"):
        grey = ((_G[0] * rgb[0]).astype(f32) + (_G[1] * rgb[1]).astype(f32)).astype(f32)
        grey = (grey + (_G[2] * rgb[2]).astype(f32)).astype(f32)
        d = depth.astype(f32)
        seen = np.ones((H, W), bool)
        if sil is not None:
            seen = sil > SIL_THRES
            d = (d / sil.astype(f32)).astype(f32)
        gv = seen & np.isfinite(grey)
        dv = seen & np.isfinite(d) & (d > 0)
    out = np.empty((2, h, w), f32)
    for c, (val, ok) in enumerate(((grey, gv), (d, dv))):
        val = np.where(ok, val, f32(0))[:h * s, :w * s].reshape(h, s, w, s)
        ok = ok[:h * s, :w * s].reshape(h, s, w, s)
        acc = np.zeros((h, w), f32)
        cnt = np.zeros((h, w), np.int64)
        for yy in range(s):                          # row-major order inside each block, as the kernel sums
            for xx in range(s):
                acc = (acc + val[:, yy, :, xx]).astype(f32)
                cnt += ok[:, yy, :, xx]
        with np.errstate(all="ignore"):
            mean = (acc / cnt.astype(f32)).astype(f32)
        out[c] = np.where(2 * cnt >= s * s, mean, f32(np.nan))
    return out


def _blur(x):
    """3x3 binomial blur of a [h,w] float32 plane over its valid (non-NaN) neighbours; NaN stays NaN."""
    h, w = x.shape
    f32 = np.float32
    acc = np.zeros((h, w), f32)
    ws = np.zeros((h, w), f32)
    pad = np.full((h + 2, w + 2), np.nan, f32)
    pad[1:-1, 1:-1] = x
    for dy in (-1, 0, 1):
        for dx in (-1, 0, 1):
            v = pad[1 + dy:1 + dy + h, 1 + dx:1 + dx + w]
            wt = f32((2 if dy == 0 else 1) * (2 if dx == 0 else 1))
            ok = ~np.isnan(v)
            acc = np.where(ok, (acc + (wt * np.where(ok, v, f32(0))).astype(f32)).astype(f32), acc)
            ws = np.where(ok, (ws + wt).astype(f32), ws)
    with np.errstate(all="ignore"):
        out = (acc / ws).astype(f32)
    return np.where(np.isnan(x), f32(np.nan), out)


def thumbnails(rgb, depth, sil=None):
    """rgb [B,3,H,W], depth [B,H,W], sil [B,H,W] or None -> descriptors float32 [B,2,h,w]."""
    rgb, depth = np.asarray(rgb, np.float32), np.asarray(depth, np.float32)
    sil = None if sil is None else np.asarray(sil, np.float32)
    out = []
    for b in range(depth.shape[0]):
        m = _block_means(rgb[b], depth[b], None if sil is None else sil[b])
        out.append(np.stack([_blur(m[0]), _blur(m[1])]))
    return np.stack(out)


def score(query, database):
    """query [2,h,w], database [N,2,h,w] -> scores float64 [N] (zero-mean NCC per channel, their mean; -2 where
    fewer than half of the query's valid pixels are valid in both, in either channel)."""
    q = np.asarray(query, np.float64).reshape(2, -1)
    d = np.asarray(database, np.float64).reshape(len(database), 2, -1)
    out = np.empty(len(d))
    for e in range(len(d)):
        sc = 0.0
        for c in range(2):
            qv = ~np.isnan(q[c])
            both = qv & ~np.isnan(d[e, c])
            n, nq = int(both.sum()), int(qv.sum())
            if nq == 0 or n < 2 or 2 * n < nq:
                sc = None
                break
            a, b = q[c][both], d[e, c][both]
            ea, eb = a - a.mean(), b - b.mean()
            va, vb = (ea * ea).sum(), (eb * eb).sum()
            sc += (ea * eb).sum() / np.sqrt(va * vb) if va > 0 and vb > 0 else 0.0
        out[e] = -2.0 if sc is None else 0.5 * sc
    return out


def topk(scores, k):
    """(indices, scores) of the k best: numpy's stable argsort of -score (ties: the lower index); NaN last."""
    s = np.where(np.isnan(scores), -np.inf, np.asarray(scores, np.float64))
    idx = np.argsort(-s, kind="stable")[:k]
    return idx.astype(np.int32), s[idx]


def health(depth_sil, frame_depth, tau_abs, tau_rel, min_coverage, min_inliers):
    """sb_track_health's record [valid, covered, inliers, rms, healthy] (float64)."""
    f32 = np.float32
    acc, sil = np.asarray(depth_sil[0], f32), np.asarray(depth_sil[1], f32)
    df = np.asarray(frame_depth, f32).reshape(acc.shape)
    with np.errstate(all="ignore"):
        valid = np.isfinite(df) & (df > 0)
        cov = valid & (sil > SIL_THRES)
        r = ((acc / sil).astype(f32) - df).astype(f32)
        lim = np.maximum(f32(tau_abs), (f32(tau_rel) * df).astype(f32))
        inl = cov & (np.abs(r) < lim)
    nv, nc, ni = float(valid.sum()), float(cov.sum()), float(inl.sum())
    rms = float(np.sqrt((r[cov].astype(np.float64) ** 2).sum() / nc)) if nc > 0 else np.inf
    ok = nv > 0 and nc > 0 and nc / nv >= min_coverage and ni / nc >= min_inliers
    return np.array([nv, nc, ni, rms, 1.0 if ok else 0.0])
