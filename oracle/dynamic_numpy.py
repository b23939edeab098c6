"""float32 numpy statement of the motion-mask rule (include/splatam_b200.h `sb_dynamic_*`, csrc/dynamic.cu,
splatam_b200/dynamic.py): the same bits as the CUDA kernels and the torch statement."""
import numpy as np

BINS = 32768
f32 = np.float32


def _threshold(k, scale, floor):
    t = f32(k) * f32(scale)
    return t if t > floor else f32(floor)          # a NaN product (inf * 0) takes the floor


def _shift(a, dy, dx, fill):
    """out[y, x] = a[y + dy, x + dx], `fill` outside."""
    H, W = a.shape
    out = np.full_like(a, fill)
    ys, yd = (slice(dy, H), slice(0, H - dy)) if dy >= 0 else (slice(0, H + dy), slice(-dy, H))
    xs, xd = (slice(dx, W), slice(0, W - dx)) if dx >= 0 else (slice(0, W + dx), slice(-dx, W))
    out[yd, xd] = a[ys, xs]
    return out


def _keep_supported(seed):
    n = np.zeros(seed.shape, np.int32)
    for dy in (-1, 0, 1):
        for dx in (-1, 0, 1):
            if dy or dx:
                n += _shift(seed, dy, dx, False)
    return seed & (n >= 4)


def _dilate(a, r):
    out = a.copy()
    for dy in range(-r, r + 1):
        for dx in range(-r, r + 1):
            out |= _shift(a, dy, dx, False)
    return out


def scale_of(depth_sil, gt_depth, sil_thres=0.99):
    """(r [H,W] float32, valid [H,W] bool, scale float32) of the rule."""
    d, s = depth_sil[0].astype(f32), depth_sil[1].astype(f32)
    g = np.asarray(gt_depth, f32).reshape(d.shape)
    with np.errstate(divide="ignore", invalid="ignore"):
        r = (d - g) / g
    valid = (g > 0) & np.isfinite(d) & (s > f32(sil_thres))
    hist = np.bincount((np.abs(r[valid]).view(np.uint32) >> 16).astype(np.int64), minlength=BINS)
    n = int(valid.sum())
    if n == 0:
        return r, valid, f32(0)
    b = int(np.searchsorted(np.cumsum(hist), (n - 1) // 2, side="right"))
    return r, valid, np.array([b << 16], np.uint32).view(f32)[0]


def motion_masks(depth_sil, gt_depth, k_high, k_low, r_min, tau, radius, dilate, sil_thres=0.99):
    """(dynamic [H,W] bool, inconsistent [H,W] bool, stats float32 [6] = (valid, scale, occ seeds, dis seeds,
    dynamic, inconsistent)) of one [3,H,W] depth/silhouette render and the frame's depth [H,W] (or [1,H,W])."""
    depth_sil = np.asarray(depth_sil, f32)
    s = depth_sil[1]
    g = np.asarray(gt_depth, f32).reshape(s.shape)
    r, valid, scale = scale_of(depth_sil, g, sil_thres)
    hi = _threshold(k_high, scale, f32(r_min))
    lo = _threshold(k_low, scale, f32(r_min) * f32(0.5))
    with np.errstate(invalid="ignore"):
        occ = _keep_supported(valid & (r > hi))
        dis = _keep_supported(valid & (-r > hi))
        cand = (g > 0) & ((valid & (r > lo)) | (s <= f32(sil_thres)))
    dyn = occ.copy()
    tau = f32(tau)
    for _ in range(int(radius)):
        grow = np.zeros_like(dyn)
        for dy, dx in ((-1, 0), (1, 0), (0, -1), (0, 1)):
            nd, ng = _shift(dyn, dy, dx, False), _shift(g, dy, dx, f32(0))
            grow |= nd & (np.abs(ng - g) <= tau * np.minimum(ng, g))
        dyn = dyn | (cand & grow)
    dynamic, inconsistent = _dilate(dyn, int(dilate)), _dilate(dis, int(dilate))
    stats = np.array([valid.sum(), scale, occ.sum(), dis.sum(), dynamic.sum(), inconsistent.sum()], f32)
    return dynamic, inconsistent, stats
