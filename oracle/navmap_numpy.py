"""NumPy restatement of csrc/navmap.cu's rules (include/splatam_b200.h, "navigation maps"), so the kernels can be
compared bit for bit.  The distance transform is restated from its definition -- per axis, the minimum over every
site of (q - v)^2 + f(v), as whole-array shifts -- not from the kernels' envelope algorithm; every float32 operation
is rounded on its own, as the kernels' __fadd_rn / __fmul_rn / __fdiv_rn / __fsqrt_rn are.

    labels(tsdf, weight, trunc, min_weight, occ_dist) -> uint8 [nz,ny,nx]
    obstacles(labels, unknown_is_obstacle) -> bool [nz,ny,nx]
    signed_sq_distance(obstacle_mask) -> sd2 int32 [nz,ny,nx]
    esdf_from_sd2(sd2, voxel) -> float32 [nz,ny,nx]
    query(esdf, origin, voxel, points [N,3]) -> dist [N], grad [N,3]"""
import numpy as np

f32 = np.float32
INT32_MAX = 2 ** 31 - 1
_INF = 2 ** 62          # no site in reach; finite squared distances stay below 2^28


def labels(tsdf, weight, trunc, min_weight, occ_dist):
    """0 (unknown) where W < min_weight, else 2 (occupied) where T * trunc <= occ_dist, else 1 (free)."""
    t, w = np.asarray(tsdf, f32), np.asarray(weight, f32)
    occ = t * f32(trunc) <= f32(occ_dist)
    return np.where(w < f32(min_weight), 0, np.where(occ, 2, 1)).astype(np.uint8)


def obstacles(lab, unknown_is_obstacle=True):
    lab = np.asarray(lab)
    return (lab == 2) | (bool(unknown_is_obstacle) & (lab == 0))


def _min_plus_parabola(f, axis):
    """d(q) = min over v of (q - v)^2 + f(v) along `axis` (int64, _INF where a line has no site)."""
    f = np.moveaxis(f, axis, -1)
    d = f.copy()
    n = f.shape[-1]
    has_site = (f < _INF).any(axis=-1, keepdims=True)
    for delta in range(1, n):
        dd = delta * delta
        if not (np.where(has_site, d, 0) >= dd).any():
            break                       # no sample of a line with a site can still improve
        np.minimum(d[..., delta:], f[..., :-delta] + dd, out=d[..., delta:])
        np.minimum(d[..., :-delta], f[..., delta:] + dd, out=d[..., :-delta])
    return np.moveaxis(d, -1, axis)


def _sq_distance_to(sites):
    d = np.where(sites, 0, _INF).astype(np.int64)
    for axis in (2, 1, 0):              # x, y, z
        d = _min_plus_parabola(d, axis)
    return d


def signed_sq_distance(obstacle):
    """+min |s - o|^2 over obstacles o outside the set, -min |s - f|^2 over free f inside it; INT32_MAX everywhere
    for an empty set, -INT32_MAX everywhere for a full one."""
    obstacle = np.asarray(obstacle, bool)
    a, b = _sq_distance_to(obstacle), _sq_distance_to(~obstacle)
    a = np.where(a >= _INF, INT32_MAX, a)
    b = np.where(b >= _INF, INT32_MAX, b)
    return np.where(obstacle, -b, a).astype(np.int32)


def esdf_from_sd2(sd2, voxel):
    """sign(sd2) * (voxel * sqrt(float32(|sd2|))), the sentinels +-inf."""
    sd2 = np.asarray(sd2, np.int32)
    mag = np.abs(sd2.astype(np.int64))
    with np.errstate(over="ignore"):
        m = f32(voxel) * np.sqrt(mag.astype(f32))
    m = np.where(mag == INT32_MAX, f32(np.inf), m).astype(f32)
    return np.where(sd2 < 0, -m, m).astype(f32)


def _lerp(a, b, t):
    return a + t * (b - a)


def query(esdf, origin, voxel, points):
    """Trilinear distance and its exact gradient at points [N,3] (the header's operation order); NaN outside."""
    esdf = np.asarray(esdf, f32)
    nz, ny, nx = esdf.shape
    if min(nx, ny, nz) < 2:
        raise ValueError("the query needs every grid dimension >= 2, got %s" % (esdf.shape,))
    p = np.asarray(points, f32).reshape(-1, 3)
    o, v = np.asarray(origin, f32).reshape(3), f32(voxel)
    n = np.array([nx, ny, nz])
    with np.errstate(all="ignore"):
        u = (p - o) / v
        inside = np.all(np.isfinite(u) & (u >= f32(0)) & (u <= (n - 1).astype(f32)), axis=1)
        idx = np.where(inside[:, None], np.minimum(np.floor(u), n - 2), 0).astype(np.int64)
        t = u - idx.astype(f32)
        c = [esdf[idx[:, 2] + (q >> 2), idx[:, 1] + (q >> 1 & 1), idx[:, 0] + (q & 1)] for q in range(8)]
        tx, ty, tz = t[:, 0], t[:, 1], t[:, 2]
        e00, e01 = _lerp(c[0], c[1], tx), _lerp(c[2], c[3], tx)
        e10, e11 = _lerp(c[4], c[5], tx), _lerp(c[6], c[7], tx)
        f0, f1 = _lerp(e00, e01, ty), _lerp(e10, e11, ty)
        dist = _lerp(f0, f1, tz)
        gx = _lerp(_lerp(c[1] - c[0], c[3] - c[2], ty), _lerp(c[5] - c[4], c[7] - c[6], ty), tz) / v
        gy = _lerp(e01 - e00, e11 - e10, tz) / v
        gz = (f1 - f0) / v
    grad = np.stack([gx, gy, gz], axis=1).astype(f32)
    inf = np.zeros(len(p), f32)
    for q in range(7, -1, -1):
        inf = np.where(np.isinf(c[q]), c[q], inf)
    hit = inf != 0
    dist = np.where(hit, inf, dist).astype(f32)
    grad[hit] = 0
    dist[~inside] = np.nan
    grad[~inside] = np.nan
    return dist, grad
