"""An analytic depth scene for the ICP tests: three orthogonal planes (x = -1, y = 1, z = 3 in world metres) and a
sphere, ray-cast in float64 at a pinhole camera with the pixel centre at integer coordinates."""
import numpy as np

SPHERE_C = np.array([0.3, 0.2, 2.2])
SPHERE_R = 0.3


def rot(axis, deg):
    a = np.asarray(axis, np.float64)
    a = a / np.linalg.norm(a)
    th = np.deg2rad(deg)
    K = np.array([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]])
    return np.eye(3) + np.sin(th) * K + (1 - np.cos(th)) * K @ K


def rigid(R, t):
    M = np.eye(4)
    M[:3, :3], M[:3, 3] = R, t
    return M


def intrinsics(H, W, f=None):
    f = 0.75 * W if f is None else f
    return np.array([[f, 0, (W - 1) / 2], [0, f, (H - 1) / 2], [0, 0, 1.0]])


def depth(w2c, K, H, W, planes=((0, -1.0), (1, 1.0), (2, 3.0)), sphere=True):
    """float32 [H,W] camera depth of the scene seen by w2c; 0 where nothing is hit.  planes: (axis, offset) of the
    world planes x_axis = offset."""
    c2w = np.linalg.inv(w2c)
    u, v = np.meshgrid(np.arange(W, dtype=np.float64), np.arange(H, dtype=np.float64))
    d_cam = np.stack([(u - K[0, 2]) / K[0, 0], (v - K[1, 2]) / K[1, 1], np.ones_like(u)], -1)   # z = 1: t = depth
    d = d_cam @ c2w[:3, :3].T
    o = c2w[:3, 3]
    best = np.full((H, W), np.inf)
    for ax, off in planes:
        with np.errstate(divide="ignore", invalid="ignore"):
            t = (off - o[ax]) / d[..., ax]
        best = np.where((t > 0) & (t < best), t, best)
    if sphere:
        oc = o - SPHERE_C
        b = d @ oc
        a = (d * d).sum(-1)
        disc = b * b - a * (oc @ oc - SPHERE_R ** 2)
        with np.errstate(invalid="ignore"):
            t = (-b - np.sqrt(disc)) / a
        best = np.where((disc > 0) & (t > 0) & (t < best), t, best)
    return np.where(np.isfinite(best), best, 0.0).astype(np.float32)


def depth_sil(w2c, K, H, W, **kw):
    """[2,H,W] float32 (depth, silhouette) as the map's depth render gives them: silhouette 1 where hit."""
    d = depth(w2c, K, H, W, **kw)
    return np.stack([d, (d > 0).astype(np.float32)])
