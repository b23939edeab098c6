"""NumPy float32 restatement of csrc/mesh_eval.cu, operation for operation, so the kernels can be compared bit for bit.
Every float32 operation below is rounded on its own (numpy does not contract a * b + c), as the kernels'
__fadd_rn / __fmul_rn / __fdiv_rn are.

    points_visible(points [N,3], depth [B,H,W], w2c [B,4,4], K, occlusion_eps, mask=None) -> mask [N] uint8
    min_sq_dist(queries [M,3], refs [N,3], chunk) -> d2 [M] float32, the brute-force minimum"""
import numpy as np

f32 = np.float32


def points_visible(points, depth, w2c, K, occlusion_eps, mask=None):
    """mask[i] |= some frame sees point i: sb_tsdf_integrate's projection, then d > 0 and z <= d + occlusion_eps."""
    p = np.asarray(points, f32).reshape(-1, 3)
    depth = np.asarray(depth, f32).reshape(-1, *np.shape(depth)[-2:])
    B, H, W = depth.shape
    w2c = np.asarray(w2c, f32).reshape(B, 4, 4)
    fx, fy, cx, cy = (f32(K[0][0]), f32(K[1][1]), f32(K[0][2]), f32(K[1][2]))
    eps = f32(occlusion_eps)
    out = np.zeros(len(p), np.uint8) if mask is None else np.asarray(mask, np.uint8).copy()
    px, py, pz = p[:, 0], p[:, 1], p[:, 2]
    for b in range(B):
        m = w2c[b]
        x, y, z = [((m[r, 0] * px + m[r, 1] * py) + m[r, 2] * pz) + m[r, 3] for r in range(3)]
        with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
            col = np.floor(((fx * x) / z + cx) + f32(0.5))
            row = np.floor(((fy * y) / z + cy) + f32(0.5))
            ok = (z > 0) & (col >= 0) & (col < W) & (row >= 0) & (row < H)
        ci = np.where(ok, col, 0).astype(np.int64)
        ri = np.where(ok, row, 0).astype(np.int64)
        d = np.where(ok, depth[b][ri, ci], f32(0))
        with np.errstate(invalid="ignore"):
            ok &= (d > 0) & (z <= d + eps)
        out[ok] = 1
    return out


def min_sq_dist(queries, refs, chunk=256):
    """For each query, min over refs of (dx dx + dy dy) + dz dz with dx = qx - px, in float32, in chunks of queries."""
    q = np.asarray(queries, f32).reshape(-1, 3)
    r = np.asarray(refs, f32).reshape(-1, 3)
    out = np.empty(len(q), f32)
    for s in range(0, len(q), chunk):
        qq = q[s:s + chunk]
        dx = qq[:, None, 0] - r[None, :, 0]
        dy = qq[:, None, 1] - r[None, :, 1]
        dz = qq[:, None, 2] - r[None, :, 2]
        out[s:s + chunk] = ((dx * dx + dy * dy) + dz * dz).min(axis=1)
    return out
