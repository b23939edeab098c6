"""NumPy float32 restatement of csrc/mesh_render.cu (sb_mesh_depth), operation for operation, so the rasterizer can be
compared bit for bit.  Every float32 operation below is rounded on its own (numpy does not contract a * b + c), as the
kernel's __fadd_rn / __fmul_rn / __fdiv_rn are; np.fmin / np.fmax ignore NaN as fminf / fmaxf do.

    mesh_depth(vertices [V,3], faces [F,3], w2c [B,4,4], K, height, width, near) -> (depth [B,H,W] float32,
                                                                                     face_id [B,H,W] int32)"""
import numpy as np

f32 = np.float32
EMPTY = np.uint64(0xFFFFFFFFFFFFFFFF)
CHUNK = 1 << 21


def _cross_near(P, Q, near):
    """The point on P -> Q at z = near (P inside, Q outside), per row of P, Q [F,3]."""
    s = (near - P[:, 2]) / (Q[:, 2] - P[:, 2])
    return np.stack([P[:, 0] + s * (Q[:, 0] - P[:, 0]), P[:, 1] + s * (Q[:, 1] - P[:, 1]),
                     np.full(len(P), near, f32)], axis=1)


def _pieces(v, f, m, near):
    """Camera-space clipped polygons of every face: (poly [F,4,3], vertex count [F]); count 0 for a dropped face."""
    F = len(f)
    ok = np.all((f >= 0) & (f < len(v)), axis=1)
    p = v[np.where(ok[:, None], f, 0)]                          # [F,3 vertices,3]
    cam = np.stack([((m[r, 0] * p[..., 0] + m[r, 1] * p[..., 1]) + m[r, 2] * p[..., 2]) + m[r, 3]
                    for r in range(3)], axis=-1)
    ok &= np.all(np.isfinite(cam), axis=(1, 2))
    inside = cam[..., 2] >= near
    poly = np.zeros((F, 4, 3), f32)
    cnt = np.zeros(F, np.int64)
    rows = np.arange(F)

    def put(sel, q):
        poly[rows[sel], cnt[sel]] = q[sel]
        cnt[sel] += 1

    for k in range(3):
        P, Q = cam[:, k], cam[:, (k + 1) % 3]
        inP, inQ = inside[:, k], inside[:, (k + 1) % 3]
        put(inP, P)
        put(inP & ~inQ, _cross_near(P, Q, near))
        put(~inP & inQ, _cross_near(Q, P, near))
    cnt[~ok | (cnt < 3)] = 0
    return poly, cnt


def _edge(uP, vP, uQ, vQ, c, r):
    swap = (uQ < uP) | ((uQ == uP) & (vQ < vP))
    u0, v0 = np.where(swap, uQ, uP), np.where(swap, vQ, vP)
    u1, v1 = np.where(swap, uP, uQ), np.where(swap, vP, vQ)
    e = (u1 - u0) * (r - v0) - (v1 - v0) * (c - u0)
    return np.where(swap, -e, e)


def _draw(keys, f_idx, U, Vv, Z, H, W):
    """Tests the clamped bounding-box pixels of the triangles (U, Vv, Z [n,3]) of faces f_idx into keys [H*W]."""
    umin = np.fmin(np.fmin(np.fmin(f32(np.inf), U[:, 0]), U[:, 1]), U[:, 2])
    umax = np.fmax(np.fmax(np.fmax(f32(-np.inf), U[:, 0]), U[:, 1]), U[:, 2])
    vmin = np.fmin(np.fmin(np.fmin(f32(np.inf), Vv[:, 0]), Vv[:, 1]), Vv[:, 2])
    vmax = np.fmax(np.fmax(np.fmax(f32(-np.inf), Vv[:, 0]), Vv[:, 1]), Vv[:, 2])
    c0, c1 = np.fmax(np.ceil(umin), f32(0)), np.fmin(np.floor(umax), f32(W - 1))
    r0, r1 = np.fmax(np.ceil(vmin), f32(0)), np.fmin(np.floor(vmax), f32(H - 1))
    keep = (c0 <= c1) & (r0 <= r1)
    f_idx, U, Vv, Z = f_idx[keep], U[keep], Vv[keep], Z[keep]
    c0, c1, r0, r1 = (a[keep].astype(np.int64) for a in (c0, c1, r0, r1))
    nc, nr = c1 - c0 + 1, r1 - r0 + 1
    n = nc * nr
    start = 0
    while start < len(n):                    # about CHUNK (piece, pixel) pairs at a time
        stop = start + max(1, int(np.searchsorted(np.cumsum(n[start:]), CHUNK, side="right")))
        sl = slice(start, stop)
        _draw_pixels(keys, f_idx[sl], U[sl], Vv[sl], Z[sl], c0[sl], r0[sl], nc[sl], n[sl], W)
        start = stop


def _draw_pixels(keys, f_idx, U, Vv, Z, c0, r0, nc, n, W):
    if n.sum() == 0:
        return
    t = np.repeat(np.arange(len(n)), n)
    k = np.arange(n.sum()) - np.repeat(np.cumsum(n) - n, n)
    ci, ri = c0[t] + k % nc[t], r0[t] + k // nc[t]
    c, r = ci.astype(f32), ri.astype(f32)
    u, v, z = U[t], Vv[t], Z[t]
    ea = _edge(u[:, 1], v[:, 1], u[:, 2], v[:, 2], c, r)
    eb = _edge(u[:, 2], v[:, 2], u[:, 0], v[:, 0], c, r)
    ec = _edge(u[:, 0], v[:, 0], u[:, 1], v[:, 1], c, r)
    s = (ea + eb) + ec
    cov = (((ea >= 0) & (eb >= 0) & (ec >= 0)) | ((ea <= 0) & (eb <= 0) & (ec <= 0))) & (s != 0)
    iz = (((ea / z[:, 0]) + (eb / z[:, 1])) + (ec / z[:, 2])) / s
    zz = f32(1) / iz
    cov &= np.isfinite(zz) & (zz > 0)
    key = (zz[cov].view(np.uint32).astype(np.uint64) << np.uint64(32)) | f_idx[t][cov].astype(np.uint64)
    np.minimum.at(keys, ri[cov] * W + ci[cov], key)


def mesh_depth(vertices, faces, w2c, K, height, width, near=0.01):
    """sb_mesh_depth's rule (include/splatam_b200.h) in float32, one view at a time."""
    v = np.asarray(vertices, f32).reshape(-1, 3)
    f = np.asarray(faces, np.int64).reshape(-1, 3)
    w2c = np.asarray(w2c, f32).reshape(-1, 4, 4)
    fx, fy, cx, cy = (f32(K[0][0]), f32(K[1][1]), f32(K[0][2]), f32(K[1][2]))
    near = f32(near)
    H, W = int(height), int(width)
    B = len(w2c)
    depth = np.zeros((B, H, W), f32)
    face_id = np.full((B, H, W), -1, np.int32)
    with np.errstate(divide="ignore", invalid="ignore", over="ignore", under="ignore"):
        for b in range(B):
            poly, cnt = _pieces(v, f, w2c[b], near)
            u = ((fx * poly[..., 0]) / poly[..., 2]) + cx
            vv = ((fy * poly[..., 1]) / poly[..., 2]) + cy
            keys = np.full(H * W, EMPTY, np.uint64)
            fid = np.arange(len(f))
            for t, sel in ((0, cnt >= 3), (1, cnt == 4)):
                idx = [0, t + 1, t + 2]
                _draw(keys, fid[sel], u[sel][:, idx], vv[sel][:, idx], poly[sel][:, idx, 2], H, W)
            hit = keys != EMPTY
            depth[b].reshape(-1)[hit] = (keys[hit] >> np.uint64(32)).astype(np.uint32).view(f32)
            face_id[b].reshape(-1)[hit] = (keys[hit] & np.uint64(0xFFFFFFFF)).astype(np.int32)
    return depth, face_id
