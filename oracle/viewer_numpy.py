"""Float32 numpy restatement of csrc/viewer.cu (sb_viewer_compose, sb_viewer_points, sb_viewer_lines), in the
kernels' operation order, so the GPU tests can ask for bit-equal frames.  Every elementwise float32 operation of numpy
is IEEE round-to-nearest, as the kernels' __fmul_rn / __fdiv_rn / __fadd_rn are."""
import numpy as np

F = np.float32
NO_KEY = np.uint64(0xFFFFFFFFFFFFFFFF)


def rgb_u8(x):
    """round_half_even(clamp(x, 0, 1) * 255f), NaN -> 0."""
    x = np.asarray(x, F)
    c = np.minimum(np.maximum(x, F(0)), F(1))
    c[np.isnan(x)] = 0
    return np.rint(c * F(255)).astype(np.uint8)


def compose(color, depth, sil, mode, s, lut):
    """color [3,h,w], depth [h,w], sil [h,w] or None, mode 0/1/2 -> (out [h*s, w*s, 3] uint8, zbuf [h*s, w*s])."""
    depth = np.asarray(depth, F)
    h, w = depth.shape
    fg = depth > 0
    white = ~fg
    if mode == 0:
        px = np.stack([rgb_u8(c) for c in np.asarray(color, F)], -1)
    elif mode == 1:
        sel = fg & (depth < F(15))
        vmax = F(depth[sel].max()) if sel.any() else F(0)
        with np.errstate(divide="ignore", invalid="ignore"):
            x = (depth / vmax) * F(256) if vmax > 0 else np.zeros_like(depth)
        idx = np.where(x >= F(256), 255, np.nan_to_num(x, nan=0.0, posinf=255.0)).astype(np.int64)
        idx = np.clip(idx, 0, 255)
        px = lut[idx]
        white = white | ~(depth < F(15))
    else:
        g = rgb_u8(F(1) - np.asarray(sil, F))
        px = np.stack([g, g, g], -1)
    px = px.copy()
    px[white] = 255
    z = np.where(fg, depth, F(np.inf)).astype(F)
    up = lambda a: np.repeat(np.repeat(a, s, axis=0), s, axis=1)
    return np.ascontiguousarray(up(px)), np.ascontiguousarray(up(z))


def to_camera(w2c, p):
    """p [N,3] float32 -> camera coordinates [N,3], ((r0 x + r1 y) + r2 z) + t per row."""
    m = np.asarray(w2c, F).reshape(4, 4)
    p = np.asarray(p, F)
    return np.stack([((m[r, 0] * p[:, 0] + m[r, 1] * p[:, 1]) + m[r, 2] * p[:, 2]) + m[r, 3] for r in range(3)], -1)


def _project(c, fx, fy, cx, cy):
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        u = (F(fx) * c[:, 0]) / c[:, 2] + F(cx)
        v = (F(fy) * c[:, 1]) / c[:, 2] + F(cy)
    return u, v


def points(means, colors, timestep, t_max, w2c, k, W, H, s, near, far):
    """Centre splat: k = (fx, fy, cx, cy) at output size.  Returns (out [H,W,3] uint8, zbuf [H,W])."""
    means = np.asarray(means, F)
    keys = np.full(H * W, NO_KEY, np.uint64)
    if len(means):
        c = to_camera(w2c, means)
        u, v = _project(c, *k)
        ok = (c[:, 2] > F(near)) & (c[:, 2] < F(far)) & np.isfinite(u) & np.isfinite(v)
        if timestep is not None:
            ok &= np.asarray(timestep, F) <= F(t_max)
        x0, y0 = np.floor(u + F(0.5)), np.floor(v + F(0.5))
        ok &= ~((x0 >= W) | (y0 >= H) | (x0 + s <= 0) | (y0 + s <= 0))
        idx = np.nonzero(ok)[0]
        key = (c[idx, 2].view(np.uint32).astype(np.uint64) << np.uint64(32)) | idx.astype(np.uint64)
        x0, y0 = x0[idx].astype(np.int64), y0[idx].astype(np.int64)
        for dy in range(s):
            for dx in range(s):
                x, y = x0 + dx, y0 + dy
                inb = (x >= 0) & (x < W) & (y >= 0) & (y < H)
                np.minimum.at(keys, y[inb] * W + x[inb], key[inb])
    out = np.full((H * W, 3), 255, np.uint8)
    z = np.full(H * W, np.inf, F)
    hit = keys != NO_KEY
    i = (keys[hit] & np.uint64(0xFFFFFFFF)).astype(np.int64)
    out[hit] = rgb_u8(np.asarray(colors, F)[i])
    z[hit] = (keys[hit] >> np.uint64(32)).astype(np.uint32).view(F)
    return out.reshape(H, W, 3), z.reshape(H, W)


def lines(segments, colors, w2c, k, W, H, near, zbuf, out):
    """Draws segments [S,6] with uint8 colors [S,3] over a copy of out [H,W,3], depth-tested against zbuf [H,W]."""
    fx, fy, cx, cy = (F(a) for a in k)
    near = F(near)
    segments = np.asarray(segments, F).reshape(-1, 6)
    zb = np.asarray(zbuf, F).reshape(-1)
    keys = np.full(H * W, NO_KEY, np.uint64)
    for j, e in enumerate(segments):
        a = to_camera(w2c, e[None, :3])[0]
        b = to_camera(w2c, e[None, 3:])[0]
        if not (a[2] > near) and not (b[2] > near):
            continue
        if not (a[2] > near) or not (b[2] > near):
            if not (a[2] > near):
                a, b = b, a
            f = (near - a[2]) / (b[2] - a[2])
            b = np.array([a[0] + f * (b[0] - a[0]), a[1] + f * (b[1] - a[1]), near], F)
        with np.errstate(all="ignore"):
            u0, v0 = (fx * a[0]) / a[2] + cx, (fy * a[1]) / a[2] + cy
            u1, v1 = (fx * b[0]) / b[2] + cx, (fy * b[1]) / b[2] + cy
        if not all(np.isfinite([u0, v0, u1, v1])):
            continue
        du, dv = u1 - u0, v1 - v0
        if du == 0 and dv == 0:
            continue
        xmajor = abs(du) >= abs(dv)
        p0, p1, q0 = (u0, u1, v0) if xmajor else (v0, v1, u0)
        dp, dq = (du, dv) if xmajor else (dv, du)
        nmaj, nmin = (W, H) if xmajor else (H, W)
        lo = max(np.ceil(min(p0, p1) - F(0.5)), F(0))
        hi = min(np.floor(max(p0, p1) - F(0.5)), F(nmaj - 1))
        if lo > hi:
            continue
        iz0, iz1 = F(1) / a[2], F(1) / b[2]
        c = np.arange(int(lo), int(hi) + 1)
        t = ((c.astype(F) + F(0.5)) - p0) / dp
        r = np.floor(q0 + t * dq)
        ok = (r >= 0) & (r < nmin)
        c, t, r = c[ok], t[ok], r[ok].astype(np.int64)
        X, Y = (c, r) if xmajor else (r, c)
        z = F(1) / ((F(1) - t) * iz0 + t * iz1)
        q = Y * W + X
        vis = z < zb[q]
        key = (z[vis].view(np.uint32).astype(np.uint64) << np.uint64(32)) | np.uint64(j)
        np.minimum.at(keys, q[vis], key)
    res = np.array(out, np.uint8).reshape(H * W, 3).copy()
    hit = keys != NO_KEY
    res[hit] = np.asarray(colors, np.uint8)[(keys[hit] & np.uint64(0xFFFFFFFF)).astype(np.int64)]
    return res.reshape(H, W, 3)
