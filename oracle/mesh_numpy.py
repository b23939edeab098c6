"""NumPy float32 restatement of csrc/mesh.cu: TSDF integration and marching cubes, operation for operation, so the
kernels can be compared bit for bit.  Every float32 operation below is rounded on its own (numpy does not contract
a * b + c), as the kernels' __fadd_rn / __fmul_rn / __fdiv_rn are.

    integrate(tsdf, weight, color, origin, voxel, trunc, depth [B,H,W], rgb [B,3,H,W], w2c [B,4,4], K, depth_max)
    marching_cubes(tsdf, weight, color, origin, voxel, min_weight) -> vertices [V,3], colors [V,3], faces [F,3]"""
import numpy as np

from splatam_b200 import mc_table

f32 = np.float32


def sample_coords(shape, origin, voxel):
    """Per-axis sample positions o + v * float(idx): x [nx], y [ny], z [nz]."""
    nz, ny, nx = shape
    o = np.asarray(origin, f32)
    v = f32(voxel)
    return [o[a] + v * np.arange(n, dtype=f32) for a, n in enumerate((nx, ny, nz))]


def integrate(tsdf, weight, color, origin, voxel, trunc, depth, rgb, w2c, K, depth_max=None):
    """Fuses frames in order into (tsdf, weight, color) in place: tsdf, weight [nz,ny,nx], color [nz,ny,nx,3]."""
    depth = np.asarray(depth, f32).reshape(-1, *np.shape(depth)[-2:])
    B, H, W = depth.shape
    rgb = np.asarray(rgb, f32).reshape(B, 3, H, W)
    w2c = np.asarray(w2c, f32).reshape(B, 4, 4)
    fx, fy, cx, cy = (f32(K[0][0]), f32(K[1][1]), f32(K[0][2]), f32(K[1][2]))
    tr = f32(trunc)
    dmax = f32(np.inf if depth_max is None else depth_max)
    xs, ys, zs = sample_coords(tsdf.shape, origin, voxel)
    pz, py, px = np.meshgrid(zs, ys, xs, indexing="ij")
    for b in range(B):
        m = w2c[b]
        cam = [((m[r, 0] * px + m[r, 1] * py) + m[r, 2] * pz) + m[r, 3] for r in range(3)]
        x, y, z = cam
        front = z > 0
        with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
            u = (fx * x) / z + cx
            v = (fy * y) / z + cy
            col = np.floor(u + f32(0.5))
            row = np.floor(v + f32(0.5))
        ok = front & (col >= 0) & (col < W) & (row >= 0) & (row < H)
        ci = np.where(ok, col, 0).astype(np.int64)
        ri = np.where(ok, row, 0).astype(np.int64)
        d = np.where(ok, depth[b][ri, ci], f32(0))
        ok &= (d > 0) & (d <= dmax)
        sdf = d - z
        ok &= ~(sdf < -tr)
        f = np.minimum(f32(1), sdf / tr)
        w0 = weight
        w1 = w0 + f32(1)
        t1 = (tsdf * w0 + f) / w1
        c_px = np.stack([rgb[b, c][ri, ci] for c in range(3)], -1)
        c1 = (color * w0[..., None] + c_px) / w1[..., None]
        tsdf[...] = np.where(ok, t1, tsdf)
        color[...] = np.where(ok[..., None], c1, color)
        weight[...] = np.where(ok, w1, weight)
    return tsdf, weight, color


def _shift(a, dz, dy, dx):
    nz, ny, nx = a.shape[:3]
    return a[dz:nz - 1 + dz, dy:ny - 1 + dy, dx:nx - 1 + dx]


def marching_cubes(tsdf, weight, color, origin, voxel, min_weight=1.0):
    """The indexed mesh of csrc/mesh.cu: one vertex per crossed edge used by a live cell, in ascending edge id
    (3 * sample index + axis); faces by ascending cell, then table order; int32 indices."""
    tsdf = np.asarray(tsdf, f32)
    weight = np.asarray(weight, f32)
    color = np.asarray(color, f32)
    nz, ny, nx = tsdf.shape
    empty = (np.zeros((0, 3), f32), np.zeros((0, 3), f32), np.zeros((0, 3), np.int32))
    if min(nz, ny, nx) < 2:
        return empty
    obs = weight >= f32(min_weight)
    inside = tsdf < 0
    live = np.ones((nz - 1, ny - 1, nx - 1), bool)
    case = np.zeros((nz - 1, ny - 1, nx - 1), np.int64)
    for c in range(8):
        dx, dy, dz = c & 1, c >> 1 & 1, c >> 2 & 1
        live &= _shift(obs, dz, dy, dx)
        case |= _shift(inside, dz, dy, dx).astype(np.int64) << c
    # flags[k, j, i, axis]: the edge from sample (i, j, k) along `axis` carries a vertex
    livep = np.zeros((nz + 1, ny + 1, nx + 1), bool)       # livep[k+1, j+1, i+1] = live[k, j, i]
    livep[1:nz, 1:ny, 1:nx] = live
    flags = np.zeros((nz, ny, nx, 3), bool)
    strides = (1, nx, nx * ny)
    for a in range(3):
        sl_a = [slice(None)] * 3
        sl_b = [slice(None)] * 3
        sl_a[2 - a] = slice(0, -1)
        sl_b[2 - a] = slice(1, None)
        crossed = np.zeros((nz, ny, nx), bool)
        crossed[tuple(sl_a)] = inside[tuple(sl_a)] != inside[tuple(sl_b)]
        # cells touching the edge: offsets 0 / -1 on the two other axes
        others = [b for b in range(3) if b != a]
        adj = np.zeros((nz, ny, nx), bool)
        for o0 in (0, 1):
            for o1 in (0, 1):
                off = [1, 1, 1]                               # livep index = cell index + 1
                off[others[0]] -= o0
                off[others[1]] -= o1
                adj |= livep[off[2]:off[2] + nz, off[1]:off[1] + ny, off[0]:off[0] + nx]
        flags[..., a] = crossed & adj
    flat = flags.reshape(-1)
    vid = np.cumsum(flat, dtype=np.int64) - 1
    eid = np.nonzero(flat)[0]
    s, a = eid // 3, eid % 3
    stride = np.array(strides)[a]
    ta, tb = tsdf.reshape(-1)[s], tsdf.reshape(-1)[s + stride]
    t = ta / (ta - tb)
    k, rem = np.divmod(s, nx * ny)
    j, i = np.divmod(rem, nx)
    xs, ys, zs = sample_coords(tsdf.shape, origin, voxel)
    verts = np.stack([xs[i], ys[j], zs[k]], 1)
    rows = np.arange(len(s))
    verts[rows, a] = verts[rows, a] + t * f32(voxel)
    ca, cb = color.reshape(-1, 3)[s], color.reshape(-1, 3)[s + stride]
    cols = ca + t[:, None] * (cb - ca)
    # faces
    cells = np.nonzero(live.reshape(-1))[0]
    cc = case.reshape(-1)[cells]
    ntri = np.array([len(x) for x in mc_table.TRIANGLES])[cc]
    cells, cc, ntri = cells[ntri > 0], cc[ntri > 0], ntri[ntri > 0]
    if len(cells) == 0:
        return verts.astype(f32), cols.astype(f32), np.zeros((0, 3), np.int32)
    ck, crem = np.divmod(cells, (nx - 1) * (ny - 1))
    cj, ci = np.divmod(crem, nx - 1)
    base = (ck * ny + cj) * nx + ci
    table = np.full((256, mc_table.MAX_TRIANGLES, 3), -1, np.int64)
    for c, tris in enumerate(mc_table.TRIANGLES):
        if tris:
            table[c, :len(tris)] = tris
    tri_cell = np.repeat(np.arange(len(cells)), ntri)
    tri_slot = np.arange(len(tri_cell)) - np.repeat(np.cumsum(ntri) - ntri, ntri)
    local = table[cc[tri_cell], tri_slot]                       # [F, 3] local edges
    corner = np.array([c for c, _ in mc_table.EDGES])[local]
    axis = np.array([a for _, a in mc_table.EDGES])[local]
    cs = base[tri_cell][:, None] + (corner & 1) + (corner >> 1 & 1) * nx + (corner >> 2 & 1) * nx * ny
    faces = vid[3 * cs + axis].astype(np.int32)
    return verts.astype(f32), cols.astype(f32), faces
