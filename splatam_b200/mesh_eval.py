"""Scores a reconstructed triangle mesh against the scene's ground-truth mesh, as dense RGB-D SLAM is scored in 3D:

* accuracy     mean distance from the reconstruction to the ground truth (metres)
* completion   mean distance from the ground truth to the reconstruction (metres)
* precision    share of reconstruction samples within `threshold` of the ground truth
* recall       share of ground-truth samples within `threshold` of the reconstruction (the completion ratio)
* fscore       2 P R / (P + R)

Both meshes are sampled by area; the ground-truth samples are culled to what the sequence observed
(``visible_mask``, csrc/mesh_eval.cu: sb_points_visible); distances are exact nearest-neighbour distances between the
two sample sets (``NearestGrid``: sb_nn_grid_build / sb_nn_query, bit-equal to a brute-force minimum).  Both meshes
must already be in the map's frame: ``datasets.SequenceFiles.world_to_map`` moves a dataset's ground-truth mesh there.

``depth_l1`` adds the rendered-depth column of the same table: both meshes are drawn from random viewpoints
(``MeshDepth``: sb_mesh_depth, a z-buffer triangle rasterizer bit-equal to oracle/mesh_render_numpy.py) and their depth
maps compared, which sees floaters in front of the surface and holes that the sample distances miss.
CUDA only; no CPU fallback for the kernels."""
import itertools

import numpy as np
import torch

from . import _lib
from .mesh import _Timer

# the grid holds at most this many cells (the library accepts up to 2^28); a denser default grows its cells
MAX_GRID_CELLS = 1 << 26
POINTS_PER_CELL = 4.0


def _device(device):
    dev = torch.device(device)
    if dev.type == "cuda" and dev.index is None:
        dev = torch.device("cuda", torch.cuda.current_device())
    return dev


def sample_surface(vertices, faces, n, generator=None, device="cuda"):
    """`n` points on the triangle mesh (vertices [V,3], faces [F,3]), uniform over its area: faces are drawn with
    torch.multinomial over their areas (zero-area faces get zero weight) and barycentrics (u, v) uniform in [0, 1)^2,
    reflected to (1 - u, 1 - v) when u + v > 1; p = a + u (b - a) + v (c - a), in float64, returned as float32.
    Returns (points [n,3] float32, face index [n] int64) on `device`.  ValueError for an empty mesh or one whose total
    area is zero (the area sum is read on the host)."""
    dev = _device(device)
    v = torch.as_tensor(vertices).to(dev, torch.float64).reshape(-1, 3)
    f = torch.as_tensor(faces).to(dev, torch.int64).reshape(-1, 3)
    if v.shape[0] == 0 or f.shape[0] == 0:
        raise ValueError("the mesh is empty (%d vertices, %d faces)" % (v.shape[0], f.shape[0]))
    if int(n) != n or n < 1:
        raise ValueError("the sample count must be a positive integer, got %r" % (n,))
    a, b, c = v[f[:, 0]], v[f[:, 1]], v[f[:, 2]]
    area = 0.5 * torch.linalg.vector_norm(torch.linalg.cross(b - a, c - a), dim=1)
    area = torch.nan_to_num(area, nan=0.0, posinf=0.0)
    if not float(area.sum()) > 0:
        raise ValueError("the mesh has zero total area")
    fid = torch.multinomial(area, int(n), replacement=True, generator=generator)
    uv = torch.rand(int(n), 2, dtype=torch.float64, device=dev, generator=generator)
    flip = uv.sum(1) > 1
    uv = torch.where(flip[:, None], 1 - uv, uv)
    a, b, c = a[fid], b[fid], c[fid]
    p = a + uv[:, :1] * (b - a) + uv[:, 1:] * (c - a)
    return p.float().contiguous(), fid


def visible_mask(points, frames, K, occlusion_eps=0.03, batch=8, mask=None):
    """uint8 [N] on the points' device: 1 where some frame sees the point.  frames: an iterable of dicts with depth
    [1,H,W] (or [H,W]) in metres and gt_w2c [4,4] mapping the points' frame to the camera, all at one image size;
    K: 3x3 intrinsics at that size, read on the host.  A point is seen when sb_tsdf_integrate's projection puts it
    inside the image, the depth d there is > 0 and z <= d + occlusion_eps; a non-finite pose sees nothing.  Frames
    are copied into batches of `batch` and each batch is one sb_points_visible launch; the loop issues no host
    synchronisation.  `mask`, when given, is updated in place and returned."""
    pts = torch.as_tensor(points)
    _lib.need_cuda("visible_mask", pts)
    dev = pts.device
    pts = pts.to(torch.float32).reshape(-1, 3).contiguous()
    if int(batch) != batch or batch < 1:
        raise ValueError("batch must be a positive integer, got %r" % (batch,))
    eps = float(occlusion_eps)
    if not (np.isfinite(eps) and eps >= 0):
        raise ValueError("occlusion_eps must be finite and >= 0, got %r" % (occlusion_eps,))
    K = np.asarray(K, dtype=np.float64)
    if mask is None:
        mask = torch.zeros(pts.shape[0], dtype=torch.uint8, device=dev)
    depth_b = w2c_b = None
    n = 0

    def flush(n):
        _lib.call("sb_points_visible", pts.shape[0], pts, n, depth_b.shape[1], depth_b.shape[2], depth_b, w2c_b,
                  float(K[0, 0]), float(K[1, 1]), float(K[0, 2]), float(K[1, 2]), eps, mask, device=dev)

    with torch.cuda.device(dev), torch.no_grad():
        for fr in frames:
            d = torch.as_tensor(fr["depth"])
            if depth_b is None:
                H, W = d.shape[-2:]
                depth_b = torch.empty(int(batch), H, W, dtype=torch.float32, device=dev)
                w2c_b = torch.empty(int(batch), 4, 4, dtype=torch.float32, device=dev)
            if d.numel() != depth_b.shape[1] * depth_b.shape[2]:
                raise ValueError("frames differ in size: %s after %s" % (tuple(d.shape), tuple(depth_b.shape[1:])))
            depth_b[n].copy_(d.reshape(depth_b.shape[1:]), non_blocking=True)
            w2c_b[n].copy_(torch.as_tensor(fr["gt_w2c"]).reshape(4, 4), non_blocking=True)
            n += 1
            if n == batch:
                flush(n)
                n = 0
        if n:
            flush(n)
    return mask


def _grid_geometry(lo, hi, n, cell=None, max_cells=MAX_GRID_CELLS):
    """(origin float32 [3], cell, dims [3]) of a grid over the box [lo, hi] holding n points.  Default cell: about
    POINTS_PER_CELL points per cell if the points lie on surfaces that fill the box's faces, sqrt(k * area / n).  The
    cell count is capped at min(4 n, max_cells): the cell grows until the grid fits."""
    lo, hi = np.asarray(lo, np.float64), np.asarray(hi, np.float64)
    ext = np.maximum(hi - lo, 0.0)
    if cell is None:
        area = 2.0 * (ext[0] * ext[1] + ext[1] * ext[2] + ext[2] * ext[0])
        cell = np.sqrt(POINTS_PER_CELL * area / n) if area > 0 else POINTS_PER_CELL * ext.max() / n
        if not cell > 0:
            cell = 1.0
    cell = float(cell)
    if not (np.isfinite(cell) and cell > 0):
        raise ValueError("the cell size must be finite and positive, got %r" % (cell,))
    cap = min(4 * n + 64, int(max_cells))
    while True:
        cell = float(np.float32(cell))
        dims = np.floor(ext / cell).astype(np.int64) + 1
        total = int(np.prod(dims))
        if total <= cap:
            break
        cell *= max(1.01, (total / cap) ** (1.0 / 3.0))
    return lo.astype(np.float32), cell, dims


class NearestGrid:
    """Exact nearest-neighbour distances to a fixed set of reference points [N,3] (float32, finite, N >= 1) on the
    GPU: a uniform grid over their bounding box with cells of `cell` metres (default ``_grid_geometry``), built
    once (sb_nn_grid_build: cell keys sorted by the project's radix sort, per-cell offsets, coordinates in cell
    order).  The box and a finiteness check are read on the host.  ``query(q)`` returns the squared distances
    [M] float32 from each query to its nearest reference point, bit-equal to a brute-force minimum of
    (dx dx + dy dy) + dz dz."""

    def __init__(self, points, cell=None, max_cells=MAX_GRID_CELLS):
        pts = torch.as_tensor(points)
        _lib.need_cuda("NearestGrid", pts)
        self.device = pts.device
        self.points = pts.to(torch.float32).reshape(-1, 3).contiguous()
        self.n = n = self.points.shape[0]
        if n == 0:
            raise ValueError("NearestGrid needs at least one reference point")
        if n >= 1 << 30:
            raise ValueError("NearestGrid takes fewer than 2^30 points, got %d" % n)
        lo, hi = self.points.aminmax(dim=0)
        lohi = torch.stack([lo, hi]).double().cpu().numpy()
        if not np.all(np.isfinite(lohi)):
            raise ValueError("the reference points must be finite")
        self.origin, self.cell, self.dims = _grid_geometry(lohi[0], lohi[1], n, cell, max_cells)
        gx, gy, gz = (int(d) for d in self.dims)
        with _lib.on_device(self.device):
            nb = _lib.nbytes("sb_nn_grid_workspace_bytes", n, gx, gy, gz)
        self.ws = torch.empty(nb, dtype=torch.uint8, device=self.device)
        _lib.call("sb_nn_grid_build", n, self.points, *self._grid_args(), self.ws, nb, device=self.device)

    def _grid_args(self):
        o = self.origin
        return (float(o[0]), float(o[1]), float(o[2]), self.cell, *(int(d) for d in self.dims))

    def query(self, queries, out=None):
        q = torch.as_tensor(queries)
        _lib.need_cuda("NearestGrid.query", q)
        q = q.to(self.device, torch.float32).reshape(-1, 3).contiguous()
        if out is None:
            out = torch.empty(q.shape[0], dtype=torch.float32, device=self.device)
        _lib.call("sb_nn_query", q.shape[0], q, self.n, *self._grid_args(), self.ws, self.ws.numel(), out,
                  device=self.device)
        return out


def scores(acc_d2, comp_d2, threshold=0.05):
    """The metric from squared distances: acc_d2 [M] from each reconstruction sample to the ground truth, comp_d2
    [N] from each kept ground-truth sample to the reconstruction.  Distances are sqrt(float64(d2)) and every sum is in
    float64; a sample counts as close when its distance is < threshold.  fscore is 0 when precision and recall are."""
    acc = torch.as_tensor(acc_d2).double().sqrt()
    comp = torch.as_tensor(comp_d2).double().sqrt()
    if acc.numel() == 0 or comp.numel() == 0:
        raise ValueError("both sample sets must be non-empty")
    p = float((acc < threshold).double().mean())
    r = float((comp < threshold).double().mean())
    return dict(accuracy=float(acc.mean()), completion=float(comp.mean()), precision=p, recall=r,
                fscore=0.0 if p + r == 0 else 2 * p * r / (p + r))


def _first_intrinsics(frames):
    it = iter(frames)
    first = next(it, None)
    if first is None:
        raise ValueError("frames is empty")
    if "intrinsics" not in first:
        raise ValueError("give K: the frames carry no 'intrinsics'")
    return np.asarray(torch.as_tensor(first["intrinsics"]).cpu(), np.float64)[:3, :3], itertools.chain([first], it)


def evaluate_mesh(pred, gt, frames=None, K=None, samples=200_000, threshold=0.05, occlusion_eps=0.03, seed=0,
                  device="cuda", batch=8, cell=None, depth_views=0):
    """Scores the reconstruction `pred` against the ground truth `gt`, both (vertices [V,3], faces [F,3]) in the
    map's frame.  `samples` points are drawn on each mesh by area (``sample_surface``, one torch.Generator seeded
    with `seed`: the prediction first, then the ground truth).

    With `frames` (an iterable of dicts with depth [1,H,W] and gt_w2c [4,4], e.g. datasets.RGBDSequence; K: their 3x3
    intrinsics, default the first frame's `intrinsics`) only the ground-truth samples some frame observed are kept
    (``visible_mask``); the prediction is never culled, as it exists only where frames were fused.  Culling works on
    the samples, not on the mesh's vertices, so the result does not depend on how finely the ground truth is
    tessellated (evaluations that cull per vertex do).  With frames=None nothing is culled: the mode for a ground
    truth that is already culled.

    Returns a dict: accuracy, completion (metres), precision, recall (the completion ratio), fscore (``scores``),
    pred_samples, gt_samples, gt_samples_kept, and the device times cull_ms, grid_ms and query_ms.

    With depth_views > 0 it also scores rendered depth (``depth_l1`` with views=depth_views and the same frames, K,
    seed and occlusion_eps; the view centres are drawn in the box of the kept ground-truth samples) and adds
    depth_l1, depth_l1_surface (metres), hole_ratio, depth_views_used, depth_views_drawn and the device times
    depth_render_ms and depth_cull_ms.  The frames' depth is then held on the device (``_FrameStack``)."""
    dev = _device(device)
    if dev.type != "cuda":
        raise _lib.SplatamB200Error("evaluate_mesh needs a CUDA device (there is no CPU fallback)")
    if not (np.isfinite(threshold) and threshold > 0):
        raise ValueError("threshold must be finite and positive, got %r" % (threshold,))
    if int(depth_views) != depth_views or depth_views < 0:
        raise ValueError("depth_views must be a non-negative integer, got %r" % (depth_views,))
    if frames is not None and K is None:
        K, frames = _first_intrinsics(frames)
    if depth_views and frames is not None:
        frames = _FrameStack(frames, dev)
    t_cull, t_grid, t_query = _Timer(), _Timer(), _Timer()
    with torch.cuda.device(dev):
        gen = torch.Generator(dev).manual_seed(int(seed))
        p_pts, _ = sample_surface(*pred, samples, gen, dev)
        g_pts, _ = sample_surface(*gt, samples, gen, dev)
        if frames is not None:
            t_cull.start()
            if isinstance(frames, _FrameStack):
                mask = frames.cull(g_pts, K, occlusion_eps)
            else:
                mask = visible_mask(g_pts, frames, K, occlusion_eps, batch)
            t_cull.stop()
            g_kept = g_pts[mask.bool()]
            if g_kept.shape[0] == 0:
                raise ValueError("no ground-truth sample is observed by the frames: check that the meshes are in the "
                                 "map's frame (datasets.SequenceFiles.world_to_map)")
        else:
            g_kept = g_pts
        t_grid.start()
        to_gt = NearestGrid(g_kept, cell)
        t_grid.stop()
        t_query.start()
        acc_d2 = to_gt.query(p_pts)
        t_query.stop()
        t_grid.start()
        to_pred = NearestGrid(p_pts, cell)
        t_grid.stop()
        t_query.start()
        comp_d2 = to_pred.query(g_kept)
        t_query.stop()
        out = scores(acc_d2, comp_d2, threshold)
        torch.cuda.synchronize(dev)
    out.update(pred_samples=int(p_pts.shape[0]), gt_samples=int(g_pts.shape[0]), gt_samples_kept=int(g_kept.shape[0]),
               cull_ms=t_cull.ms() if t_cull.pairs else 0.0, grid_ms=t_grid.ms(), query_ms=t_query.ms())
    if depth_views:
        d = depth_l1(pred, gt, frames, K, views=depth_views, seed=seed, occlusion_eps=occlusion_eps, gt_kept=g_kept,
                     device=dev)
        out.update(depth_l1=d["depth_l1"], depth_l1_surface=d["depth_l1_surface"], hole_ratio=d["hole_ratio"],
                   depth_views_used=d["views_used"], depth_views_drawn=d["views_drawn"],
                   depth_render_ms=d["render_ms"], depth_cull_ms=d["cull_ms"])
    return out


# ---- rendered depth ----------------------------------------------------------------------------------------------
# The random-view protocol (the NICE-SLAM image and intrinsics; the views themselves are this project's own draw).
DEPTH_VIEW_HW = (500, 500)
DEPTH_VIEW_K = np.array([[300.0, 0.0, 249.5], [0.0, 300.0, 249.5], [0.0, 0.0, 1.0]])
DEPTH_VIEW_NEAR = 0.01
CULL_FRAMES_PER_LAUNCH = 32


class MeshDepth:
    """A triangle mesh (vertices [V,3], faces [F,3]) uploaded once to `device` and checked once on the host: face
    indices in [0, V), the vertices that faces use finite in float32, V < 2^31 and F < 2^31 - 1 (ValueError
    otherwise).  ``render(w2c, K, height, width, near)`` draws it from the cameras w2c [B,4,4] (a CUDA tensor; K a
    3x3 on the host) with sb_mesh_depth and returns (depth [B,H,W] float32, 0 where nothing drew, face_id [B,H,W]
    int32, -1 there).  It issues no host synchronisation; the workspace is kept between calls.  CUDA only."""

    def __init__(self, vertices, faces, device="cuda"):
        dev = _device(device)
        if dev.type != "cuda":
            raise _lib.SplatamB200Error("MeshDepth needs a CUDA device (there is no CPU fallback)")
        v = np.asarray(torch.as_tensor(vertices).detach().cpu()).reshape(-1, 3).astype(np.float32)
        f = np.asarray(torch.as_tensor(faces).detach().cpu()).reshape(-1, 3)
        if len(v) == 0 or len(f) == 0:
            raise ValueError("the mesh is empty (%d vertices, %d faces)" % (len(v), len(f)))
        if not np.issubdtype(f.dtype, np.integer):
            raise ValueError("face indices must be integers, got %s" % f.dtype)
        if len(v) >= 1 << 31 or len(f) >= (1 << 31) - 1:
            raise ValueError("MeshDepth takes fewer than 2^31 vertices and 2^31 - 1 faces, got %d and %d"
                             % (len(v), len(f)))
        if f.min() < 0 or f.max() >= len(v):
            raise ValueError("face indices must lie in [0, %d), got [%d, %d]" % (len(v), f.min(), f.max()))
        used = np.zeros(len(v), bool)
        used[f.ravel()] = True
        if not np.all(np.isfinite(v[used])):
            raise ValueError("the vertices that faces use must be finite")
        self.device = dev
        self.vertices = torch.from_numpy(v).to(dev)
        self.faces = torch.from_numpy(f.astype(np.int32)).to(dev)
        self.ws = torch.empty(0, dtype=torch.uint8, device=dev)

    def render(self, w2c, K, height, width, near=DEPTH_VIEW_NEAR, out=None):
        w = torch.as_tensor(w2c)
        _lib.need_cuda("MeshDepth.render", w)
        w = w.to(self.device, torch.float32).reshape(-1, 4, 4).contiguous()
        B, H, W = w.shape[0], int(height), int(width)
        K = np.asarray(K, np.float64)
        V, F = self.vertices.shape[0], self.faces.shape[0]
        with _lib.on_device(self.device):
            nb = _lib.nbytes("sb_mesh_depth_workspace_bytes", F, B, H, W)
        if self.ws.numel() < nb:
            self.ws = torch.empty(nb, dtype=torch.uint8, device=self.device)
        if out is None:
            out = (torch.empty(B, H, W, dtype=torch.float32, device=self.device),
                   torch.empty(B, H, W, dtype=torch.int32, device=self.device))
        depth, face_id = out
        for t, dt in ((depth, torch.float32), (face_id, torch.int32)):
            if t.shape != (B, H, W) or t.dtype != dt or t.device != self.device or not t.is_contiguous():
                raise ValueError("out must be contiguous (float32, int32) tensors [%d,%d,%d] on %s"
                                 % (B, H, W, self.device))
        _lib.call("sb_mesh_depth", V, self.vertices, F, self.faces, B, H, W, w, float(K[0, 0]), float(K[1, 1]),
                  float(K[0, 2]), float(K[1, 2]), float(near), self.ws, self.ws.numel(), depth, face_id,
                  device=self.device)
        return depth, face_id


def depth_views(gt_kept, n, seed=0):
    """n random cameras w2c [n,4,4] float32 (numpy) for ``depth_l1``, one view at a time from one
    numpy.random.Generator(seed) in float64, so the first k of n views do not depend on n:

    * centre: uniform in the axis-aligned box of the points gt_kept [N,3] (the kept ground-truth samples)
    * direction (the camera's +z): uniform on the sphere, drawn again while it lies within 0.99 of +-y
    * no roll: the camera's x axis is y_map x z_cam, normalised (perpendicular to the map's y axis, the first
      camera's "down"), and its y axis z_cam x x_cam"""
    p = torch.as_tensor(gt_kept).reshape(-1, 3)
    if p.shape[0] == 0:
        raise ValueError("depth_views needs at least one point to bound the view centres")
    lo, hi = torch.stack(p.double().aminmax(dim=0)).cpu().numpy()
    if not (np.all(np.isfinite(lo)) and np.all(np.isfinite(hi))):
        raise ValueError("the points bounding the view centres must be finite")
    if int(n) != n or n < 0:
        raise ValueError("the view count must be a non-negative integer, got %r" % (n,))
    rng = np.random.default_rng(int(seed))
    out = np.tile(np.eye(4, dtype=np.float32), (int(n), 1, 1))
    for i in range(int(n)):
        c = lo + (hi - lo) * rng.random(3)
        while True:
            d = rng.standard_normal(3)
            norm = np.linalg.norm(d)
            if norm > 0 and abs(d[1] / norm) < 0.99:
                break
        z = d / norm
        x = np.cross([0.0, 1.0, 0.0], z)
        x /= np.linalg.norm(x)
        R = np.stack([x, np.cross(z, x), z])
        out[i, :3, :3] = R
        out[i, :3, 3] = -R @ c
    return out


class _FrameStack:
    """The frames' depth and gt_w2c (dicts as ``visible_mask`` takes) copied once to the device in chunks of
    CULL_FRAMES_PER_LAUNCH, for culling many point sets against the same frames.  Holds T H W float32 on the device."""

    def __init__(self, frames, dev):
        self.device = dev
        self.chunks = []
        ds, ws, hw = [], [], None
        for fr in frames:
            d = torch.as_tensor(fr["depth"]).to(dev, torch.float32)
            hw = hw or tuple(d.shape[-2:])
            if d.numel() != hw[0] * hw[1]:
                raise ValueError("frames differ in size: %s after %s" % (tuple(d.shape), hw))
            ds.append(d.reshape(hw))
            ws.append(torch.as_tensor(fr["gt_w2c"]).to(dev, torch.float32).reshape(4, 4))
            if len(ds) == CULL_FRAMES_PER_LAUNCH:
                self.chunks.append((torch.stack(ds), torch.stack(ws)))
                ds, ws = [], []
        if ds:
            self.chunks.append((torch.stack(ds), torch.stack(ws)))
        if not self.chunks:
            raise ValueError("frames is empty")

    def cull(self, points, K, occlusion_eps, mask=None):
        """visible_mask's result for points [N,3] on the device: one sb_points_visible launch per chunk."""
        eps = float(occlusion_eps)
        if not (np.isfinite(eps) and eps >= 0):
            raise ValueError("occlusion_eps must be finite and >= 0, got %r" % (occlusion_eps,))
        pts = points.to(self.device, torch.float32).reshape(-1, 3).contiguous()
        if mask is None:
            mask = torch.zeros(pts.shape[0], dtype=torch.uint8, device=self.device)
        K = np.asarray(K, np.float64)
        for d, w in self.chunks:
            _lib.call("sb_points_visible", pts.shape[0], pts, d.shape[0], d.shape[1], d.shape[2], d, w,
                      float(K[0, 0]), float(K[1, 1]), float(K[0, 2]), float(K[1, 2]), eps, mask, device=self.device)
        return mask


def backproject(depth, w2c, K):
    """The points [B,H,W,3] (float32, map frame) that depth [B,H,W] puts on the pixel centres of cameras w2c
    [B,4,4] with intrinsics K: camera (x, y, z) = ((c - cx) d / fx, (r - cy) d / fy, d), then R^T (p - t)."""
    B, H, W = depth.shape
    K = np.asarray(K, np.float64)
    dev = depth.device
    c = (torch.arange(W, device=dev, dtype=torch.float32) - float(K[0, 2])) / float(K[0, 0])
    r = (torch.arange(H, device=dev, dtype=torch.float32) - float(K[1, 2])) / float(K[1, 1])
    cam = torch.stack([c[None, None, :] * depth, r[None, :, None] * depth, depth], dim=-1)
    R, t = w2c[:, :3, :3], w2c[:, :3, 3]
    return (cam - t[:, None, None, :]) @ R[:, None]


def depth_sums(d_pred, d_gt, scored):
    """Per-view float64 sums [B,4] of depth maps [B,H,W] over their scored pixels (bool [B,H,W]): the scored pixel
    count, the sum of |d_pred - d_gt| (a hole, d_pred = 0, costs d_gt), the count of scored pixels where the
    prediction has a surface (d_pred > 0) and the sum of |d_pred - d_gt| over those."""
    sc = scored.double()
    err = (d_pred.double() - d_gt.double()).abs() * sc
    surf = sc * (d_pred > 0).double()
    return torch.stack([sc.sum((1, 2)), err.sum((1, 2)), surf.sum((1, 2)), (err * surf).sum((1, 2))], dim=1)


def depth_scores(sums, pixels, views):
    """The metric from per-view sums [n,4] (``depth_sums``, read on the host) of views with `pixels` pixels each: a
    view is accepted when at least half its pixels are scored, in order, up to `views` of them.  depth_l1 is the mean
    over accepted views of the view's mean |d_pred - d_gt|; depth_l1_surface the same over the pixels with a predicted
    surface (over the accepted views that have any; NaN if none has); hole_ratio the share of all accepted scored
    pixels without a predicted surface.  ValueError when no view is accepted."""
    s = np.asarray(sums, np.float64).reshape(-1, 4)
    acc = s[s[:, 0] >= 0.5 * pixels][:int(views)]
    if len(acc) == 0:
        raise ValueError("no view had at least half its pixels on an observed ground-truth surface: check that the "
                         "meshes are in the map's frame (datasets.SequenceFiles.world_to_map)")
    has = acc[:, 2] > 0
    return dict(depth_l1=float(np.mean(acc[:, 1] / acc[:, 0])),
                depth_l1_surface=float(np.mean(acc[has, 3] / acc[has, 2])) if has.any() else float("nan"),
                hole_ratio=float(1.0 - acc[:, 2].sum() / acc[:, 0].sum()), views_used=len(acc))


def depth_l1(pred, gt, frames=None, K=None, views=1000, seed=0, occlusion_eps=0.03, batch=8, *, gt_kept=None,
             device="cuda"):
    """Scores the reconstruction `pred` against the ground truth `gt` (both (vertices [V,3], faces [F,3]) in the
    map's frame) by rendered depth, from ``depth_views`` cameras at DEPTH_VIEW_HW with DEPTH_VIEW_K and near
    DEPTH_VIEW_NEAR.  Views are drawn `batch` at a time and each batch is rendered once per mesh (``MeshDepth``).

    A view's scored pixels are those where the ground-truth render has a surface; with `frames` (as for
    ``evaluate_mesh``; K their intrinsics, default the first frame's) only those whose surface point -- the pixel
    back-projected at the ground-truth depth -- some frame observed, by ``visible_mask``'s rule with
    `occlusion_eps` (sb_points_visible; the frames' depth is held on the device).  The host reads the per-view sums
    once per batch; drawing stops after `views` accepted views (``depth_scores``) or 20 views draws.

    gt_kept: the points whose box holds the view centres; default 200,000 area samples of `gt` (torch.Generator
    seeded with `seed`), culled by `frames`.  Returns depth_l1, depth_l1_surface (metres), hole_ratio, views_used,
    views_drawn, and the device times render_ms and cull_ms."""
    dev = _device(device)
    if dev.type != "cuda":
        raise _lib.SplatamB200Error("depth_l1 needs a CUDA device (there is no CPU fallback)")
    if int(views) != views or views < 1:
        raise ValueError("views must be a positive integer, got %r" % (views,))
    if int(batch) != batch or batch < 1:
        raise ValueError("batch must be a positive integer, got %r" % (batch,))
    if not (np.isfinite(occlusion_eps) and occlusion_eps >= 0):
        raise ValueError("occlusion_eps must be finite and >= 0, got %r" % (occlusion_eps,))
    if frames is not None and K is None and not isinstance(frames, _FrameStack):
        K, frames = _first_intrinsics(frames)
    H, W = DEPTH_VIEW_HW
    t_render, t_cull = _Timer(), _Timer()
    with torch.cuda.device(dev):
        if frames is not None and not isinstance(frames, _FrameStack):
            frames = _FrameStack(frames, dev)
        g_mesh, p_mesh = MeshDepth(*gt, dev), MeshDepth(*pred, dev)
        if gt_kept is None:
            gen = torch.Generator(dev).manual_seed(int(seed))
            gt_kept, _ = sample_surface(*gt, 200_000, gen, dev)
            if frames is not None:
                gt_kept = gt_kept[frames.cull(gt_kept, K, occlusion_eps).bool()]
        cams = torch.from_numpy(depth_views(gt_kept, 20 * int(views), seed)).to(dev)
        bufs = None
        sums, drawn, used = [], 0, 0
        while used < views and drawn < cams.shape[0]:
            nb = min(int(batch), cams.shape[0] - drawn)
            w = cams[drawn:drawn + nb]
            t_render.start()
            d_gt, _ = g_mesh.render(w, DEPTH_VIEW_K, H, W)
            d_pred, _ = p_mesh.render(w, DEPTH_VIEW_K, H, W)
            t_render.stop()
            scored = d_gt > 0
            if frames is not None:
                t_cull.start()
                pts = backproject(d_gt, w, DEPTH_VIEW_K)
                if bufs is None or bufs.numel() != nb * H * W:
                    bufs = torch.empty(nb * H * W, dtype=torch.uint8, device=dev)
                bufs.zero_()
                frames.cull(pts, K, occlusion_eps, bufs)
                scored &= bufs.view(nb, H, W).bool()
                t_cull.stop()
            s = depth_sums(d_pred, d_gt, scored).cpu().numpy()
            drawn += nb
            sums.append(s)
            used += int((s[:, 0] >= 0.5 * H * W).sum())
        out = depth_scores(np.concatenate(sums), H * W, views)
        torch.cuda.synchronize(dev)
    out.update(views_drawn=drawn, render_ms=t_render.ms(), cull_ms=t_cull.ms() if t_cull.pairs else 0.0)
    return out
