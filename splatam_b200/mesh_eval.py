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
                  device="cuda", batch=8, cell=None):
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
    pred_samples, gt_samples, gt_samples_kept, and the device times cull_ms, grid_ms and query_ms."""
    dev = _device(device)
    if dev.type != "cuda":
        raise _lib.SplatamB200Error("evaluate_mesh needs a CUDA device (there is no CPU fallback)")
    if not (np.isfinite(threshold) and threshold > 0):
        raise ValueError("threshold must be finite and positive, got %r" % (threshold,))
    if frames is not None and K is None:
        K, frames = _first_intrinsics(frames)
    t_cull, t_grid, t_query = _Timer(), _Timer(), _Timer()
    with torch.cuda.device(dev):
        gen = torch.Generator(dev).manual_seed(int(seed))
        p_pts, _ = sample_surface(*pred, samples, gen, dev)
        g_pts, _ = sample_surface(*gt, samples, gen, dev)
        if frames is not None:
            t_cull.start()
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
    return out
