"""A coloured triangle mesh from a SplaTAM map: the map's depth, rendered at the tracked poses, fused into a truncated
signed distance field (TSDF) and meshed by marching cubes, both on the GPU (csrc/mesh.cu).

* ``TSDFVolume``   a dense volume: ``integrate`` fuses depth/colour frames, ``extract`` returns the indexed mesh
* ``mesh_record``  meshes a saved run record (viewer.load_record: this project's, the reference's and the offline
                   `params.npz`) from the renders the evaluation makes, or from any frames given as `source`

The mesh is in the map's frame (that of `means3D` and `splat.ply`); its triangles face free space.  Write it with
``formats.save_mesh_ply``.  CUDA only; no CPU fallback."""
import numpy as np
import torch

from . import _lib
from . import datasets as D
from . import formats
from . import mapping as M
from . import mc_table

MAX_VOXELS = 500_000_000
# marching cubes packs each sample's triangle count (<= MAX_TRIANGLES) and vertex count (<= 3) into the two 32-bit
# halves of one scanned uint64, so a volume may hold at most this many samples (sb_mc_* reject larger grids)
MC_MAX_SAMPLES = (2 ** 32 - 1) // mc_table.MAX_TRIANGLES


def _grid(lo, hi, voxel):
    origin = np.floor(lo / voxel) * voxel
    dims = np.ceil((hi - origin) / voxel - 1e-6).astype(np.int64) + 1     # the last sample at or past hi
    return origin, dims


class TSDFVolume:
    """A dense TSDF volume over the axis-aligned box `bounds` = (x0, y0, z0, x1, y1, z1) (or [[x0, y0, z0],
    [x1, y1, z1]]) with cubic voxels of `voxel_size` metres and truncation `trunc` (default 4 voxels).  The origin is
    snapped down to a multiple of the voxel size and the grid covers the box.  State, on `device`: tsdf, weight
    [nz,ny,nx] (x fastest) and color [nz,ny,nx,3], float32, starting at T = 1, W = 0, C = 0.  A volume of more than
    `max_voxels` voxels raises ValueError naming its voxel count and a voxel size that would fit; `max_voxels` is
    capped at MC_MAX_SAMPLES, the largest grid marching cubes accepts."""

    def __init__(self, bounds, voxel_size, trunc=None, device="cuda", max_voxels=MAX_VOXELS):
        b = np.asarray(bounds, dtype=np.float64).reshape(-1)
        if b.shape != (6,) or not np.all(np.isfinite(b)):
            raise ValueError("bounds must be 6 finite numbers (x0, y0, z0, x1, y1, z1), got %r" % (bounds,))
        lo, hi = b[:3], b[3:]
        if np.any(hi < lo):
            raise ValueError("bounds need x0 <= x1, y0 <= y1, z0 <= z1, got %r" % (bounds,))
        v = float(voxel_size)
        if not (np.isfinite(v) and v > 0):
            raise ValueError("voxel_size must be finite and positive, got %r" % (voxel_size,))
        t = 4.0 * v if trunc is None else float(trunc)
        if not (np.isfinite(t) and t > 0):
            raise ValueError("trunc must be finite and positive, got %r" % (trunc,))
        max_voxels = min(int(max_voxels), MC_MAX_SAMPLES)
        origin, dims = _grid(lo, hi, v)
        n = int(np.prod(dims))
        if n > max_voxels:
            fit = v * (n / max_voxels) ** (1.0 / 3.0)
            while int(np.prod(_grid(lo, hi, fit)[1])) > max_voxels:
                fit *= 1.01
            raise ValueError("a %.6g m voxel grid over these bounds needs %d voxels (%d x %d x %d), more than "
                             "max_voxels = %d; a voxel size of %.4g m would fit"
                             % (v, n, dims[0], dims[1], dims[2], max_voxels, fit))
        self.device = torch.device(device)
        if self.device.type == "cuda" and self.device.index is None:
            self.device = torch.device("cuda", torch.cuda.current_device())
        self.voxel_size, self.trunc = np.float32(v), np.float32(t)
        self.origin = origin.astype(np.float32)
        self.nx, self.ny, self.nz = (int(d) for d in dims)
        shape = (self.nz, self.ny, self.nx)
        self.tsdf = torch.ones(shape, dtype=torch.float32, device=self.device)
        self.weight = torch.zeros(shape, dtype=torch.float32, device=self.device)
        self.color = torch.zeros(shape + (3,), dtype=torch.float32, device=self.device)
        self._ws = None
        self._totals = torch.zeros(2, dtype=torch.int32, device=self.device)

    @property
    def num_voxels(self):
        return self.nx * self.ny * self.nz

    def integrate(self, depth, color, K, w2c, depth_max=None):
        """Fuses one frame -- depth [H,W] or [1,H,W] (metres, 0 = no measurement), color [3,H,W], w2c [4,4] -- or a
        batch -- depth [B,H,W] or [B,1,H,W], color [B,3,H,W], w2c [B,4,4] -- in order (sb_tsdf_integrate).  K: the
        3x3 pinhole intrinsics, read on the host; a pixel's centre is at its integer coordinates.  depth_max: depth
        beyond it is ignored.  Enqueues one launch on the current stream; no host synchronisation."""
        dev = self.device
        c = lambda x: torch.as_tensor(x).to(dev, torch.float32).contiguous()
        depth, color, w2c = c(depth), c(color), c(w2c)
        _lib.need_cuda("TSDFVolume.integrate", self.tsdf)
        if color.dim() == 3:
            depth, color, w2c = depth.reshape(1, *depth.shape[-2:]), color[None], w2c.reshape(1, 4, 4)
        if color.dim() != 4 or color.shape[1] != 3:
            raise ValueError("color must be [3,H,W] or [B,3,H,W], got %s" % (tuple(color.shape),))
        B, _, H, W = color.shape
        if depth.numel() != B * H * W or tuple(depth.shape[-2:]) != (H, W) or w2c.shape != (B, 4, 4):
            raise ValueError("depth %s and w2c %s do not match color %s" % (tuple(depth.shape), tuple(w2c.shape),
                                                                          tuple(color.shape)))
        K = np.asarray(K, dtype=np.float64)
        dmax = np.inf if depth_max is None else float(depth_max)
        if not dmax > 0:
            raise ValueError("depth_max must be positive, got %r" % (depth_max,))
        o, v = self.origin, self.voxel_size
        _lib.call("sb_tsdf_integrate", self.nx, self.ny, self.nz, float(o[0]), float(o[1]), float(o[2]), float(v),
                  float(self.trunc), B, H, W, depth, color, w2c, float(K[0, 0]), float(K[1, 1]), float(K[0, 2]),
                  float(K[1, 2]), dmax, self.tsdf, self.weight, self.color, device=dev)

    def extract(self, min_weight=1.0):
        """Marching cubes over the cells whose 8 samples have weight >= min_weight: (vertices [V,3] float32,
        colors [V,3] float32, faces [F,3] int32) on the device.  Reads the two counts on the host (the one
        synchronisation); an empty or fully inside volume gives empty arrays."""
        dev = self.device
        _lib.need_cuda("TSDFVolume.extract", self.tsdf)
        if self._ws is None:
            with _lib.on_device(dev):            # the scan's temporary size is queried for this device
                nb = _lib.nbytes("sb_mc_workspace_bytes", self.nx, self.ny, self.nz)
            self._ws = torch.empty(nb, dtype=torch.uint8, device=dev)
        _lib.call("sb_mc_count", self.nx, self.ny, self.nz, self.tsdf, self.weight, float(min_weight), self._ws,
                  self._ws.numel(), self._totals, device=dev)
        nv, nf = (int(x) for x in self._totals.cpu())
        if nv < 0 or nf < 0:
            raise _lib.SplatamB200Error("the mesh has more than %d vertices or faces" % ((2 ** 31 - 1) // 3))
        verts = torch.empty(nv, 3, dtype=torch.float32, device=dev)
        cols = torch.empty(nv, 3, dtype=torch.float32, device=dev)
        faces = torch.empty(nf, 3, dtype=torch.int32, device=dev)
        o, v = self.origin, self.voxel_size
        _lib.call("sb_mc_emit", self.nx, self.ny, self.nz, float(o[0]), float(o[1]), float(o[2]), float(v), self.tsdf,
                  self.color, self._ws, self._ws.numel(), verts, cols, faces, device=dev)
        return verts, cols, faces


def default_bounds(means3D, trunc):
    """Per-axis 0.1 % / 99.9 % quantiles of the Gaussian centres [P,3] (host), padded by 2 trunc."""
    m = np.asarray(means3D, dtype=np.float64)
    lo, hi = np.quantile(m, 0.001, axis=0), np.quantile(m, 0.999, axis=0)
    return np.concatenate([lo - 2 * trunc, hi + 2 * trunc])


class _Timer:
    """Device time of the enqueued work between start() and stop(), summed over intervals and read once."""

    def __init__(self):
        self.pairs = []

    def start(self):
        e = torch.cuda.Event(enable_timing=True)
        e.record()
        self.pairs.append([e, None])

    def stop(self):
        e = torch.cuda.Event(enable_timing=True)
        e.record()
        self.pairs[-1][1] = e

    def ms(self):
        return sum(a.elapsed_time(b) for a, b in self.pairs)


class RecordFusion:
    """The fusion of one run record (mesh_record's loop), set up once: the record, read and checked as
    viewer.load_record reads it (formats.read_record), its Gaussians and cameras on `device`, the poses of the frames
    t = 0, every, 2 every, ... and the batch buffers.  ``fuse(vol)`` renders or reads those frames and integrates them
    into `vol`, with no host synchronisation.  `source`, when given, must hold exactly one frame per camera of the
    record (frame t is fused at the record's pose t): ValueError otherwise."""

    def __init__(self, path, every=1, sil_thres=0.99, depth_max=None, batch=8, device="cuda", source=None,
                 camera=None):
        if int(every) != every or every < 1:
            raise ValueError("every must be a positive integer, got %r" % (every,))
        if int(batch) != batch or batch < 1:
            raise ValueError("batch must be a positive integer, got %r" % (batch,))
        dev = torch.device(device)
        if dev.type == "cuda" and dev.index is None:
            dev = torch.device("cuda", torch.cuda.current_device())
        self.device, self.sil_thres, self.depth_max, self.source = dev, float(sil_thres), depth_max, source
        raw = formats.read_record(path, formats.CHECKPOINT_KEYS + formats.CAMERA_KEYS, camera)
        T = np.asarray(raw["cam_unnorm_rots"]).shape[-1]
        if source is not None and len(source) != T:
            raise ValueError("%s has %d cameras but the source has %d frames: frame t is fused at the record's pose "
                             "t, so the source must select the run's frames (start, end, stride, frame cap)"
                             % (path, T, len(source)))
        self.means_host = np.asarray(raw["means3D"], np.float32)
        self.w, self.h = w, h = int(raw["org_width"]), int(raw["org_height"])
        self.K = np.array(raw["intrinsics"], np.float32)[:3, :3]
        first_w2c = np.array(raw["w2c"], np.float32).reshape(4, 4)
        self.ids = list(range(0, T, int(every)))
        with torch.cuda.device(dev), torch.no_grad():
            self.params = formats.record_tensors(raw, formats.CHECKPOINT_KEYS, dev)
            self.cam = D.setup_camera(w, h, self.K, first_w2c, dev)
            self.w2c0 = torch.from_numpy(first_w2c).to(dev)
            self.poses = [M.pose_matrices(self.params, t) for t in self.ids]
            # the render projects w2c0 @ rel_w2c(t) @ p: the fusion uses the same camera
            self.w2cs = torch.stack([self.w2c0 @ rel for rel, _ in self.poses]).contiguous()
            self.B = B = min(int(batch), len(self.ids))
            self.depth_b = torch.empty(B, h, w, dtype=torch.float32, device=dev)
            self.rgb_b = torch.empty(B, 3, h, w, dtype=torch.float32, device=dev)
            self.zero = torch.zeros((), dtype=torch.float32, device=dev)
        self.t_render, self.t_fuse = _Timer(), _Timer()

    def _frame_into(self, q, k):
        """Frame ids[k]'s depth and colour into batch slot q."""
        if self.source is None:
            fr = dict(id=self.ids[k], cam=self.cam, w2c=self.w2c0, pose=self.poses[k])
            with torch.no_grad():
                im, depth_sil, _, _ = M._render_pair(self.params, fr, M.default_render, True, camera_grad=False)
            d, sil = depth_sil[0], depth_sil[1]
            torch.where(sil > self.sil_thres, d / sil, self.zero, out=self.depth_b[q])
            self.rgb_b[q].copy_(im)
        else:
            fr = self.source[self.ids[k]]
            self.depth_b[q].copy_(fr["depth"].reshape(self.h, self.w))
            self.rgb_b[q].copy_(fr["im"])

    def fuse(self, vol):
        with torch.cuda.device(self.device), torch.no_grad():
            for b0 in range(0, len(self.ids), self.B):
                n = min(self.B, len(self.ids) - b0)
                self.t_render.start()
                for q in range(n):
                    self._frame_into(q, b0 + q)
                self.t_render.stop()
                self.t_fuse.start()
                vol.integrate(self.depth_b[:n], self.rgb_b[:n], self.K, self.w2cs[b0:b0 + n], self.depth_max)
                self.t_fuse.stop()
        return vol


def mesh_record(path, voxel_size, every=1, sil_thres=0.99, depth_max=None, bounds=None, batch=8, trunc=None,
                min_weight=1.0, device="cuda", source=None, max_voxels=MAX_VOXELS, camera=None):
    """Meshes a saved run record.  For every `every`-th estimated pose t the final map is rendered at the record's
    camera (intrinsics at org_width x org_height) with the evaluation's fused colour plus depth/silhouette render,
    and depth = depth_acc / sil on pixels with sil > sil_thres (0 elsewhere) is fused with the rendered colour, in
    batches of `batch` frames.  With `source` (a sequence of frame dicts with `im` [3,H,W] and `depth` [1,H,W], e.g.
    datasets.RGBDSequence at the record's image size) frame t's own colour and depth are fused instead.  bounds:
    (x0, y0, z0, x1, y1, z1); default the 0.1 % / 99.9 % quantiles of means3D per axis, padded by 2 trunc.  camera:
    as for viewer.load_record.  With `source`, len(source) must equal the record's camera count.  The
    render-and-integrate loop issues no host synchronisation (RecordFusion).  Returns (vertices, colors, faces, info): the mesh on the device in the map's frame, and info = dict(voxels, dims,
    origin, voxel_size, trunc, frames, render_ms, integrate_ms, extract_ms), the last three device times."""
    rf = RecordFusion(path, every, sil_thres, depth_max, batch, device, source, camera)
    tr = 4.0 * float(voxel_size) if trunc is None else float(trunc)
    if bounds is None:
        bounds = default_bounds(rf.means_host, tr)
    vol = TSDFVolume(bounds, voxel_size, tr, rf.device, max_voxels)
    rf.fuse(vol)
    t_extract = _Timer()
    with torch.cuda.device(rf.device):
        t_extract.start()
        verts, cols, faces = vol.extract(min_weight)
        t_extract.stop()
        torch.cuda.synchronize(rf.device)
    info = dict(voxels=vol.num_voxels, dims=(vol.nx, vol.ny, vol.nz), origin=vol.origin.tolist(),
                voxel_size=float(vol.voxel_size), trunc=float(vol.trunc), frames=len(rf.ids),
                render_ms=rf.t_render.ms(), integrate_ms=rf.t_fuse.ms(), extract_ms=t_extract.ms())
    return verts, cols, faces, info
