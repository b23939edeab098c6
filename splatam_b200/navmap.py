"""Navigation maps from a SplaTAM map: which space is free, occupied or unobserved, and how far each point is from the
nearest obstacle, with a gradient -- what a planner needs, computed on the GPU (csrc/navmap.cu).

* ``NavMap``      occupancy labels and an exact Euclidean signed distance field (ESDF) on the grid of a
                  ``mesh.TSDFVolume``; ``distance`` queries it at any points
* ``nav_record``  the navigation map of a saved run record, fused as ``mesh.mesh_record`` fuses it

The rules (labels, obstacle set, signed squared distance, query interpolation) are stated in include/splatam_b200.h.
The map is in the map's frame, that of `means3D`.  CUDA only; no CPU fallback."""
import numpy as np
import torch

from . import _lib
from . import formats
from . import mesh

LABEL_UNKNOWN, LABEL_FREE, LABEL_OCCUPIED = 0, 1, 2


def _check_grid(nx, ny, nz):
    if max(nx, ny, nz) > 8192 or nx * ny * nz >= 2 ** 31:
        raise ValueError("a navigation map needs every dimension <= 8192 and fewer than 2^31 samples, got %d x %d x %d"
                         % (nx, ny, nz))


class NavMap:
    """labels uint8 [nz,ny,nx] (0 unknown, 1 free, 2 occupied) and esdf float32 [nz,ny,nx] (metres; > 0 outside the
    obstacles, < 0 inside, +-inf when the obstacle set is empty / everything) on one device, with the grid (origin,
    voxel_size) and the parameters they were built with.  sd2 (int32, the signed squared distance in lattice units)
    is kept when the map was built here, and is None for a loaded map."""

    def __init__(self, labels, esdf, origin, voxel_size, trunc, min_weight, occ_dist, unknown_is_obstacle, sd2=None):
        self.labels, self.esdf, self.sd2 = labels, esdf, sd2
        self.device = labels.device
        self.nz, self.ny, self.nx = (int(d) for d in labels.shape)
        self.origin = np.asarray(origin, np.float32).reshape(3)
        self.voxel_size, self.trunc = np.float32(voxel_size), np.float32(trunc)
        self.min_weight, self.occ_dist = np.float32(min_weight), np.float32(occ_dist)
        self.unknown_is_obstacle = bool(unknown_is_obstacle)

    @classmethod
    def from_volume(cls, vol, min_weight=1.0, occ_dist=None, unknown_is_obstacle=True, timers=None):
        """Labels, sd2 and esdf of a TSDFVolume on its device (sb_nav_labels, sb_esdf): unknown where W <
        min_weight, else occupied where T * trunc <= occ_dist (default half a voxel), else free.  The obstacles are
        the occupied samples, and the unknown ones too with `unknown_is_obstacle`.  The map keeps no reference to
        the volume, which can be freed afterwards.  timers: two mesh._Timer that time the labels and the ESDF
        launches.  No host synchronisation."""
        dev = vol.device
        _lib.need_cuda("NavMap.from_volume", vol.tsdf)
        nx, ny, nz = vol.nx, vol.ny, vol.nz
        _check_grid(nx, ny, nz)
        occ = 0.5 * float(vol.voxel_size) if occ_dist is None else float(occ_dist)
        mw = float(min_weight)
        if not (np.isfinite(occ) and np.isfinite(mw)):
            raise ValueError("min_weight and occ_dist must be finite, got %r and %r" % (min_weight, occ_dist))
        with torch.cuda.device(dev):
            labels = torch.empty((nz, ny, nx), dtype=torch.uint8, device=dev)
            sd2 = torch.empty((nz, ny, nx), dtype=torch.int32, device=dev)
            esdf = torch.empty((nz, ny, nx), dtype=torch.float32, device=dev)
            nb = _lib.nbytes("sb_esdf_workspace_bytes", nx, ny, nz)
            ws = torch.empty(nb, dtype=torch.uint8, device=dev)
            if timers:
                timers[0].start()
            _lib.call("sb_nav_labels", nx, ny, nz, vol.tsdf, vol.weight, float(vol.trunc), mw, occ, labels,
                      device=dev)
            if timers:
                timers[0].stop()
                timers[1].start()
            _lib.call("sb_esdf", nx, ny, nz, labels, float(vol.voxel_size), int(bool(unknown_is_obstacle)), ws, nb,
                      sd2, esdf, device=dev)
            if timers:
                timers[1].stop()
        return cls(labels, esdf, vol.origin, vol.voxel_size, vol.trunc, mw, occ, unknown_is_obstacle, sd2)

    def distance(self, points):
        """(dist [N], grad [N,3]) float32 on the map's device at points [N,3] (or [3]) in metres (sb_esdf_query):
        trilinear in the esdf and its exact gradient; NaN for a point outside the grid, so `dist > r` fails safe;
        an infinite distance and a zero gradient next to an infinite sample.  No host synchronisation."""
        dev = self.device
        p = torch.as_tensor(points).to(dev, torch.float32).reshape(-1, 3).contiguous()
        _lib.need_cuda("NavMap.distance", self.esdf, p)
        if min(self.nx, self.ny, self.nz) < 2:
            raise ValueError("distance queries need every grid dimension >= 2, got %d x %d x %d"
                             % (self.nx, self.ny, self.nz))
        N = p.shape[0]
        dist = torch.empty(N, dtype=torch.float32, device=dev)
        grad = torch.empty(N, 3, dtype=torch.float32, device=dev)
        o = self.origin
        _lib.call("sb_esdf_query", self.nx, self.ny, self.nz, float(o[0]), float(o[1]), float(o[2]),
                  float(self.voxel_size), self.esdf, N, p, dist, grad, device=dev)
        return dist, grad

    def counts(self):
        """dict(free, occupied, unknown) sample counts; the one host read."""
        c = torch.bincount(self.labels.reshape(-1).to(torch.int64), minlength=3).cpu().tolist()
        return dict(free=int(c[LABEL_FREE]), occupied=int(c[LABEL_OCCUPIED]), unknown=int(c[LABEL_UNKNOWN]))

    def save(self, path):
        """formats.save_nav_map of the labels, the esdf and the grid; returns the path."""
        return formats.save_nav_map(path, self.labels, self.esdf, self.origin, self.voxel_size, self.trunc,
                                    self.min_weight, self.occ_dist, self.unknown_is_obstacle)

    @classmethod
    def load(cls, path, device="cuda"):
        """A map saved by `save`, read through formats.load_nav_map (a checked reader: ValueError naming the key)."""
        d = formats.load_nav_map(path)
        dev = torch.device(device)
        labels = torch.from_numpy(d["labels"]).to(dev)
        esdf = torch.from_numpy(d["esdf"]).to(dev)
        return cls(labels, esdf, d["origin"], d["voxel_size"], d["trunc"], d["min_weight"], d["occ_dist"],
                   d["unknown_is_obstacle"])


def nav_record(path, voxel_size, every=1, sil_thres=0.99, depth_max=None, bounds=None, batch=8, trunc=None,
               min_weight=1.0, occ_dist=None, unknown_is_obstacle=True, device="cuda", source=None,
               max_voxels=mesh.MAX_VOXELS, camera=None):
    """The navigation map of a saved run record: its frames fused into a TSDF volume exactly as mesh.mesh_record
    fuses them (rendered depth, or `source`'s frames; the same bounds, every, batch and trunc), then
    NavMap.from_volume.  Returns (NavMap, info): info = dict(voxels, dims, origin, voxel_size, trunc, frames,
    render_ms, integrate_ms, labels_ms, esdf_ms -- the last four device times -- and clearance, the esdf in metres at
    the record's camera centres inside the grid, for the frames fused)."""
    rf = mesh.RecordFusion(path, every, sil_thres, depth_max, batch, device, source, camera)
    tr = 4.0 * float(voxel_size) if trunc is None else float(trunc)
    if bounds is None:
        bounds = mesh.default_bounds(rf.means_host, tr)
    vol = mesh.TSDFVolume(bounds, voxel_size, tr, rf.device, max_voxels)
    _check_grid(vol.nx, vol.ny, vol.nz)
    rf.fuse(vol)
    t_labels, t_esdf = mesh._Timer(), mesh._Timer()
    with torch.cuda.device(rf.device):
        nm = NavMap.from_volume(vol, min_weight, occ_dist, unknown_is_obstacle, timers=(t_labels, t_esdf))
        w2c = rf.w2cs
        centres = -(w2c[:, :3, :3].transpose(1, 2) @ w2c[:, :3, 3:]).reshape(-1, 3)
        dist, _ = nm.distance(centres)
        torch.cuda.synchronize(rf.device)
    d = dist.cpu().numpy()
    info = dict(voxels=vol.num_voxels, dims=(vol.nx, vol.ny, vol.nz), origin=vol.origin.tolist(),
                voxel_size=float(vol.voxel_size), trunc=float(vol.trunc), frames=len(rf.ids),
                render_ms=rf.t_render.ms(), integrate_ms=rf.t_fuse.ms(), labels_ms=t_labels.ms(),
                esdf_ms=t_esdf.ms(), clearance=[float(x) for x in d[~np.isnan(d)]])
    return nm, info
