"""Headless versions of the reference's viewers (R/viz_scripts/final_recon.py and online_recon.py): the pictures they
show in an Open3D window, computed on the GPU as uint8 RGB frames and written as PNGs, with no window and no Open3D.

* ``load_record``      a run record as load_camera / load_scene_data read it: this project's and the reference's
                       `params.npz`, the 13-key offline records and, with ``camera=``, checkpoint `params{t}.npz` files
* ``ViewerConfig``     the `viz` dict of the shipped configs
* ``final_view``       final_recon: the whole map from the first frame's camera (+0.5 on z with offset_first_viz_cam),
                       every frustum and the trajectory
* ``online_frames``    online_recon: frame t shows the Gaussians with timestep <= t from first_view_w2c @ w2c_t, the
                       frustum of frame t and the trajectory up to t
* ``render_record``    either, written as DIR/final.png or DIR/online/%06d.png (and optionally one raw RGB24 stream)

What Open3D draws is restated as pixel rules (csrc/viewer.cu, DESIGN.md): the render's back-projected pixels seen from
the render's own camera at k * view_scale are the render upsampled view_scale times (sb_viewer_compose); `centers`
mode draws every selected Gaussian centre as a view_scale-pixel square (sb_viewer_points); frustums and trajectory are
1 px lines depth-tested against the picture (sb_viewer_lines).  Renders go through this project's rasterizer with the
viewer's white background.  CUDA only; no CPU fallback."""
import numbers
import os
from dataclasses import dataclass, fields

import numpy as np
import torch
import torch.nn.functional as F

from . import _lib
from . import evaluate as EV
from . import formats
from . import map_ops
from . import mapping as M
from .rasterizer import GaussianRasterizationSettings, GaussianRasterizer

MODES = ("color", "depth", "centers")
_COMPOSE_COLOR, _COMPOSE_DEPTH, _COMPOSE_SIL = 0, 1, 2
FRUSTUM_SIZE = 0.045               # final_recon / online_recon frustum_size
VIEW_OFFSET_Z = 0.5                # the view camera's offset on its translation's z
DEPTH_FAR = 15.0                   # depth mode: pixels at d >= 15 are white

# matplotlib's segment data (matplotlib/_cm.py): (x, y0, y1) per channel
JET_DATA = {"red": ((0.00, 0, 0), (0.35, 0, 0), (0.66, 1, 1), (0.89, 1, 1), (1.00, 0.5, 0.5)),
            "green": ((0.000, 0, 0), (0.125, 0, 0), (0.375, 1, 1), (0.640, 1, 1), (0.910, 0, 0), (1.000, 0, 0)),
            "blue": ((0.00, 0.5, 0.5), (0.11, 1, 1), (0.34, 1, 1), (0.65, 0, 0), (1.00, 0, 0))}
COOL_DATA = {"red": ((0., 0., 0.), (1.0, 1.0, 1.0)), "green": ((0., 1., 1.), (1.0, 0., 0.)),
             "blue": ((0., 1., 1.), (1.0, 1., 1.))}


def segment_lut(data, N=256):
    """matplotlib's LinearSegmentedColormap table (colors._create_lookup_table, gamma 1): float64 [N, 3] in [0, 1],
    in its operation order -- breakpoints and sample positions both scaled by N - 1 before the interpolation, which
    decides the last bit and with it which entries land on a .5 tie at 255 scale."""
    xind = (N - 1) * np.linspace(0, 1, N) ** 1.0
    out = []
    for ch in ("red", "green", "blue"):
        a = np.array(data[ch], dtype=float)
        x, y0, y1 = a[:, 0] * (N - 1), a[:, 1], a[:, 2]
        ind = np.searchsorted(x, xind)[1:-1]
        distance = (xind[1:-1] - x[ind - 1]) / (x[ind] - x[ind - 1])
        lut = np.concatenate([[y1[0]], distance * (y0[ind] - y1[ind - 1]) + y1[ind - 1], [y0[-1]]])
        out.append(np.clip(lut, 0.0, 1.0))
    return np.stack(out, -1)


def to_u8(x):
    """round_half_even(clip(x, 0, 1) * 255) of float64 colours, the frames' colour rule."""
    return np.rint(np.clip(np.asarray(x, float), 0.0, 1.0) * 255).astype(np.uint8)


JET_LUT = segment_lut(JET_DATA)
COOL_LUT = segment_lut(COOL_DATA)
JET_U8 = to_u8(JET_LUT)


def cmap_index(x, N=256):
    """The table index matplotlib's Colormap.__call__ takes for a Python float x: trunc(x * N), N -> N - 1, clamped
    below to 0 and above to N - 1 (x < 0 and x > 1 fall to the under / over colours, the end entries)."""
    xa = float(x) * N
    if xa == N:
        xa = N - 1
    if xa < 0:
        return 0
    if xa >= N:
        return N - 1
    return int(xa)


def cool(x):
    """matplotlib cool(x)[:3] as float64 for a Python float x."""
    return COOL_LUT[cmap_index(x)]


@dataclass
class ViewerConfig:
    """The `viz` dict of the shipped configs.  viz_fps and enter_interactive_post_online are accepted and unused:
    frames are taken at every `every`-th timestep rather than by wall clock, and there is no interactive mode."""
    render_mode: str = "color"
    offset_first_viz_cam: bool = True
    show_sil: bool = False
    visualize_cams: bool = True
    viz_w: int = 600
    viz_h: int = 340
    viz_near: float = 0.01
    viz_far: float = 100.0
    view_scale: int = 2
    viz_fps: float = 5
    enter_interactive_post_online: bool = True

    def __post_init__(self):
        s = self.view_scale
        if isinstance(s, bool) or not isinstance(s, numbers.Real) or s != int(s) or s < 1:
            raise ValueError("view_scale must be an integer >= 1, got %r" % (s,))
        self.view_scale = int(s)
        if self.render_mode not in MODES:
            raise ValueError("render_mode must be one of %s, got %r" % (MODES, self.render_mode))
        for name in ("viz_w", "viz_h"):
            v = getattr(self, name)
            if isinstance(v, bool) or not isinstance(v, numbers.Real) or v != int(v) or v < 1:
                raise ValueError("%s must be a positive integer, got %r" % (name, v))
            setattr(self, name, int(v))
        if not (0 < self.viz_near < self.viz_far):
            raise ValueError("need 0 < viz_near < viz_far, got %r, %r" % (self.viz_near, self.viz_far))

    @classmethod
    def from_viz(cls, viz=None, **overrides):
        """From a config's `viz` dict (unknown keys raise ValueError), with keyword overrides."""
        d = dict(viz or {}, **overrides)
        known = {f.name for f in fields(cls)}
        unknown = sorted(set(d) - known)
        if unknown:
            raise ValueError("unknown viz keys: %s" % ", ".join(unknown))
        return cls(**d)


def _as_cfg(cfg):
    if cfg is None:
        return ViewerConfig()
    return cfg if isinstance(cfg, ViewerConfig) else ViewerConfig.from_viz(cfg)


def scaled_intrinsics(intrinsics, org_width, org_height, cfg):
    """load_camera's k: intrinsics[:3, :3] with row 0 scaled by viz_w / org_width and row 1 by viz_h / org_height,
    as the reference's numpy statements compute it (float32 array, float64 factors)."""
    k = np.array(intrinsics, dtype=np.float32)[:3, :3].copy()
    k[0, :] *= cfg.viz_w / np.asarray(org_width)
    k[1, :] *= cfg.viz_h / np.asarray(org_height)
    return k


def _build_rotation(q):
    """build_rotation of R/utils/slam_external.py in its operation order (the norm as a left-to-right sum of squares,
    not a reduction), so the host result is the reference's bit for bit on the same device."""
    norm = torch.sqrt(q[:, 0] * q[:, 0] + q[:, 1] * q[:, 1] + q[:, 2] * q[:, 2] + q[:, 3] * q[:, 3])
    q = q / norm[:, None]
    r, x, y, z = q[:, 0], q[:, 1], q[:, 2], q[:, 3]
    return torch.stack([1 - 2 * (y * y + z * z), 2 * (x * y - r * z), 2 * (x * z + r * y),
                        2 * (x * y + r * z), 1 - 2 * (x * x + z * z), 2 * (y * z - r * x),
                        2 * (x * z - r * y), 2 * (y * z + r * x), 1 - 2 * (x * x + y * y)], -1).reshape(-1, 3, 3)


def trajectory_w2cs(cam_unnorm_rots, cam_trans):
    """load_scene_data's all_w2cs: float32 [T, 4, 4] from F.normalize(cam_unnorm_rots[..., t]) and cam_trans[..., t]
    with build_rotation, one frame at a time as the reference does, on the host."""
    rots = torch.as_tensor(np.asarray(cam_unnorm_rots, np.float32))
    trans = torch.as_tensor(np.asarray(cam_trans, np.float32))
    T = rots.shape[-1]
    out = torch.eye(4).repeat(T, 1, 1)
    for t in range(T):
        out[t, :3, :3] = _build_rotation(F.normalize(rots[..., t]))[0]
        out[t, :3, 3] = trans[..., t]
    return out.numpy()


class ViewerRecord:
    """A run record loaded for the viewers.  Host: intrinsics [3,3], first_w2c [4,4], all_w2cs [T,4,4] (float32
    numpy), org_width / org_height, timestep_host (float32 [P] or None), monotone, counts ([T] prefix lengths when the
    timestep is non-decreasing).  Device: the rendervars of the whole map -- means3D, colors (rgb_colors),
    rotations (normalised), opacities (sigmoid), scales (exp of log_scales, isotropic ones tiled to 3 columns) --
    and timestep."""

    def __init__(self, **kw):
        self.__dict__.update(kw)

    @property
    def P(self):
        return self.means3D.shape[0]

    @property
    def T(self):
        return self.all_w2cs.shape[0]

    def k(self, cfg=None):
        return scaled_intrinsics(self.intrinsics, self.org_width, self.org_height, _as_cfg(cfg))


def load_record(path, device, viz=None, camera=None):
    """Reads a run record as the reference's load_camera and load_scene_data do.  `path`: this project's or the
    reference's `params.npz` (formats.save_run_record), an offline record (13 keys, no keyframe_time_indices) or a
    checkpoint `params{t}.npz`; a checkpoint holds no camera, so pass ``camera=dict(intrinsics=, w2c=, org_width=,
    org_height=)`` (any of these also overrides the record's).  `viz` (a ViewerConfig or `viz` dict) only checks the
    settings early; each view takes its own config.  A missing key raises ValueError naming it, as does a
    cam_unnorm_rots / cam_trans pair whose camera counts differ (formats.read_record).  Without `timestep` only the
    final view renders."""
    _as_cfg(viz)
    raw = formats.read_record(path, formats.CHECKPOINT_KEYS + formats.CAMERA_KEYS, camera)
    rots, trans = np.asarray(raw["cam_unnorm_rots"]), np.asarray(raw["cam_trans"])
    dev = torch.device(device)
    g = formats.record_tensors(raw, formats.GAUSSIAN_KEYS, dev)
    log_scales = g["log_scales"]
    if log_scales.shape[-1] == 1:
        log_scales = torch.tile(log_scales, (1, 3))
    ts = None if "timestep" not in raw else np.ascontiguousarray(np.asarray(raw["timestep"], np.float32).reshape(-1))
    T = rots.shape[-1]
    monotone = ts is not None and bool(np.all(ts[1:] >= ts[:-1]))
    counts = np.searchsorted(ts, np.arange(T), side="right") if monotone else None
    return ViewerRecord(
        path=path, device=dev, intrinsics=np.array(raw["intrinsics"], np.float32)[:3, :3],
        first_w2c=np.array(raw["w2c"], np.float32).reshape(4, 4), org_width=np.asarray(raw["org_width"]),
        org_height=np.asarray(raw["org_height"]), all_w2cs=trajectory_w2cs(rots, trans),
        means3D=g["means3D"], colors=g["rgb_colors"], rotations=F.normalize(g["unnorm_rotations"]),
        opacities=torch.sigmoid(g["logit_opacities"]), scales=torch.exp(log_scales),
        timestep=None if ts is None else torch.from_numpy(ts).to(dev), timestep_host=ts, monotone=monotone,
        counts=counts)


def select_mask(record, t):
    """get_rendervars' selection of frame t: bool [P] (device), timestep <= t."""
    return record.timestep <= t


def view_w2cs(record, cfg, online):
    """The view cameras, float32 numpy [V, 4, 4].  Final: the first-frame w2c, +0.5 on its translation's z when
    offset_first_viz_cam.  Online: first_view_w2c @ w2c_t for every t, with the offset always applied."""
    first = record.first_w2c.copy()
    if online or cfg.offset_first_viz_cam:
        first[:3, 3] = first[:3, 3] + np.array([0, 0, VIEW_OFFSET_Z])
    if not online:
        return first[None]
    return np.stack([np.dot(first, w) for w in record.all_w2cs])


def frustum_segments(k, w, h, w2c, size=FRUSTUM_SIZE):
    """The 8 world-space segments [8, 6] of a camera frustum: the centre to the image corners (0,0), (w,0), (w,h),
    (0,h) back-projected through k at depth `size`, then the rectangle through the corners (Open3D's
    LineSet.create_camera_visualization geometry).  Float64 on the host."""
    K4 = np.eye(4)
    K4[:3, :3] = np.asarray(k, float)
    m = np.linalg.inv(K4 @ np.asarray(w2c, float))
    pts = [np.zeros(3)] + [np.array([x * size, y * size, size]) for x, y in ((0, 0), (w, 0), (w, h), (0, h))]
    pts = [(m @ np.append(p, 1.0))[:3] for p in pts]
    pairs = ((0, 1), (0, 2), (0, 3), (0, 4), (1, 2), (2, 3), (3, 4), (4, 1))
    return np.array([np.concatenate([pts[a], pts[b]]) for a, b in pairs])


def camera_lines(record, cfg):
    """(frustum segments [T*8, 6], their colours [T*8, 3] uint8, trajectory segments [T-1, 6], colours [T-1, 3]):
    frustum t coloured cool(t * 0.5 / T), trajectory segment i (centre i -> centre i+1, centres inv(w2c_t)[:3, 3])
    coloured cool(i * 0.5 / (T - 1) + 0.5).  Host arrays."""
    k, T = record.k(cfg), record.T
    fr = np.concatenate([frustum_segments(k, cfg.viz_w, cfg.viz_h, record.all_w2cs[t]) for t in range(T)])
    fc = np.repeat(to_u8(np.stack([cool(t * 0.5 / T) for t in range(T)])), 8, axis=0)
    centres = np.stack([np.linalg.inv(w)[:3, 3] for w in record.all_w2cs])
    tr = np.concatenate([centres[:-1], centres[1:]], 1).reshape(-1, 6)
    tc = to_u8(np.stack([cool(i * 0.5 / (T - 1) + 0.5) for i in range(T - 1)])) if T > 1 else np.zeros((0, 3), np.uint8)
    return fr, fc, tr, tc


class _Views:
    """Device-side cameras of every view of one pass (built once, so a frame enqueues no host-to-device copy):
    w2c [V,4,4] row-major, the raster settings' viewmatrix / projmatrix [V,1,4,4] and campos [V,3] as
    datasets.setup_camera builds them, and the intrinsics at output size."""

    def __init__(self, record, cfg, online):
        dev = record.device
        self.cfg, self.online = cfg, online
        w2c = view_w2cs(record, cfg, online)
        k = record.k(cfg)
        w, h, near, far = cfg.viz_w, cfg.viz_h, cfg.viz_near, cfg.viz_far
        fx, fy, cx, cy = k[0][0], k[1][1], k[0][2], k[1][2]
        proj = torch.tensor([[2 * fx / w, 0.0, -(w - 2 * cx) / w, 0.0],
                             [0.0, 2 * fy / h, -(h - 2 * cy) / h, 0.0],
                             [0.0, 0.0, far / (far - near), -(far * near) / (far - near)],
                             [0.0, 0.0, 1.0, 0.0]]).float().T
        w2c_t = torch.from_numpy(w2c)
        self.w2c = w2c_t.to(dev).contiguous()
        self.viewmatrix = w2c_t.transpose(1, 2).unsqueeze(1).to(dev).contiguous()
        proj = proj.to(dev).unsqueeze(0)
        self.projmatrix = torch.stack([m.bmm(proj) for m in self.viewmatrix])     # setup_camera's product, per view
        self.campos = torch.inverse(w2c_t)[:, :3, 3].to(dev).contiguous()
        self.tanfov = (w / (2 * fx), h / (2 * fy))
        s = cfg.view_scale
        ks = k * np.float32(s)
        self.k_out = (float(ks[0, 0]), float(ks[1, 1]), float(ks[0, 2]), float(ks[1, 2]))
        self.white = torch.ones(3, dtype=torch.float32, device=dev)
        self.black = torch.zeros(3, dtype=torch.float32, device=dev)
        self.H, self.W = h * s, w * s
        fr, fc, tr, tc = camera_lines(record, cfg)
        f32 = lambda a: torch.from_numpy(np.ascontiguousarray(a, np.float32)).to(dev)
        u8 = lambda a: torch.from_numpy(np.ascontiguousarray(a, np.uint8)).to(dev)
        if online:
            self.frustums, self.frustum_cols, self.traj, self.traj_cols = f32(fr), u8(fc), f32(tr), u8(tc)
        else:
            self.segs, self.seg_cols = f32(np.concatenate([fr, tr])), u8(np.concatenate([fc, tc]))
        self.zbuf = torch.empty(self.H, self.W, dtype=torch.float32, device=dev)
        self.keys = torch.empty(self.H * self.W, dtype=torch.int64, device=dev)
        self.vmax = torch.empty(1, dtype=torch.int32, device=dev)
        self.lut = torch.from_numpy(JET_U8.copy()).to(dev)

    def settings(self, v, bg):
        cfg = self.cfg
        return GaussianRasterizationSettings(
            image_height=cfg.viz_h, image_width=cfg.viz_w, tanfovx=self.tanfov[0], tanfovy=self.tanfov[1], bg=bg,
            scale_modifier=1.0, viewmatrix=self.viewmatrix[v], projmatrix=self.projmatrix[v], sh_degree=0,
            campos=self.campos[v], prefiltered=False)

    def lines(self, t):
        """(segments, colours) drawn in view t: every frustum and the whole trajectory (final), or frustum t and the
        trajectory up to t (online)."""
        if not self.online:
            return self.segs, self.seg_cols
        return (torch.cat([self.frustums[8 * t:8 * t + 8], self.traj[:t]]),
                torch.cat([self.frustum_cols[8 * t:8 * t + 8], self.traj_cols[:t]]))


def _subset(record, t, compact):
    """Rendervars (means3D, colors, rotations, opacities, scales) of the Gaussians with timestep <= t: a prefix view
    when the timestep is non-decreasing (no copy, no synchronisation), else gathered by sb_compact_plan /
    sb_compact_flat (one count read).  compact=True forces the gather."""
    keys = ("means3D", "colors", "rotations", "opacities", "scales")
    if record.timestep is None or t is None:
        return [getattr(record, k) for k in keys]
    if record.monotone and not compact:
        n = int(record.counts[t])
        return [getattr(record, k)[:n] for k in keys]
    widths = (3, 3, 4, 1, 3)
    if getattr(record, "flat", None) is None:          # the packed [w0*P | w1*P | ...] source, built once
        record.flat = torch.cat([getattr(record, k).reshape(-1) for k in keys])
    m, dst, n = map_ops.compact_plan(select_mask(record, t))
    out = map_ops.compact_flat(record.flat, record.P, widths, m, dst, n)
    parts, o = [], 0
    for w in widths:
        parts.append(out[o:o + w * n].view(n, w))
        o += w * n
    return parts


def render_view(record, views, v, t, compact=False):
    """The viewer's renders of view v over the Gaussians selected for timestep t (None: all): (im [3,h,w] on the
    white background, depth [1,h,w], sil [1,h,w] or None).  sil (channel 1 of a black-background render with colour
    (0, 1, 0)) is rendered only with show_sil."""
    means, colors, rot, opac, scales = _subset(record, t, compact)
    with torch.no_grad():
        zeros = torch.zeros_like(means)
        im, _, depth = GaussianRasterizer(views.settings(v, views.white))(
            means3D=means, means2D=zeros, opacities=opac, colors_precomp=colors, scales=scales, rotations=rot)
        sil = None
        if views.cfg.show_sil and views.cfg.render_mode == "color":
            ones = torch.zeros_like(means)
            ones[:, 1] = 1.0
            ds, _, _ = GaussianRasterizer(views.settings(v, views.black))(
                means3D=means, means2D=zeros, opacities=opac, colors_precomp=ones, scales=scales, rotations=rot)
            sil = ds[1:2]
    return im, depth, sil


def compose(im, depth, sil, mode, view_scale, lut, out, zbuf, vmax):
    """sb_viewer_compose into out [h*s, w*s, 3] uint8 and zbuf [h*s, w*s] float32 (device)."""
    c = lambda x: None if x is None else x.detach().float().contiguous()
    h, w = depth.shape[-2:]
    _lib.call("sb_viewer_compose", c(im), c(depth), c(sil), h, w, mode, view_scale, lut, vmax, out, zbuf,
              device=out.device)


def draw_points(means, colors, timestep, t_max, w2c, k_out, W, H, s, near, far, keys, out, zbuf):
    """sb_viewer_points: centres means [P,3] with colours [P,3] (and timestep <= t_max when timestep is given)."""
    _lib.call("sb_viewer_points", means.shape[0], means, colors, timestep, float(t_max), w2c, *k_out, W, H, s,
              float(near), float(far), keys, out, zbuf, device=out.device)


def draw_lines(segs, cols, w2c, k_out, W, H, near, zbuf, keys, out):
    """sb_viewer_lines: segments [S,6] with uint8 colours [S,3] over out, depth-tested against zbuf."""
    _lib.call("sb_viewer_lines", segs.shape[0], segs, cols, w2c, *k_out, W, H, float(near), zbuf, keys, out,
              device=out.device)


def _draw(record, views, v, t, out, compact=False):
    """One frame into out [H, W, 3] uint8: the picture of view v with the map at timestep t (None: whole map)."""
    cfg = views.cfg
    _lib.need_cuda("viewer", record.means3D, out)
    if cfg.render_mode == "centers":
        if t is None or record.timestep is None:
            draw_points(record.means3D, record.colors, None, 0.0, views.w2c[v], views.k_out, views.W, views.H,
                        cfg.view_scale, cfg.viz_near, cfg.viz_far, views.keys, out, views.zbuf)
        elif record.monotone and not compact:
            n = int(record.counts[t])
            draw_points(record.means3D[:n], record.colors[:n], None, 0.0, views.w2c[v], views.k_out, views.W,
                        views.H, cfg.view_scale, cfg.viz_near, cfg.viz_far, views.keys, out, views.zbuf)
        else:
            draw_points(record.means3D, record.colors, record.timestep, float(t), views.w2c[v], views.k_out, views.W,
                        views.H, cfg.view_scale, cfg.viz_near, cfg.viz_far, views.keys, out, views.zbuf)
    else:
        im, depth, sil = render_view(record, views, v, t, compact)
        mode = _COMPOSE_DEPTH if cfg.render_mode == "depth" else _COMPOSE_SIL if sil is not None else _COMPOSE_COLOR
        compose(im, depth, sil, mode, cfg.view_scale, views.lut, out, views.zbuf, views.vmax)
    if cfg.visualize_cams:
        segs, cols = views.lines(t if views.online else 0)
        if segs.shape[0]:
            draw_lines(segs, cols, views.w2c[v], views.k_out, views.W, views.H, cfg.viz_near, views.zbuf, views.keys,
                       out)
    return out


def _frame(views, device):
    return torch.empty(views.H, views.W, 3, dtype=torch.uint8, device=device)


def final_view(record, cfg=None):
    """final_recon's picture: uint8 [viz_h * s, viz_w * s, 3] on the record's device."""
    cfg = _as_cfg(cfg)
    views = _Views(record, cfg, online=False)
    with torch.cuda.device(record.device):
        return _draw(record, views, 0, None, _frame(views, record.device))


def _online_check(record):
    if record.timestep is None:
        raise ValueError("%s has no `timestep`: the online view needs each Gaussian's timestep (the final view "
                         "renders without it)" % record.path)


def online_frames(record, cfg=None, every=1, compact=False):
    """online_recon's frames: yields (t, uint8 [viz_h * s, viz_w * s, 3] device frame) for t = 0, every, 2 every, ...
    < T.  compact=True gathers each frame's Gaussians with the compaction kernels even when the record's timestep
    is non-decreasing (the frames are the same)."""
    cfg = _as_cfg(cfg)
    _online_check(record)
    if int(every) != every or every < 1:
        raise ValueError("every must be a positive integer, got %r" % (every,))
    views = _Views(record, cfg, online=True)
    for t in range(0, record.T, int(every)):
        # the record's device is current only while a frame is enqueued, never while the generator is suspended
        with torch.cuda.device(record.device):
            frame = _draw(record, views, t, t, _frame(views, record.device), compact)
        yield t, frame


def render_record(record, cfg, out_dir, mode="final", every=1, raw=None, threads=None):
    """Writes `mode`'s frames as PNGs: out_dir/final.png, or out_dir/online/{t:06d}.png for each rendered t.
    raw: a path that also receives every frame as one raw RGB24 stream (viz_w * s by viz_h * s, in t order), e.g.
    for ffmpeg -f rawvideo -pix_fmt rgb24 -s WxH -r FPS -i FILE out.mp4.  Frames are drawn into a device staging
    buffer and written by evaluate.HostWriter threads.  Returns the PNG paths."""
    cfg = _as_cfg(cfg)
    if mode not in ("final", "online"):
        raise ValueError("mode must be 'final' or 'online', got %r" % (mode,))
    if mode == "online":
        _online_check(record)
    views = _Views(record, cfg, online=mode == "online")
    if mode == "final":
        jobs = [(0, None, os.path.join(out_dir, "final.png"))]
        os.makedirs(out_dir, exist_ok=True)
    else:
        d = os.path.join(out_dir, "online")
        os.makedirs(d, exist_ok=True)
        jobs = [(t, t, os.path.join(d, "%06d.png" % t)) for t in range(0, record.T, int(every))]
    pngs = EV.HostWriter((views.H, views.W, 3), record.device, threads, name="viewer-png")
    stream = None if raw is None else EV.HostWriter((views.H, views.W, 3), record.device, 1, name="viewer-raw")
    f = None if raw is None else open(raw, "wb")
    try:
        with torch.cuda.device(record.device):
            for v, t, path in jobs:
                fill = lambda st, v=v, t=t: _draw(record, views, v, t, st)
                pngs.put(fill, lambda px, path=path: EV.save_png(px, path))
                if stream is not None:
                    stream.put(lambda st: st.copy_(pngs.staging), lambda px: f.write(px.tobytes()))
    finally:
        pngs.close()
        if stream is not None:
            stream.close()
            f.close()
    return [p for _, _, p in jobs]
