"""Per-frame motion masks from the map's depth residual: the pixels where a frame sees something in front of the map
(a moving object, `dynamic`) or past it (the map is stale there, `inconsistent`).  Tracking ignores both, mapping and
map growth ignore `dynamic` (slam.run_slam's `dynamic`).

The rule, on one [3,H,W] depth/silhouette render (d = channel 0, s = channel 1) and the frame's depth g, in float32
rounded as written (include/splatam_b200.h `sb_dynamic_*`; oracle/dynamic_numpy.py is the numpy statement):
- valid = g > 0 & isfinite(d) & s > sil_thres;  r = (d - g) / g  (r > 0: the frame sees something in front of the map).
- scale = the float whose bits are b << 16, b the top 16 bits of the lower-middle valid |r| (a 32768-bin histogram).
- seeds: occ = valid & r > max(k_high scale, r_min), dis = valid & -r > max(k_high scale, r_min); a seed is kept
  when at least 4 of its 8 neighbours are seeds of its kind.
- growth: `radius` Jacobi steps of 4-connected dilation of the kept occ seeds into candidates, g > 0 pixels that are
  weakly occluding (valid & r > max(k_low scale, r_min / 2)) or not covered by the map (s <= sil_thres), across steps
  with |g_p - g_q| <= tau min(g_p, g_q).
- dynamic, inconsistent = the grown mask and the kept dis seeds, each dilated by a Chebyshev radius `dilate`.
CUDA tensors go through csrc/dynamic.cu (five sync-free, graph-capturable kernels); `motion_masks_torch` is the same
rule in torch operations, for the CPU path."""
import math
import numbers

import torch
import torch.nn.functional as F

from . import _lib

# k_high / k_low: seed / growth thresholds in units of the frame's median |relative depth residual|; r_min: the least
# relative residual of a seed; tau: the relative depth step growth may cross; radius: growth steps, in pixels at the
# tracking size; dilate: the final Chebyshev dilation; refresh_every: tracking recomputes its mask every this many
# iterations from that iteration's render.
DEFAULTS = dict(k_high=4.0, k_low=1.5, r_min=0.05, tau=0.05, radius=16, dilate=2, refresh_every=10)
STATS = 6           # valid, scale, occ seeds, dis seeds, dynamic, inconsistent
BINS = 32768


def config(dynamic):
    """run_slam's `dynamic` dict with DEFAULTS filled in; ValueError for unknown keys or bad values."""
    if not isinstance(dynamic, dict):
        raise ValueError("dynamic must be None or a dict of %s, got %r" % (sorted(DEFAULTS), dynamic))
    unknown = sorted(set(dynamic) - set(DEFAULTS))
    if unknown:
        raise ValueError("unknown dynamic keys %s (known: %s)" % (unknown, sorted(DEFAULTS)))
    cfg = dict(DEFAULTS, **dynamic)
    for k in ("k_high", "k_low"):
        v = cfg[k]
        if isinstance(v, bool) or not isinstance(v, numbers.Real) or math.isnan(v) or v < 0:
            raise ValueError("dynamic %s must be a number >= 0 (inf: never), got %r" % (k, v))
        cfg[k] = float(v)
    for k in ("r_min", "tau"):
        v = cfg[k]
        if isinstance(v, bool) or not isinstance(v, numbers.Real) or not math.isfinite(v) or v < 0:
            raise ValueError("dynamic %s must be a finite number >= 0, got %r" % (k, v))
        cfg[k] = float(v)
    for k, lo, hi in (("radius", 0, 1 << 16), ("dilate", 0, 64), ("refresh_every", 1, 1 << 30)):
        v = cfg[k]
        if isinstance(v, bool) or not isinstance(v, numbers.Integral) or not lo <= v <= hi:
            raise ValueError("dynamic %s must be an integer in [%d, %d], got %r" % (k, lo, hi, v))
        cfg[k] = int(v)
    return cfg


def _threshold(k, scale, floor):
    t = torch.tensor(k, dtype=torch.float32, device=scale.device) * scale
    return torch.where(t > floor, t, floor)            # a NaN product (inf * 0) takes the floor


def _shift(a, dy, dx):
    """out[y, x] = a[y + dy, x + dx], zero outside."""
    H, W = a.shape
    p = F.pad(a[None, None].float() if a.dtype == torch.bool else a[None, None], (1, 1, 1, 1))[0, 0]
    out = p[1 + dy:1 + dy + H, 1 + dx:1 + dx + W]
    return out.bool() if a.dtype == torch.bool else out


def _keep_supported(seed):
    n = sum(_shift(seed, dy, dx).int() for dy in (-1, 0, 1) for dx in (-1, 0, 1) if dy or dx)
    return seed & (n >= 4)


def _dilate(a, r):
    return F.max_pool2d(a[None, None].float(), 2 * r + 1, stride=1, padding=r)[0, 0].bool() if r else a


def motion_masks_torch(depth_sil, gt_depth, cfg, sil_thres=0.99):
    """The rule in torch operations (any device): (dynamic [H,W] bool, inconsistent [H,W] bool, stats float32 [6])."""
    d, s = depth_sil[0].detach().float(), depth_sil[1].detach().float()
    g = gt_depth.detach().float().reshape(d.shape)
    sil = torch.tensor(sil_thres, dtype=torch.float32)
    r = (d - g) / g
    valid = (g > 0) & torch.isfinite(d) & (s > sil)
    bins = (r.abs()[valid].view(torch.int32) >> 16)
    n = bins.numel()
    b = int(bins.sort().values[(n - 1) // 2]) if n else 0
    scale = torch.tensor([b << 16], dtype=torch.int32).view(torch.float32).to(d.device)[0]
    r_min = torch.tensor(cfg["r_min"], dtype=torch.float32, device=d.device)
    hi = _threshold(cfg["k_high"], scale, r_min)
    lo = _threshold(cfg["k_low"], scale, r_min * 0.5)
    occ = _keep_supported(valid & (r > hi))
    dis = _keep_supported(valid & (-r > hi))
    cand = (g > 0) & ((valid & (r > lo)) | (s <= sil))
    tau = torch.tensor(cfg["tau"], dtype=torch.float32, device=d.device)
    dyn = occ
    for _ in range(cfg["radius"]):
        grow = torch.zeros_like(dyn)
        for dy, dx in ((-1, 0), (1, 0), (0, -1), (0, 1)):
            nd, ng = _shift(dyn, dy, dx), _shift(g, dy, dx)
            grow = grow | (nd & ((ng - g).abs() <= tau * torch.minimum(ng, g)))
        dyn = dyn | (cand & grow)
    dynamic, inconsistent = _dilate(dyn, cfg["dilate"]), _dilate(dis, cfg["dilate"])
    stats = torch.stack([valid.sum().float(), scale, occ.sum().float(), dis.sum().float(), dynamic.sum().float(),
                         inconsistent.sum().float()])
    return dynamic, inconsistent, stats


def motion_masks(depth_sil, gt_depth, cfg, sil_thres=0.99):
    """The rule on CUDA tensors through csrc/dynamic.cu: (dynamic [H,W] bool, inconsistent [H,W] bool, stats float32
    [6] on the device).  Never synchronises the host, so it can run inside a captured CUDA graph."""
    _lib.need_cuda("motion_masks", depth_sil, gt_depth)
    if depth_sil.dim() != 3 or depth_sil.shape[0] != 3:
        raise ValueError("motion_masks: depth_sil must be [3,H,W], got %s" % (tuple(depth_sil.shape),))
    H, W = depth_sil.shape[-2:]
    if gt_depth.numel() != H * W or gt_depth.shape[-2:] != (H, W):
        raise ValueError("motion_masks: the frame depth %s does not match the %dx%d render"
                         % (tuple(gt_depth.shape), H, W))
    ds, g = depth_sil.detach().contiguous().float(), gt_depth.detach().contiguous().float()
    dev = ds.device
    residual = torch.empty(H * W, dtype=torch.float32, device=dev)
    hist = torch.empty(BINS, dtype=torch.int32, device=dev)
    stats = torch.empty(STATS, dtype=torch.float32, device=dev)
    flags, dyn, tmp, dynamic, inconsistent = torch.empty(5, H, W, dtype=torch.uint8, device=dev).unbind(0)
    _lib.call("sb_dynamic_residual", H, W, ds, g, float(sil_thres), residual, hist, stats, device=dev)
    _lib.call("sb_dynamic_scale", hist, stats, device=dev)
    _lib.call("sb_dynamic_seeds", H, W, ds, g, residual, float(sil_thres), cfg["k_high"], cfg["k_low"], cfg["r_min"],
              flags, dyn, stats, device=dev)
    _lib.call("sb_dynamic_grow", H, W, g, flags, cfg["tau"], cfg["radius"], dyn, tmp, device=dev)
    _lib.call("sb_dynamic_dilate", H, W, dyn, flags, cfg["dilate"], dynamic, inconsistent, stats, device=dev)
    return dynamic.view(torch.bool), inconsistent.view(torch.bool), stats


def masks(depth_sil, gt_depth, cfg, sil_thres=0.99, fused=True):
    """`motion_masks` (fused, CUDA) or `motion_masks_torch`."""
    if fused:
        return motion_masks(depth_sil, gt_depth, cfg, sil_thres)
    return motion_masks_torch(depth_sil, gt_depth, cfg, sil_thres)


def footprint(mask, shape):
    """A [H,W] bool mask carried to a [h,w] grid: a cell is set where any pixel of its footprint is (max-pooling), as
    SplaTAM-S's densification frame needs."""
    if tuple(mask.shape) == tuple(shape):
        return mask
    return F.adaptive_max_pool2d(mask[None, None].float(), tuple(shape))[0, 0].bool()
