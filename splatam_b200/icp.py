"""Pose initialisation by frame-to-model point-to-plane ICP on the GPU (csrc/icp.cu, sb_icp_align).

The map's depth, rendered at frame t-1's estimated pose, is aligned with frame t's sensor depth, coarse to fine over a
three-level pyramid, starting from the constant-velocity guess.  A pose that fails the acceptance test (too few
inliers, a large residual or an ill-conditioned system, such as a single plane) is not used: the guess stays.  The
whole alignment runs on the device with no host synchronisation, so it can be captured into a CUDA graph.

* ``align``        one alignment: (w2c [4,4] float32, stats [STATS] float64), both on the device
* ``read_stats``   the host view of a stats record (accepted, inlier fraction, RMS residual, ...)
* ``model_depth_sil``  the depth/silhouette render of a SplaTAM map at one frame's pose
* ``align_rgbd``   joint geometric and photometric alignment (sb_rgbd_icp_align): the map's RGB render and the
                   frame's RGB add a weighted intensity term, so a textured plane is no longer degenerate
* ``model_render`` the RGB and the depth/silhouette render of a SplaTAM map at one frame's pose
* ``init_pose``    run_slam's step: align frame t and write the pose into column t of the camera tensors

CUDA only; CPU tensors raise."""
import ctypes
import math

import numpy as np
import torch
import torch.nn.functional as F

from . import _lib
from . import mapping as M

LEVELS = 3
STATS = 36
RGBD_STATS = 66
DEFAULT_ITERS = (10, 5, 4)       # levels 0 (full size), 1, 2
DEFAULT_WEIGHT = 0.05            # align_rgbd's lambda [m per unit of intensity]; DESIGN.md, "RGB-D ICP"

_WS = {}


def _workspace(dev, H, W, kind="sb_icp_workspace_bytes"):
    key = (dev, H, W) if kind == "sb_icp_workspace_bytes" else (dev, H, W, kind)
    ws = _WS.get(key)
    if ws is None:
        with _lib.on_device(dev):
            nb = _lib.nbytes(kind, H, W)
        ws = _WS[key] = torch.empty(nb, dtype=torch.uint8, device=dev)
    return ws


def _intrinsics(K):
    K = np.asarray(K.detach().cpu() if isinstance(K, torch.Tensor) else K, dtype=np.float64)
    return float(K[0, 0]), float(K[1, 1]), float(K[0, 2]), float(K[1, 2])


def _f32(x, dev):
    return x.to(dev, torch.float32).contiguous()


def align(model_depth_sil, data_depth, intrinsics, w2c_prev, w2c_init, iters=DEFAULT_ITERS):
    """Frame t's w2c from the map's depth/silhouette render at frame t-1 and frame t's depth.

    model_depth_sil [C>=2,H,W]: channels 0 and 1 are depth_acc and silhouette of the render at w2c_prev;
    data_depth [H,W] or [1,H,W]: frame t's depth (<= 0, NaN or inf: no measurement); intrinsics: 3x3 pinhole, read on
    the host (pass a CPU array inside a captured region); w2c_prev, w2c_init [4,4]: frame t-1's pose and frame t's
    guess; iters: iterations of levels 0, 1, 2.  Returns (w2c [4,4] float32, stats [STATS] float64) on the device:
    w2c is the ICP pose if it passed the acceptance test, else w2c_init.  Workspaces are kept per (device, H, W)."""
    for name, t in (("model_depth_sil", model_depth_sil), ("data_depth", data_depth), ("w2c_prev", w2c_prev),
                    ("w2c_init", w2c_init)):
        if not isinstance(t, torch.Tensor):
            raise TypeError("%s must be a tensor" % name)
    _lib.need_cuda("icp.align", model_depth_sil, data_depth, w2c_prev, w2c_init)
    dev = model_depth_sil.device
    if dev.index is None:
        dev = torch.device("cuda", torch.cuda.current_device())
    if model_depth_sil.dim() != 3 or model_depth_sil.shape[0] < 2:
        raise ValueError("model_depth_sil must be [C>=2,H,W], got %s" % (tuple(model_depth_sil.shape),))
    H, W = model_depth_sil.shape[1:]
    if data_depth.numel() != H * W or tuple(data_depth.shape[-2:]) != (H, W):
        raise ValueError("data_depth %s does not match the render's %dx%d" % (tuple(data_depth.shape), H, W))
    if tuple(w2c_prev.shape) != (4, 4) or tuple(w2c_init.shape) != (4, 4):
        raise ValueError("w2c_prev and w2c_init must be [4,4]")
    if len(iters) != LEVELS or any(int(i) != i or not 0 <= i <= 1000 for i in iters):
        raise ValueError("iters must be %d integers in [0, 1000], got %r" % (LEVELS, iters))
    fx, fy, cx, cy = _intrinsics(intrinsics)
    ds = _f32(model_depth_sil[:2], dev)
    ws = _workspace(dev, H, W)
    out = torch.empty(4, 4, dtype=torch.float32, device=dev)
    stats = torch.empty(STATS, dtype=torch.float64, device=dev)
    it = (ctypes.c_int * LEVELS)(*[int(i) for i in iters])
    _lib.call("sb_icp_align", H, W, ds, _f32(data_depth, dev), fx, fy, cx, cy, _f32(w2c_prev, dev),
              _f32(w2c_init, dev), it, ws, ws.numel(), out, stats, device=dev)
    return out, stats


def align_rgbd(model_depth_sil, model_rgb, data_depth, data_rgb, intrinsics, w2c_prev, w2c_init, iters=DEFAULT_ITERS,
               weight=DEFAULT_WEIGHT):
    """`align` with a photometric term (sb_rgbd_icp_align): model_rgb [3,H,W] is the map's RGB render at w2c_prev,
    data_rgb [3,H,W] frame t's colour, weight (lambda >= 0, metres per unit of intensity) scales the intensity
    residuals against the point-to-plane ones.  Returns (w2c [4,4] float32, stats [RGBD_STATS] float64) on the device;
    with weight 0 both equal align's (stats 0..35) bit for bit.  Workspaces are kept per (device, H, W)."""
    for name, t in (("model_depth_sil", model_depth_sil), ("model_rgb", model_rgb), ("data_depth", data_depth),
                    ("data_rgb", data_rgb), ("w2c_prev", w2c_prev), ("w2c_init", w2c_init)):
        if not isinstance(t, torch.Tensor):
            raise TypeError("%s must be a tensor" % name)
    _lib.need_cuda("icp.align_rgbd", model_depth_sil, model_rgb, data_depth, data_rgb, w2c_prev, w2c_init)
    dev = model_depth_sil.device
    if dev.index is None:
        dev = torch.device("cuda", torch.cuda.current_device())
    if model_depth_sil.dim() != 3 or model_depth_sil.shape[0] < 2:
        raise ValueError("model_depth_sil must be [C>=2,H,W], got %s" % (tuple(model_depth_sil.shape),))
    H, W = model_depth_sil.shape[1:]
    if data_depth.numel() != H * W or tuple(data_depth.shape[-2:]) != (H, W):
        raise ValueError("data_depth %s does not match the render's %dx%d" % (tuple(data_depth.shape), H, W))
    for name, t in (("model_rgb", model_rgb), ("data_rgb", data_rgb)):
        if tuple(t.shape) != (3, H, W):
            raise ValueError("%s must be [3,%d,%d], got %s" % (name, H, W, tuple(t.shape)))
    if tuple(w2c_prev.shape) != (4, 4) or tuple(w2c_init.shape) != (4, 4):
        raise ValueError("w2c_prev and w2c_init must be [4,4]")
    if len(iters) != LEVELS or any(int(i) != i or not 0 <= i <= 1000 for i in iters):
        raise ValueError("iters must be %d integers in [0, 1000], got %r" % (LEVELS, iters))
    if isinstance(weight, bool) or not (isinstance(weight, (int, float)) and math.isfinite(weight) and weight >= 0):
        raise ValueError("weight must be a finite number >= 0, got %r" % (weight,))
    fx, fy, cx, cy = _intrinsics(intrinsics)
    ws = _workspace(dev, H, W, "sb_rgbd_icp_workspace_bytes")
    out = torch.empty(4, 4, dtype=torch.float32, device=dev)
    stats = torch.empty(RGBD_STATS, dtype=torch.float64, device=dev)
    it = (ctypes.c_int * LEVELS)(*[int(i) for i in iters])
    _lib.call("sb_rgbd_icp_align", H, W, _f32(model_depth_sil[:2], dev), _f32(model_rgb, dev), _f32(data_depth, dev),
              _f32(data_rgb, dev), fx, fy, cx, cy, _f32(w2c_prev, dev), _f32(w2c_init, dev), it, float(weight), ws,
              ws.numel(), out, stats, device=dev)
    return out, stats


def export_level_rgbd(H, W, level, device):
    """The grey maps of `level` from the latest align_rgbd on (device, H, W): dict(model_grey, data_grey [H_l,W_l],
    model_grad [2,H_l,W_l], photo uint8 [H_l,W_l]) and the geometric maps of export_level, on the device."""
    dev = torch.device(device)
    ws = _WS[(dev, H, W, "sb_rgbd_icp_workspace_bytes")]
    h, w = H >> level, W >> level
    o = dict(model_grey=torch.empty(h, w, device=dev), data_grey=torch.empty(h, w, device=dev),
             model_grad=torch.empty(2, h, w, device=dev), photo=torch.empty(h, w, dtype=torch.uint8, device=dev))
    _lib.call("sb_rgbd_icp_export", H, W, ws, ws.numel(), int(level), o["model_grey"], o["data_grey"],
              o["model_grad"], o["photo"], device=dev)
    g = dict(model_depth=torch.empty(h, w, device=dev), data_depth=torch.empty(h, w, device=dev),
             model_vertex=torch.empty(3, h, w, device=dev), model_normal=torch.empty(3, h, w, device=dev),
             data_vertex=torch.empty(3, h, w, device=dev), assoc=torch.empty(h, w, dtype=torch.uint8, device=dev))
    _lib.call("sb_icp_export", H, W, ws, ws.numel(), int(level), g["model_depth"], g["data_depth"], g["model_vertex"],
              g["model_normal"], g["data_vertex"], g["assoc"], device=dev)
    return dict(g, **o)


def export_level(H, W, level, device):
    """The maps of `level` from the latest align on (device, H, W): dict(model_depth, data_depth [H_l,W_l],
    model_vertex, model_normal, data_vertex [3,H_l,W_l], assoc uint8 [H_l,W_l]), on the device (for inspection)."""
    dev = torch.device(device)
    ws = _WS[(dev, H, W)]
    h, w = H >> level, W >> level
    o = dict(model_depth=torch.empty(h, w, device=dev), data_depth=torch.empty(h, w, device=dev),
             model_vertex=torch.empty(3, h, w, device=dev), model_normal=torch.empty(3, h, w, device=dev),
             data_vertex=torch.empty(3, h, w, device=dev), assoc=torch.empty(h, w, dtype=torch.uint8, device=dev))
    _lib.call("sb_icp_export", H, W, ws, ws.numel(), int(level), o["model_depth"], o["data_depth"], o["model_vertex"],
              o["model_normal"], o["data_vertex"], o["assoc"], device=dev)
    return o


def read_stats(stats):
    """Host dict of a stats record (one device read): accepted, inlier_frac, rms, inliers, valid, pivot_ratio,
    skipped (some Gauss-Newton update was skipped); for an align_rgbd record also photo_pairs and photo_rms."""
    s = stats.detach().cpu().numpy()
    d = dict(accepted=bool(s[0]), inlier_frac=float(s[1]), rms=float(s[2]), inliers=int(s[3]), valid=int(s[4]),
             pivot_ratio=float(s[5]), skipped=bool(s[6]))
    if len(s) >= RGBD_STATS:
        d.update(photo_pairs=int(s[36]), photo_rms=float(s[37]))
    return d


def model_depth_sil(params, t, frame, render=None, fused=None):
    """The map's depth/silhouette render [3,H,W] at frame t's pose in `params`, with `frame`'s camera and first-frame
    w2c (no gradient)."""
    render = M.default_render if render is None else render
    fused = (params["means3D"].is_cuda and render is M.default_render) if fused is None else fused
    with torch.no_grad():
        _, ds, _, _ = M._render_pair(params, dict(id=t, cam=frame["cam"], w2c=frame["w2c"]), render, fused,
                                     camera_grad=False)
    return ds


def model_render(params, t, frame, render=None, fused=None):
    """(RGB [3,H,W], depth/silhouette [3,H,W]) renders of the map at frame t's pose in `params`, with `frame`'s camera
    and first-frame w2c (no gradient)."""
    render = M.default_render if render is None else render
    fused = (params["means3D"].is_cuda and render is M.default_render) if fused is None else fused
    with torch.no_grad():
        im, ds, _, _ = M._render_pair(params, dict(id=t, cam=frame["cam"], w2c=frame["w2c"]), render, fused,
                                      camera_grad=False)
    return im, ds


def init_pose(params, frame, t, intrinsics, render=None, fused=None, iters=DEFAULT_ITERS, photometric=False):
    """Refines column t of params' cam_unnorm_rots / cam_trans (holding the constant-velocity guess) by `align`
    (with `photometric`, `align_rgbd` at DEFAULT_WEIGHT against the map's RGB render too) against the map rendered at
    column t - 1, in place; a rejected alignment leaves the column as it was.  The quaternion is normalised, with the
    sign nearest column t - 1's.  Returns the stats record (device)."""
    rots, trans = params["cam_unnorm_rots"], params["cam_trans"]
    with torch.no_grad():
        w2c0 = frame["w2c"].float()
        prev = w2c0 @ M.camera_w2c(rots[..., t - 1], trans[..., t - 1])[0]
        guess = w2c0 @ M.camera_w2c(rots[..., t], trans[..., t])[0]
        if photometric:
            im, ds = model_render(params, t - 1, frame, render, fused)
            w2c, stats = align_rgbd(ds, im, frame["depth"], frame["im"], intrinsics, prev, guess, iters)
        else:
            ds = model_depth_sil(params, t - 1, frame, render, fused)
            w2c, stats = align(ds, frame["depth"], intrinsics, prev, guess, iters)
        inv0 = torch.eye(4, device=w2c0.device)                  # w2c0 is rigid: its inverse needs no solver
        inv0[:3, :3] = w2c0[:3, :3].T
        inv0[:3, 3] = -(w2c0[:3, :3].T @ w2c0[:3, 3])
        rel = inv0 @ w2c
        q = F.normalize(M.matrix_to_quaternion(rel[:3, :3]), dim=0)
        q = torch.where((q * F.normalize(rots[0, :, t - 1], dim=0)).sum() < 0, -q, q)
        ok = stats[0] > 0
        rots[0, :, t] = torch.where(ok, q, rots[0, :, t])
        trans[0, :, t] = torch.where(ok, rel[:3, 3], trans[0, :, t])
    return stats
