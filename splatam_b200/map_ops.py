"""Map maintenance of the SLAM loop over libsplatam_b200.so (csrc/map_ops.cu): pruning and growing the Gaussian
set as mask -> scan -> scatter kernels.  Host-side mirror of the reference functions

* ``prune_gaussians`` / ``remove_points``  (R/utils/slam_external.py:144-190)
* ``add_new_gaussians`` / ``get_pointcloud`` / ``initialize_new_params``  (R/scripts/splatam.py:67-118,348-420)

CUDA only; there is no CPU fallback (the parity tests compare against oracle/map_ops_torch.py)."""
import ctypes

import torch

from . import _lib


def prune_mask(logit_opacities, log_scales, opacity_threshold, big_threshold=None):
    """bool[P] keep mask: not (sigmoid(logit) < opacity_threshold or exp(log_scales).max(1) > big_threshold)."""
    _lib.need_cuda("prune_mask", logit_opacities)
    lo = logit_opacities.detach().contiguous().float()
    ls = log_scales.detach().contiguous().float()
    P = lo.shape[0]
    keep = torch.empty(P, dtype=torch.uint8, device=lo.device)
    _lib.call("sb_prune_mask", P, lo, ls, ls.shape[1] if ls.dim() > 1 else 1, float(opacity_threshold),
              float(big_threshold) if big_threshold else 0.0, keep, device=lo.device)
    return keep.bool()


def compact_plan(mask):
    """Exclusive scan of a bool/uint8 mask -> (mask_u8, dst_index uint32-as-int32 tensor, count).  Synchronises."""
    _lib.need_cuda("compact_plan", mask)
    m = mask.contiguous().view(torch.uint8) if mask.dtype == torch.bool else mask.contiguous().to(torch.uint8)
    n = m.numel()
    dst = torch.empty(max(n, 1), dtype=torch.int32, device=m.device)
    temp = torch.empty(_lib.nbytes("sb_compact_plan_bytes", n), dtype=torch.uint8, device=m.device)
    count = ctypes.c_int()
    _lib.call("sb_compact_plan", n, m, dst, temp, temp.numel(), ctypes.byref(count), device=m.device)
    return m, dst, count.value


def compact_flat(flat, P, widths, mask_u8, dst_index, P_new):
    """Kept rows of a packed buffer [w0*P | w1*P | ...] -> new packed buffer with P_new rows."""
    _lib.need_cuda("compact_flat", flat)
    assert flat.is_contiguous() and flat.dtype == torch.float32 and flat.numel() == sum(widths) * P
    out = torch.empty(sum(widths) * P_new, dtype=torch.float32, device=flat.device)
    w = (ctypes.c_int * len(widths))(*[int(x) for x in widths])
    _lib.call("sb_compact_flat", P, P_new, mask_u8, dst_index, len(widths), w, flat, out, device=flat.device)
    return out


def densify_accumulate(means2D_grad, seen, accum, denom):
    """accum[seen] += norm(means2D_grad[seen, :2], dim=-1); denom[seen] += 1, in place and in one launch with no host
    synchronisation (densify's statistic, R/utils/slam_external.py:200-204).  means2D_grad: contiguous float32 [P, >=2];
    seen: bool [P]; accum, denom: contiguous float32 [P]."""
    _lib.need_cuda("densify_accumulate", means2D_grad, seen, accum, denom)
    P = accum.shape[0]
    g = means2D_grad.detach()
    if not (g.is_contiguous() and g.dtype == torch.float32 and g.dim() == 2 and g.shape[0] == P and g.shape[1] >= 2):
        raise _lib.SplatamB200Error("densify_accumulate expects a contiguous float32 [%d, >=2] gradient, got %s %s"
                                    % (P, g.dtype, tuple(g.shape)))
    if seen.dtype != torch.bool or seen.numel() != P or not seen.is_contiguous():
        raise _lib.SplatamB200Error("densify_accumulate expects a contiguous bool [%d] seen mask" % P)
    for t in (accum, denom):
        if t.dtype != torch.float32 or t.numel() != P or not t.is_contiguous():
            raise _lib.SplatamB200Error("densify_accumulate expects contiguous float32 [%d] accum and denom" % P)
    _lib.call("sb_densify_accumulate", P, g, g.shape[1], seen.view(torch.uint8), accum, denom, device=accum.device)


def depth_error(depth_sil, gt_depth):
    """|gt - depth| * (gt > 0) over the frame (R/scripts/splatam.py:391)."""
    _lib.need_cuda("depth_error", depth_sil)
    ds, gt = depth_sil.detach().contiguous().float(), gt_depth.detach().contiguous().float()
    H, W = ds.shape[-2:]
    err = torch.empty(H, W, dtype=torch.float32, device=ds.device)
    _lib.call("sb_depth_error", H, W, ds, gt, err, device=ds.device)
    return err


def new_gaussian_mask(depth_sil, gt_depth, sil_thres, depth_err_thres):
    """bool[H*W] non-presence mask of add_new_gaussians (already AND-ed with gt_depth > 0)."""
    _lib.need_cuda("new_gaussian_mask", depth_sil)
    ds, gt = depth_sil.detach().contiguous().float(), gt_depth.detach().contiguous().float()
    H, W = ds.shape[-2:]
    mask = torch.empty(H * W, dtype=torch.uint8, device=ds.device)
    _lib.call("sb_new_gaussian_mask", H, W, ds, gt, float(sil_thres), float(depth_err_thres), mask, device=ds.device)
    return mask.bool()


def backproject(color, depth, intrinsics, w2c, mask=None, scale_dim=1, plan=None):
    """Pixels -> Gaussian rows (get_pointcloud + initialize_new_params).  intrinsics: 3x3 (tensor or nested list);
    w2c: 4x4 world-to-camera of the frame.  Returns dict(means3D, rgb_colors, unnorm_rotations, logit_opacities,
    log_scales) and mean_sq_dist, each with one row per selected pixel (row-major pixel order)."""
    _lib.need_cuda("backproject", color)
    dev = color.device
    color, depth = color.detach().contiguous().float(), depth.detach().contiguous().float()
    H, W = color.shape[-2:]
    K = torch.as_tensor(intrinsics, dtype=torch.float32).cpu()
    fx, fy, cx, cy = float(K[0][0]), float(K[1][1]), float(K[0][2]), float(K[1][2])
    c2w = torch.inverse(torch.as_tensor(w2c).detach().float()).cpu().contiguous()     # splatam.py:90 (4x4, tiny)
    c2w_host = (ctypes.c_float * 16)(*c2w.reshape(-1).tolist())
    if mask is None:
        m8, dst, n = None, None, H * W
    else:
        m8, dst, n = plan if plan is not None else compact_plan(mask.reshape(-1))
    means = torch.empty(n, 3, dtype=torch.float32, device=dev)
    rgb = torch.empty(n, 3, dtype=torch.float32, device=dev)
    ls = torch.empty(n, scale_dim, dtype=torch.float32, device=dev)
    msd = torch.empty(n, dtype=torch.float32, device=dev)
    if n > 0:
        _lib.call("sb_backproject", H, W, color, depth, fx, fy, cx, cy, c2w_host, m8, dst, scale_dim, means, rgb, ls,
                  msd, device=dev)
    rots = torch.zeros(n, 4, dtype=torch.float32, device=dev)
    rots[:, 0] = 1.0
    new = dict(means3D=means, rgb_colors=rgb, unnorm_rotations=rots,
               logit_opacities=torch.zeros(n, 1, dtype=torch.float32, device=dev), log_scales=ls)
    return new, msd


def new_gaussians_from_frame(depth_sil, frame, intrinsics, curr_w2c, sil_thres, scale_dim=1, exclude=None):
    """add_new_gaussians' selection + initialisation for one frame: `depth_sil` is the [3,H,W] depth/silhouette
    render of the current map at the frame's pose, `frame` holds `im` [3,H,W] and `depth` [1,H,W].  Pixels set in
    `exclude` (bool [H,W]) are not selected.  Returns (new parameter rows, count)."""
    err = depth_error(depth_sil, frame["depth"])
    thres = 50.0 * float(err.median())               # splatam.py:392 (torch.median = lower middle element)
    mask = new_gaussian_mask(depth_sil, frame["depth"], sil_thres, thres)
    if exclude is not None:
        mask = mask & ~exclude.reshape(-1)
    plan = compact_plan(mask)
    if plan[2] == 0:
        return None, 0
    new, _ = backproject(frame["im"], frame["depth"], intrinsics, curr_w2c, mask=mask, scale_dim=scale_dim, plan=plan)
    return new, plan[2]
