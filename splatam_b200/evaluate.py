"""SplaTAM's final evaluation (R/utils/eval_helpers.py:408-623, `eval`) on the GPU: per-frame PSNR, MS-SSIM, depth
errors and the ATE of the estimated trajectory, with the metric kernels of csrc/eval_metrics.cu.

The reference renders every evaluated frame twice, computes PSNR and the depth errors in PyTorch and copies both
weighted images to the host for pytorch_msssim on the CPU.  Here the renders go through the same front end as
mapping and tracking (`mapping._render_pair`), one kernel pass per frame writes the masked images and the PSNR /
depth sums, MS-SSIM runs on the device, and the per-frame metrics stay on the device until one read at the end.
`evaluate_nvs` is the reference's novel-view evaluation (eval_helpers.py:626-841, `eval_nvs`) over a test split: the
same metrics on held-out views rendered at their ground-truth poses, averaged over the views the map covers.
LPIPS is not computed (it needs pretrained AlexNet weights): the result carries ``lpips: None``.  CUDA only; no CPU
fallback."""
import os

import numpy as np
import torch

from . import _lib
from . import mapping as M

# columns of the per-frame metric rows: the five that sb_frame_metrics writes, then MS-SSIM
_PSNR, _RMSE, _L1, _NVALID, _NMASK, _SSIM = range(6)


def _ms_ssim_into(x, y, data_range, per_channel, mean, ws=None):
    """Enqueues sb_ms_ssim on contiguous float32 [N,C,H,W] CUDA tensors; `per_channel` / `mean`: float64 device
    tensors or None."""
    N, C, H, W = x.shape
    if ws is None:
        ws = torch.empty(_lib.nbytes("sb_ms_ssim_workspace_bytes", N, C, H, W), dtype=torch.uint8, device=x.device)
    _lib.call("sb_ms_ssim", x, y, N, C, H, W, float(data_range), ws, ws.numel(), per_channel, mean, device=x.device)


def ms_ssim(x, y, data_range=1.0, size_average=True):
    """MS-SSIM of two [N,C,H,W] CUDA images as pytorch_msssim.ms_ssim defines it (11-tap sigma-1.5 Gaussian window,
    valid filtering, 5 levels with weights 0.0448, 0.2856, 0.3001, 0.2363, 0.1333), computed in double on the device.
    size_average=True returns the mean (a float64 0-d tensor); otherwise the float64 [N,C] values (pytorch_msssim
    averages those over channels).  The smaller image side must exceed 160."""
    _lib.need_cuda("ms_ssim", x, y)
    if x.dim() != 4 or x.shape != y.shape:
        raise _lib.SplatamB200Error("ms_ssim expects two [N,C,H,W] images of the same shape, got %s and %s"
                                    % (tuple(x.shape), tuple(y.shape)))
    if min(x.shape[-2:]) <= 160:
        raise _lib.SplatamB200Error("ms_ssim needs a smaller image side > 160, got %s" % (tuple(x.shape),))
    x, y = x.detach().float().contiguous(), y.detach().float().contiguous()
    N, C = x.shape[:2]
    if size_average:
        mean = torch.empty((), dtype=torch.float64, device=x.device)
        _ms_ssim_into(x, y, data_range, None, mean)
        return mean
    out = torch.empty(N, C, dtype=torch.float64, device=x.device)
    _ms_ssim_into(x, y, data_range, out, None)
    return out


def select_frames(num_frames, eval_every=1):
    """Indices the reference evaluates: frame 0, then every frame with (t + 1) % eval_every == 0
    (eval_helpers.py:447-448)."""
    return [t for t in range(num_frames) if t == 0 or (t + 1) % eval_every == 0]


def trajectory_ate(params, first_w2c, gt_w2c):
    """ATE of the estimated trajectory (eval_helpers.py:545-575): estimate 0 is the first frame's w2c, estimate t the
    w2c of the normalised camera quaternion and translation of frame t; frames t >= 1 whose ground-truth w2c contains
    NaN are skipped; slam.ate_horn aligns and averages.  Host code over the pose tensors."""
    from .slam import ate_horn
    rots, trans = params["cam_unnorm_rots"].detach(), params["cam_trans"].detach()
    gt = [torch.as_tensor(m) for m in gt_w2c]
    est, ref = [first_w2c], [gt[0]]
    for t in range(1, rots.shape[-1]):
        if torch.isnan(gt[t]).any():
            continue
        est.append(M.camera_w2c(rots[..., t], trans[..., t])[0])
        ref.append(gt[t])
    return ate_horn(ref, est)


def _check_inputs(name, params, frames):
    _lib.need_cuda(name, params["means3D"], frames[0]["im"])
    H, W = frames[0]["im"].shape[-2:]
    if min(H, W) <= 160:
        raise _lib.SplatamB200Error("%s: MS-SSIM needs a smaller image side > 160, got %dx%d" % (name, W, H))
    return H, W


def _score_frames(params, frames, ids, cam, sil_thres, use_presence, render, fused, at_gt_pose=False,
                  count_holes=False):
    """Renders frames[t] for t in `ids` and scores each with sb_frame_metrics and MS-SSIM: float64 device rows
    [len(ids), 6] (columns _PSNR .. _SSIM).  at_gt_pose: render at the frame's gt_w2c instead of its estimated pose.
    count_holes: also returns [len(ids), 6] rows of a presence-masked sb_frame_metrics call into scratch images, whose
    _NVALID - _NMASK is the number of valid-depth pixels the silhouette leaves uncovered (None otherwise)."""
    render = M.default_render if render is None else render
    if fused is None:
        fused = render is M.default_render
    dev = params["means3D"].device
    H, W = frames[0]["im"].shape[-2:]
    metrics = torch.zeros(len(ids), 6, dtype=torch.float64, device=dev)
    presence = torch.zeros_like(metrics) if count_holes else None
    w_im = torch.empty(3, H, W, dtype=torch.float32, device=dev)
    w_gt = torch.empty_like(w_im)
    ws_frame = torch.empty(_lib.nbytes("sb_frame_metrics_workspace_bytes", H, W), dtype=torch.uint8, device=dev)
    ws_ssim = torch.empty(_lib.nbytes("sb_ms_ssim_workspace_bytes", 1, 3, H, W), dtype=torch.uint8, device=dev)
    with torch.no_grad(), torch.cuda.device(dev):
        for k, t in enumerate(ids):
            fr = dict(frames[t], cam=cam)
            if at_gt_pose:
                fr["pose"] = M.gt_pose(fr["gt_w2c"].to(dev).float())
            im, depth_sil, _, _ = M._render_pair(params, fr, render, fused, camera_grad=False)
            im, depth_sil = im.float().contiguous(), depth_sil.float().contiguous()
            gt_im, gt_d = fr["im"].float().contiguous(), fr["depth"].float().contiguous()
            _lib.call("sb_frame_metrics", im, depth_sil, gt_im, gt_d, H, W, float(sil_thres), use_presence, w_im, w_gt,
                      ws_frame, ws_frame.numel(), metrics[k], device=dev)
            _ms_ssim_into(w_im[None], w_gt[None], 1.0, None, metrics[k, _SSIM], ws_ssim)
            if count_holes:
                if use_presence:
                    presence[k].copy_(metrics[k])
                else:
                    _lib.call("sb_frame_metrics", im, depth_sil, gt_im, gt_d, H, W, float(sil_thres), 1, w_im, w_gt,
                              ws_frame, ws_frame.numel(), presence[k], device=dev)
    return metrics, presence


def _per_frame(m):
    return dict(psnr_per_frame=m[:, _PSNR], ms_ssim_per_frame=m[:, _SSIM], depth_rmse_per_frame=m[:, _RMSE],
                depth_l1_per_frame=m[:, _L1], valid_pixels=m[:, _NVALID].astype(np.int64),
                mask_pixels=m[:, _NMASK].astype(np.int64))


def _write_lists(out_dir, out):
    os.makedirs(out_dir, exist_ok=True)
    for name, key in (("psnr", "psnr_per_frame"), ("rmse", "depth_rmse_per_frame"), ("l1", "depth_l1_per_frame"),
                      ("ssim", "ms_ssim_per_frame")):
        np.savetxt(os.path.join(out_dir, name + ".txt"), out[key])


def evaluate(params, frames, cam, sil_thres, mapping_iters, add_new_gaussians, eval_every=1, gt_w2c=None, fused=None,
             render=None, out_dir=None):
    """The reference's final `eval` over this repo's frame dicts (id, im [3,H,W] in [0,1], depth [1,H,W], w2c = the
    first frame's w2c, as slam.render_frame builds them).  `params`: the final Gaussians plus cam_unnorm_rots /
    cam_trans [.., T]; `cam`: the raster settings; frames are evaluated as `select_frames` picks them.

    Masks as in the reference: valid = gt depth > 0; when mapping_iters == 0 and not add_new_gaussians the images and
    the depth error are also masked by silhouette > sil_thres.  Rendered images are not clamped.
      psnr        mean over the three channels of the per-channel PSNR of the weighted images, each MSE taken over
                  all H*W pixels (calc_psnr)
      ms_ssim     MS-SSIM of the weighted images (`ms_ssim`)
      depth_rmse  sum(sqrt(e^2) * valid) / sum(valid): the reference takes sqrt(x^2) element-wise, so this is a
                  masked mean absolute error; it is reported as the reference defines it
      depth_l1    sum(|e| * valid) / sum(valid)
      ate         `trajectory_ate` against gt_w2c (a list of T ground-truth w2c matrices), None without it
      lpips       None (not computed)
    Returns those averages plus frame_ids and the per-frame arrays psnr_per_frame, ms_ssim_per_frame,
    depth_rmse_per_frame, depth_l1_per_frame, valid_pixels, mask_pixels.  `out_dir`: also writes psnr.txt, rmse.txt,
    l1.txt and ssim.txt as the reference does (np.savetxt, one value per evaluated frame).
    fused / render: as for mapping (`mapping._render_pair`); fused defaults to the fast path on CUDA."""
    _check_inputs("evaluate", params, frames)
    ids = select_frames(len(frames), eval_every)
    use_presence = int(mapping_iters == 0 and not add_new_gaussians)
    metrics, _ = _score_frames(params, frames, ids, cam, sil_thres, use_presence, render, fused)
    m = metrics.cpu().numpy()                    # the one device-to-host read
    out = dict(frame_ids=[int(frames[t]["id"]) for t in ids], **_per_frame(m))
    out.update(psnr=float(m[:, _PSNR].mean()), ms_ssim=float(m[:, _SSIM].mean()),
               depth_rmse=float(m[:, _RMSE].mean()), depth_l1=float(m[:, _L1].mean()), lpips=None,
               ate=None if gt_w2c is None else trajectory_ate(params, frames[0]["w2c"], gt_w2c))
    if out_dir is not None:
        _write_lists(out_dir, out)
    return out


def select_nvs_frames(num_frames, eval_every=1):
    """Indices the reference's eval_nvs evaluates in a test split: frame 0 (the first train frame) never; frame t >= 1
    (test view k = t - 1) when k == 0 or (k + 1) % eval_every == 0 (eval_helpers.py:666-669)."""
    return [t for t in range(1, num_frames) if t == 1 or t % eval_every == 0]


def evaluate_nvs(params, frames, cam, sil_thres, mapping_iters, add_new_gaussians, eval_every=1, fused=None,
                 render=None, out_dir=None):
    """The reference's novel-view evaluation `eval_nvs` over a test split (datasets.RGBDSequence(..., split="test"):
    frame 0 is the first train frame, frames 1.. the held-out views, each with its ground-truth `gt_w2c`).  Frames are
    picked by `select_nvs_frames` and rendered at gt_w2c -- the means transformed by it, anisotropic rotations
    composed with its normalised quaternion -- not at an estimated pose; `params` needs no camera tensors.

    Masks and per-frame metrics are those of `evaluate`.  A view is valid unless its holes -- pixels with gt depth > 0
    and silhouette <= sil_thres -- exceed 0.1 % of the image (holes * 1000 > H * W; the reference's float32 percentage
    test agrees at the datasets' image sizes).  Returns the averages psnr, ms_ssim, depth_rmse and depth_l1 over the
    valid views (NaN when none is valid), lpips None, frame_ids (indices into `frames`), the per-frame arrays of
    `evaluate` over every evaluated view, hole_pixels and valid_nvs_frames (bool).  `out_dir`: also writes psnr.txt,
    rmse.txt, l1.txt and ssim.txt over every evaluated view and valid_nvs_frames.npy, as the reference does."""
    H, W = _check_inputs("evaluate_nvs", params, frames)
    ids = select_nvs_frames(len(frames), eval_every)
    use_presence = int(mapping_iters == 0 and not add_new_gaussians)
    metrics, presence = _score_frames(params, frames, ids, cam, sil_thres, use_presence, render, fused,
                                      at_gt_pose=True, count_holes=True)
    m, p = torch.stack([metrics, presence]).cpu().numpy()          # the one device-to-host read
    holes = (p[:, _NVALID] - p[:, _NMASK]).astype(np.int64)
    valid = holes * 1000 <= H * W
    out = dict(frame_ids=[int(frames[t]["id"]) for t in ids], hole_pixels=holes, valid_nvs_frames=valid,
               **_per_frame(m))
    avg = lambda c: float(m[valid, c].mean()) if valid.any() else float("nan")
    out.update(psnr=avg(_PSNR), ms_ssim=avg(_SSIM), depth_rmse=avg(_RMSE), depth_l1=avg(_L1), lpips=None)
    if out_dir is not None:
        _write_lists(out_dir, out)
        np.save(os.path.join(out_dir, "valid_nvs_frames.npy"), valid)
    return out
