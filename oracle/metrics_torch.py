"""TEST INFRASTRUCTURE ONLY (imported by tests/ and tools/ -- never by the product path).

Plain-torch restatement of SplaTAM's final-evaluation metrics, device-agnostic, float64 by default; the checker for
csrc/eval_metrics.cu.  tests/golden/eval/ref_eval.npz pins it against the reference's own `eval`.

  frame_metrics   R/utils/eval_helpers.py:463-505 (masks, weighted images, depth errors) and calc_psnr
                  (R/utils/slam_external.py:49-51)
  ms_ssim         pytorch_msssim.ms_ssim(X, Y, data_range, size_average), which eval_helpers.py:482 calls: 11-tap
                  sigma-1.5 Gaussian window applied separably as a VALID convolution, 5 levels, 2x2 average pool with
                  padding (H % 2, W % 2) between levels, relu(cs) of levels 0-3 and relu(ssim) of level 4 raised to
                  the weights below and multiplied.
"""
import torch
import torch.nn.functional as F

MS_SSIM_WEIGHTS = (0.0448, 0.2856, 0.3001, 0.2363, 0.1333)


def frame_metrics(im, depth_sil, gt_im, gt_depth, sil_thres, use_presence, dtype=torch.float64):
    """dict(psnr, depth_rmse, depth_l1, n_valid, n_mask, weighted_im, weighted_gt) of one frame.  use_presence:
    mapping_iters == 0 and not add_new_gaussians.  "depth_rmse" is the reference's sqrt(x^2) taken element-wise, a
    masked mean absolute error; it is reproduced as defined."""
    im, depth_sil, gt_im, gt_depth = (t.to(dtype) for t in (im, depth_sil, gt_im, gt_depth))
    valid = (gt_depth > 0).to(dtype)                          # [1,H,W]
    presence = (depth_sil[1] > sil_thres).to(dtype)           # [H,W]
    mask = presence * valid if use_presence else valid
    w_im, w_gt = im * mask, gt_im * mask
    mse = ((w_im - w_gt) ** 2).reshape(3, -1).mean(1)
    psnr = (20 * torch.log10(1.0 / torch.sqrt(mse))).mean()
    e = depth_sil[0:1] * valid - gt_depth
    if use_presence:
        e = e * presence
    n_valid = valid.sum()
    return dict(psnr=psnr, depth_rmse=(torch.sqrt(e ** 2) * valid).sum() / n_valid,
                depth_l1=(torch.abs(e) * valid).sum() / n_valid, n_valid=n_valid, n_mask=mask.sum(),
                weighted_im=w_im, weighted_gt=w_gt)


def _window(dtype, device):
    coords = torch.arange(11, dtype=dtype, device=device) - 5
    g = torch.exp(-(coords ** 2) / (2 * 1.5 ** 2))
    return g / g.sum()


def _filter(x, g):
    C = x.shape[1]
    x = F.conv2d(x, g.reshape(1, 1, 1, -1).expand(C, 1, 1, 11), groups=C)      # along W, valid
    return F.conv2d(x, g.reshape(1, 1, -1, 1).expand(C, 1, 11, 1), groups=C)   # along H, valid


def ms_ssim(x, y, data_range=1.0, size_average=True, dtype=torch.float64):
    """MS-SSIM of [N,C,H,W] images computed in `dtype`: the mean with size_average, else the [N,C] values."""
    if min(x.shape[-2:]) <= 160:
        raise ValueError("MS-SSIM needs a smaller side > 160 (11-tap window over 5 levels)")
    x, y = x.to(dtype), y.to(dtype)
    g = _window(dtype, x.device)
    C1, C2 = (0.01 * data_range) ** 2, (0.03 * data_range) ** 2
    vals = []
    for level in range(len(MS_SSIM_WEIGHTS)):
        mu1, mu2 = _filter(x, g), _filter(y, g)
        s1, s2, s12 = _filter(x * x, g) - mu1 * mu1, _filter(y * y, g) - mu2 * mu2, _filter(x * y, g) - mu1 * mu2
        cs_map = (2 * s12 + C2) / (s1 + s2 + C2)
        ssim_map = (2 * mu1 * mu2 + C1) / (mu1 * mu1 + mu2 * mu2 + C1) * cs_map
        if level < len(MS_SSIM_WEIGHTS) - 1:
            vals.append(torch.relu(cs_map.flatten(2).mean(-1)))
            pad = [s % 2 for s in x.shape[2:]]
            x, y = F.avg_pool2d(x, 2, padding=pad), F.avg_pool2d(y, 2, padding=pad)
        else:
            vals.append(torch.relu(ssim_map.flatten(2).mean(-1)))
    w = torch.tensor(MS_SSIM_WEIGHTS, dtype=dtype, device=x.device).reshape(-1, 1, 1)
    out = torch.prod(torch.stack(vals) ** w, dim=0)
    return out.mean() if size_average else out
