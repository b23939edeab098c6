"""TEST INFRASTRUCTURE ONLY (imported by tests/ and tools/ -- never by the product path).

Plain-torch restatements of the per-iteration training ops, device-agnostic, float64 by default; gradients come from
autograd.  The checker for csrc/train_ops.cu and csrc/prepare.cu.  tests/golden/glue/ref_glue.npz pins them against
the reference's own Python.

  image_loss   w_l1 mean|x - y| + w_ssim (1 - mean SSIM(x, y)): SSIM with an 11x11 Gaussian window (sigma 1.5, the
               1-D weights normalised in float32 as SplaTAM builds them), zero padding 5, C1 = 0.01^2, C2 = 0.03^2
  masked_l1    the validity / silhouette masked L1 terms of SplaTAM's get_loss: mask = gt depth > 0, depth not NaN,
               depth^2 channel - depth^2 not NaN [, silhouette > threshold], detached; mean or sum over the mask
  prepare      world -> camera-frame Gaussians and both rendervars (normalised rotations, sigmoid opacities, exp
               scales tiled to 3, depth colours [z, 1, z^2]) as functions of rel_w2c and the normalised camera
               quaternion; prepare_from_camera goes on through the unnormalised camera quaternion and translation
  adam         torch.optim.Adam over segments of a flat buffer with per-segment learning rates, skipped steps and
               learning-rate changes
"""
import math

import torch
import torch.nn.functional as F

SSIM_C1, SSIM_C2 = 0.01 ** 2, 0.03 ** 2


def ssim_window(dtype=torch.float64, device="cpu"):
    """[11,11] window: outer product of the 1-D Gaussian weights exp(-(i-5)^2 / (2 1.5^2)), normalised in float32.
    In float64 the product is exact, so it is the separable window the kernel applies."""
    g = torch.tensor([math.exp(-(i - 5) ** 2 / (2 * 1.5 ** 2)) for i in range(11)], dtype=torch.float32)
    g = (g / g.sum()).to(dtype=dtype, device=device)
    return g[:, None] @ g[None, :]


def ssim(x, y, dtype=torch.float64):
    """Mean SSIM of two [C,H,W] images computed in `dtype`."""
    x, y = x.to(dtype), y.to(dtype)
    C = x.shape[-3]
    w = ssim_window(dtype, x.device)[None, None].expand(C, 1, 11, 11).contiguous()
    conv = lambda t: F.conv2d(t, w, padding=5, groups=C)
    mu1, mu2 = conv(x), conv(y)
    mu1_sq, mu2_sq, mu12 = mu1.pow(2), mu2.pow(2), mu1 * mu2
    s1, s2, s12 = conv(x * x) - mu1_sq, conv(y * y) - mu2_sq, conv(x * y) - mu12
    return (((2 * mu12 + SSIM_C1) * (2 * s12 + SSIM_C2)) / ((mu1_sq + mu2_sq + SSIM_C1) * (s1 + s2 + SSIM_C2))).mean()


def image_loss(x, y, w_l1=0.8, w_ssim=0.2, dtype=torch.float64):
    """w_l1 mean|x - y| + w_ssim (1 - mean SSIM(x, y)) of two [C,H,W] images, in `dtype`."""
    xd, yd = x.to(dtype), y.to(dtype)
    return w_l1 * torch.abs(xd - yd).mean() + w_ssim * (1.0 - ssim(xd, yd, dtype))


def loss_mask(depth_sil, gt_depth, sil_thres=0.99, use_sil=False):
    """[1,H,W] bool mask of get_loss, evaluated in float32, the precision of the renders (a silhouette equal to
    float32(sil_thres) is not above it)."""
    depth_sil, gt_depth = depth_sil.detach().float(), gt_depth.float()
    depth = depth_sil[0:1]
    unc = depth_sil[2:3] - depth ** 2
    mask = (gt_depth > 0) & ~torch.isnan(depth) & ~torch.isnan(unc)
    if use_sil:
        mask = mask & (depth_sil[1] > sil_thres)
    return mask


def masked_l1(depth_sil, gt_depth, im=None, gt_im=None, sil_thres=0.99, use_sil=False, depth_mean=True,
              dtype=torch.float64):
    """(loss_depth, loss_im) in `dtype`: |gt_depth - depth| over the mask, its mean if depth_mean else its sum, and the
    sum of |gt_im - im| over the mask tiled to 3 channels (0 without an image).  An empty mask gives a NaN mean, a
    zero sum and zero gradients, as boolean indexing does."""
    mask = loss_mask(depth_sil, gt_depth, sil_thres, use_sil)
    ds, gd = depth_sil.to(dtype), gt_depth.to(dtype)
    ld = torch.abs(gd - ds[0:1])[mask]
    ld = ld.mean() if depth_mean else ld.sum()
    if im is None:
        return ld, torch.zeros((), dtype=dtype, device=ds.device)
    li = torch.abs(gt_im.to(dtype) - im.to(dtype))[mask.expand(3, -1, -1)].sum()
    return ld, li


def quat_mult(a, b):
    """Hamilton product of (w, x, y, z) quaternions, broadcast over rows."""
    aw, ax, ay, az = a.unbind(-1)
    bw, bx, by, bz = b.unbind(-1)
    return torch.stack([aw * bw - ax * bx - ay * by - az * bz, aw * bx + ax * bw + ay * bz - az * by,
                        aw * by - ax * bz + ay * bw + az * bx, aw * bz + ax * by - ay * bx + az * bw], -1)


def rotation_matrix(q):
    """3x3 rotation of a unit quaternion (w, x, y, z) of shape [4]."""
    w, x, y, z = q.unbind(-1)
    return torch.stack([torch.stack([1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)]),
                        torch.stack([2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)]),
                        torch.stack([2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)])])


def prepare(means3D, unnorm_rotations, logit_opacities, log_scales, rel_w2c, cam_rot, w2c0, dtype=torch.float64):
    """(means_cam [P,3], rotations [P,4], opacities [P,1], scales3 [P,3], depth_sil_colors [P,3]) in `dtype`.
    rel_w2c [4,4] maps world to camera; cam_rot [1,4] or [4] is the camera quaternion that rotates anisotropic
    Gaussians (F.normalize(cam_rot * F.normalize(q)), as the reference's rendervar normalises); isotropic
    rotations are F.normalize(q).  w2c0 [4,4] is the first frame's w2c: z is row 2 of w2c0 applied to means_cam."""
    d = lambda t: t.to(dtype)
    pts, rel, w0 = d(means3D), d(rel_w2c), d(w2c0)
    means_cam = pts @ rel[:3, :3].T + rel[:3, 3]
    q = F.normalize(d(unnorm_rotations), dim=-1)
    if log_scales.shape[1] != 1:
        q = F.normalize(quat_mult(d(cam_rot).reshape(1, 4), q), dim=-1)
    ls = d(log_scales)
    scales3 = torch.exp(ls.expand(-1, 3) if ls.shape[1] == 1 else ls)
    z = means_cam @ w0[2, :3] + w0[2, 3]
    dcols = torch.stack([z, torch.ones_like(z), z * z], 1)
    return means_cam, q, torch.sigmoid(d(logit_opacities)), scales3, dcols


def camera_pose(cam_unnorm_rot, cam_tran, dtype=torch.float64):
    """(rel_w2c [4,4], normalised camera quaternion [1,4]) of an unnormalised quaternion [1,4] and a translation [1,3]."""
    cam_rot = F.normalize(cam_unnorm_rot.to(dtype), dim=-1)
    top = torch.cat([rotation_matrix(cam_rot[0]), cam_tran.to(dtype).reshape(3, 1)], 1)
    bottom = torch.tensor([[0.0, 0.0, 0.0, 1.0]], dtype=dtype, device=top.device)
    return torch.cat([top, bottom], 0), cam_rot


def prepare_from_camera(means3D, unnorm_rotations, logit_opacities, log_scales, cam_unnorm_rot, cam_tran, w2c0,
                        dtype=torch.float64):
    """prepare() at the pose camera_pose(cam_unnorm_rot, cam_tran): gradients reach the camera's own parameters."""
    rel, cam_rot = camera_pose(cam_unnorm_rot, cam_tran, dtype)
    return prepare(means3D, unnorm_rotations, logit_opacities, log_scales, rel, cam_rot, w2c0, dtype)


def adam(init, grads, seg_sizes, seg_lrs, betas=(0.9, 0.999), eps=1e-15, skip=None, lr_changes=None,
         dtype=torch.float64, state=None):
    """torch.optim.Adam (one parameter group per segment) over a flat buffer `init`, driven by the flat gradients
    `grads` in order.  skip[i] true: gradient i is not applied (the step count does not advance).  lr_changes:
    {i: (segment, lr)} set before gradient i.  state: (step, exp_avg, exp_avg_sq) to resume from.
    Returns (params, exp_avg, exp_avg_sq, steps applied), flat, in `dtype`."""
    p = [t.clone().requires_grad_(True) for t in torch.split(init.detach().to(dtype), list(seg_sizes))]
    opt = torch.optim.Adam([{"params": [t], "lr": float(lr)} for t, lr in zip(p, seg_lrs)], lr=0.0,
                           betas=betas, eps=eps, foreach=False)
    if state is not None:
        step, m0, v0 = state
        for t, m, v in zip(p, torch.split(m0.to(dtype), list(seg_sizes)), torch.split(v0.to(dtype), list(seg_sizes))):
            opt.state[t] = dict(step=torch.tensor(float(step)), exp_avg=m.clone(), exp_avg_sq=v.clone())
    applied = 0 if state is None else int(state[0])
    for i, g in enumerate(grads):
        if lr_changes and i in lr_changes:
            k, lr = lr_changes[i]
            opt.param_groups[k]["lr"] = float(lr)
        if skip is not None and skip[i]:
            continue
        for t, gs in zip(p, torch.split(g.to(dtype), list(seg_sizes))):
            t.grad = gs.clone()
        opt.step()
        applied += 1
    st = lambda key: torch.cat([opt.state[t][key] if t in opt.state else torch.zeros_like(t) for t in p])
    return torch.cat([t.detach() for t in p]), st("exp_avg"), st("exp_avg_sq"), applied
