"""Offline map optimisation over all frames: the loop of the reference's two offline drivers,
R/scripts/post_splatam_opt.py (refine a finished SplaTAM map) and R/scripts/gaussian_splatting.py (3DGS from
ground-truth poses), from line 290 of each on.

Every iteration decays the means3D learning rate, picks one frame with Python's `random.randint`, renders it at its
own pose through the mapping front end (`mapping._render_pair` with the frame's "pose"), takes the 3DGS loss
`gs_loss`, runs the backward and `ShardedMapper.densify`, and then the Adam step -- except on an iteration where
densify edits the map: the reference's densify replaces every parameter tensor there, so its optimizer step finds no
gradient and nothing is updated (`mapping.densify_due`).  The two ways to start are `from_record` (a SplaTAM record,
formats.save_run_record or the reference's params.npz) and `from_gt_poses` (frame 0 back-projected, then every frame
grown at its ground-truth pose).  Evaluation is `evaluate.evaluate(..., at_gt_pose=True)`, see tools/run_offline_opt.py.
"""
import math
import random

import numpy as np
import torch

from . import formats
from . import mapping as M

# R/configs/{replica,scannetpp}/{post_splatam_opt,gaussian_splatting}.py: the same in all four
LOSS_WEIGHTS = (0.5, 1.0)          # im, depth
LRS = dict(means3D=0.00032, rgb_colors=0.0025, unnorm_rotations=0.001, logit_opacities=0.05, log_scales=0.005)
MEANS3D_LR_FINAL = 0.0000032
DENSIFY = dict(start_after=500, remove_big_after=3000, stop_after=15000, densify_every=100, grad_thresh=0.0002,
               num_to_split_into=2, removal_opacity_threshold=0.005, final_removal_opacity_threshold=0.005,
               reset_opacities=True, reset_opacities_every=3000)


def expon_lr(step, lr_init, lr_final, max_steps):
    """get_expon_lr_func(lr_init, lr_final, lr_delay_steps=0, max_steps)(step) (R/utils/gs_external.py:269-302): the
    log-linear interpolation from lr_init at step 0 to lr_final at max_steps.  Every shipped config has
    lr_delay_steps = 0, so lr_delay_mult has no effect and is not a parameter here."""
    if step < 0 or (lr_init == 0.0 and lr_final == 0.0):
        return 0.0
    t = np.clip(step / max_steps, 0, 1)
    return float(np.exp(np.log(lr_init) * (1 - t) + np.log(lr_final) * t))


def gs_loss(params, frame, render, fused, loss_weights=LOSS_WEIGHTS):
    """get_loss_gs (R/scripts/gaussian_splatting.py:200-236, post_splatam_opt.py:127-160) of one frame -> (loss,
    radii, means2D of the RGB render with its gradient retained).

    This is not SplaTAM's mapping loss: the depth term is the mean over all H*W pixels of |depth * (gt != 0) - gt|, that
    is the sum over valid pixels divided by H*W, with no NaN or uncertainty mask; the RGB term is 0.8 L1 + 0.2 (1 -
    SSIM).  fused: the sums come from `train_ops.masked_l1` (depth_mean=False, scaled by 1 / (H*W)) and
    `train_ops.image_loss`.  masked_l1's validity mask is gt > 0 & !isnan(depth) & !isnan(depth^2 channel - depth^2):
    for depth maps (gt >= 0) and a render without NaN it selects the pixels that contribute here, and a NaN render
    would make the reference's loss NaN anyway."""
    im, depth_sil, radius, means2D = M._render_pair(params, frame, render, fused, camera_grad=False)
    means2D.retain_grad()
    gt_im, gt_depth = frame["im"], frame["depth"]
    if fused:
        from .train_ops import image_loss, masked_l1
        H, W = gt_depth.shape[-2:]
        l_depth, _ = masked_l1(depth_sil, gt_depth, depth_mean=False)
        l_depth = l_depth / float(H * W)
        l_im = image_loss(im, gt_im, 0.8, 0.2)
    else:
        depth = depth_sil[0:1] * (gt_depth != 0.0)
        l_depth = torch.abs(depth - gt_depth).mean()
        l_im = 0.8 * torch.abs(im - gt_im).mean() + 0.2 * (1.0 - M.calc_ssim(im, gt_im))
    return loss_weights[0] * l_im + loss_weights[1] * l_depth, radius, means2D


def optimize_map(mapper, frames, iters, means3D_lr_final, densify_dict, scene_radius, seed=0, eval_at=(),
                 on_eval=None, loss_weights=LOSS_WEIGHTS, trace=None):
    """`iters` iterations of the offline loop over `frames` (frame dicts with id, cam, w2c = the first frame's w2c, im,
    depth and "pose" = (w2c [4,4], normalised quaternion [1,4]) of the frame's training pose) on `mapper`, whose
    means3D learning rate at construction is the schedule's lr_init.  The frame of each iteration is
    random.Random(seed).randint(0, len(frames) - 1), the sequence of the reference's seed_everything(seed) +
    random.randint; split samples of densify come from torch's global RNG, as in the reference.
    on_eval(iteration, mapper) runs after iteration `it` when it + 1 is in `eval_at` (the reference evaluates after
    iteration 7000).  trace: a list that receives dict(frame, lr, loss (0-d device tensor), stepped) per iteration.
    Returns the Gaussian count after each iteration."""
    rng = random.Random(seed)
    lr_init = mapper.lrs["means3D"]
    counts = []
    for it in range(iters):
        lr = expon_lr(it + 1, lr_init, means3D_lr_final, iters)
        mapper.set_lr("means3D", lr)
        k = rng.randint(0, len(frames) - 1)
        mapper.g.zero_grad()
        loss, radius, means2D = gs_loss(mapper.params(), frames[k], mapper.render, mapper.fused, loss_weights)
        loss.backward()
        with torch.no_grad():
            stepped = not M.densify_due(it, densify_dict)
            counts.append(mapper.densify(it, densify_dict, scene_radius, means2D_grad=means2D.grad, seen=radius > 0))
            if stepped:
                mapper.opt.step()
        if trace is not None:
            trace.append(dict(frame=k, lr=lr, loss=loss.detach(), stepped=stepped))
        if on_eval is not None and it + 1 in eval_at:
            on_eval(it + 1, mapper)
    return counts


def _map_lrs(lrs):
    """`lrs` without camera keys: the offline loops render with camera_grad=False whatever their camera rates
    (R/scripts/post_splatam_opt.py), so a non-zero camera rate is an error rather than a request for pose refinement."""
    bad = {k: v for k, v in lrs.items() if k in M.CAM_KEYS and float(v) != 0.0}
    if bad:
        raise ValueError("offline map optimisation keeps the poses fixed; got camera rates %s" % bad)
    return {k: v for k, v in lrs.items() if k not in M.CAM_KEYS}


def from_record(path, frames, frame_indices, device, lrs=LRS, render=M.default_render, fused=None):
    """post_splatam_opt.py's start (initialize_first_timestep_from_ckpt, :68-124, and the frame loading, :243-262):
    the map of a SplaTAM record -- formats.save_run_record's or the reference's params.npz -- with its five Gaussian
    tensors and `timestep`, and each of `frames` trained at the record's camera column for that frame.

    frame_indices[t]: the original index of frames[t] in the SLAM run's sequence (start + stride * t for a reader with
    that start and stride, when the SLAM run read every frame from 0).  The reference indexes the camera tensor by loop
    position t instead, which is the same thing only at stride 1 (DESIGN.md, "Offline map optimisation").  A record
    that formats.read_record rejects, or whose camera tensor has no column for some frame, raises ValueError.
    Returns (mapper, training frames = the frame dicts with "pose", scene_radius = max depth of frames[0] / 2, the
    record as formats.read_record returns it)."""
    rec = formats.read_record(path, formats.CHECKPOINT_KEYS + ("timestep",))
    idx = [int(i) for i in frame_indices]
    if len(idx) != len(frames):
        raise ValueError("%d frame indices for %d frames" % (len(idx), len(frames)))
    formats.check_camera_columns(path, rec, idx)
    t = formats.record_tensors(rec, formats.CHECKPOINT_KEYS, device)
    rots, trans = t["cam_unnorm_rots"], t["cam_trans"]
    train = [dict(frames[i], pose=M.camera_w2c(rots[..., k], trans[..., k])) for i, k in enumerate(idx)]
    mapper = M.ShardedMapper({k: t[k] for k in formats.GAUSSIAN_KEYS}, rots, trans, lrs=_map_lrs(lrs), render=render,
                             fused=fused, timestep=rec["timestep"])
    return mapper, train, float(frames[0]["depth"].max()) / 2.0, rec


def from_gt_poses(init_frames, frames, lrs=LRS, sil_thres=0.5, render=M.default_render, fused=None):
    """gaussian_splatting.py's start (initialize_first_timestep and the growth pass, :404-495): the back-projection of
    init_frames[0] (`slam.initialize_map`, isotropic), then for t = 1 .. T-1 the ground-truth w2c of init_frames[t]
    written into camera column t and `ShardedMapper.add_new_gaussians` on that frame at `sil_thres`.  No optimisation
    runs during the growth: the reference optimises only after the last frame.  init_frames are read at the
    desired_image_*_init size, `frames` (the training frames, trained at their gt_w2c) at desired_image_*.  CUDA only,
    as add_new_gaussians.  Returns (mapper, training frames, scene_radius = max depth of init_frames[0] / 2)."""
    from . import slam
    f0 = init_frames[0]
    dev = f0["depth"].device
    T = len(init_frames)
    init, _ = slam.initialize_map(f0, f0["intrinsics"].cpu())
    rots = torch.zeros(1, 4, T, device=dev)
    rots[:, 0] = 1.0
    mapper = M.ShardedMapper(init, rots, torch.zeros(1, 3, T, device=dev), lrs=_map_lrs(lrs), render=render,
                             fused=fused)
    K = f0["intrinsics"].cpu()
    for t in range(T):
        fr = init_frames[t]
        w2c = fr["gt_w2c"].to(dev).float()
        with torch.no_grad():
            mapper.cam["cam_unnorm_rots"][..., t] = M.matrix_to_quaternion(w2c[:3, :3]).reshape(1, 4)
            mapper.cam["cam_trans"][..., t] = w2c[:3, 3].reshape(1, 3)
        if t > 0:
            mapper.add_new_gaussians(fr, t, K, sil_thres)
    train = [dict(fr, pose=M.gt_pose(fr["gt_w2c"].to(dev).float())) for fr in frames]
    return mapper, train, float(f0["depth"].max()) / 2.0


def record_poses(frames):
    """The w2c matrices of the training poses: the record's `gt_w2c_all_frames` (post_splatam_opt.py:376-379)."""
    return [fr["pose"][0] for fr in frames]


def train_psnr(mapper, frames):
    """Mean PSNR of the training frames rendered at their training poses (no gradient; one read per frame)."""
    vals = []
    with torch.no_grad():
        for fr in frames:
            im, _, _, _ = M._render_pair(mapper.params(), fr, mapper.render, mapper.fused, camera_grad=False)
            mse = float(((im - fr["im"]) ** 2).mean())
            vals.append(20 * math.log10(1.0 / math.sqrt(mse)) if mse > 0 else float("inf"))
    return float(np.mean(vals))
