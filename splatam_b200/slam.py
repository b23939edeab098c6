"""Slim SplaTAM-style RGB-D SLAM loop over a synthetic sequence (BASELINE.json configs 4/5 stand-in: the
Replica / TUM datasets are not available offline).  It is a HARNESS around the operator, not a
re-implementation of R/scripts/splatam.py: per frame it runs SplaTAM's tracking inner loop (camera-only Adam,
silhouette-masked L1 sums; `mapping.track_frame`) from a constant-velocity initialisation
(R/scripts/splatam.py:423-444) and then `mapping_iters` keyframe-sharded mapping steps (`ShardedMapper`) over
a sliding window of keyframes, and reports ATE-RMSE of the estimated trajectory and the PSNR of re-rendered
keyframes -- the two end metrics the reference prints (R/utils/eval_helpers.py:23-77,569-592).
By default the map starts from a perturbed copy of the generating scene; with `initialize_map` +
`add_new_gaussians` + `prune_dict` + `select_keyframes` it is SplaTAM's full loop from RGB-D frames alone.
"""
import math

import torch
import torch.nn.functional as F

from . import mapping as M


def look_trajectory(num_frames, device, step=(0.012, -0.004, 0.008), rot_step=(0.003, -0.002, 0.0015)):
    """Smooth camera trajectory: per-frame relative w2c as (unnormalised quaternion [1,4,T], translation [1,3,T]);
    frame 0 is the identity (SplaTAM makes all poses relative to frame 0)."""
    rots = torch.zeros(1, 4, num_frames, device=device)
    trans = torch.zeros(1, 3, num_frames, device=device)
    rots[:, 0] = 1.0
    for t in range(num_frames):
        w = 1.0 + 0.15 * math.sin(0.7 * t)
        rots[0, 1:, t] = torch.tensor(rot_step, device=device) * t * w
        trans[0, :, t] = torch.tensor(step, device=device) * t * w
    return rots, trans


def render_frame(gauss, rots, trans, t, cam, render=None):
    """RGB-D observation of frame t from the generating scene (no gradient)."""
    with torch.no_grad():
        p = dict(gauss, cam_unnorm_rots=rots, cam_trans=trans)
        tg = M.transform_to_frame(p, t, gaussians_grad=False, camera_grad=False)
        w2c0 = torch.eye(4, device=rots.device)
        render = M.default_render if render is None else render
        im, _, _ = render(cam, **M.rgb_rendervar(p, tg))
        ds, _, _ = render(cam, **M.depth_sil_rendervar(p, w2c0, tg))
    return dict(id=t, cam=cam, w2c=w2c0, im=im.clone(), depth=ds[0:1].clone(), sil=ds[1:2].clone())


def psnr(a, b):
    mse = ((a - b) ** 2).mean()
    return float(20 * torch.log10(1.0 / torch.sqrt(mse)))


def initialize_map(frame, intrinsics, scale_dim=1):
    """Initial Gaussians = back-projection of every valid-depth pixel of the first frame
    (initialize_first_timestep, R/scripts/splatam.py:169-208).  Returns (parameter dict, scene_radius)."""
    from . import map_ops
    mask = (frame["depth"][0] > 0).reshape(-1)
    new, _ = map_ops.backproject(frame["im"], frame["depth"], intrinsics, torch.eye(4), mask=mask, scale_dim=scale_dim)
    return new, float(frame["depth"].max()) / 3.0            # scene_radius_depth_ratio = 3 in every shipped config


def _curr_w2c(rots, trans, t):
    return M.camera_w2c(rots[..., t], trans[..., t])[0]


def _without_densify(frame):
    """The frame dict without its densification-size copy: keyframes are kept for the whole run, and only the frame
    being mapped needs the second resolution."""
    return {k: v for k, v in frame.items() if k != "densify"}


def run_slam(gauss_init, frames, cam, render=None, tracking_iters=20, mapping_iters=8, keyframe_every=2,
             window=4, fused=None, seed=0, intrinsics=None, add_new_gaussians=False, sil_thres=0.5, prune_dict=None,
             scene_radius=None, select_keyframes=False, checkpoint_dir=None, first_frame_iters=0, map_every=None,
             graph=False, timing=None, densify_dict=None, tracking_lrs=(0.0004, 0.002), depth_loss_thres=None):
    """Tracks every frame and maps on keyframes.  gauss_init: dict of the five Gaussian tensors (the map's
    starting point); frames: list of dict(id, cam, w2c, im, depth).  Returns dict(rots, trans, psnr, gauss).

    The optional stages follow the reference's main loop (R/scripts/splatam.py:776-925): `add_new_gaussians` grows
    the map from each mapped frame's silhouette holes before mapping -- from the frame's ``densify`` entry, with that
    entry's camera and intrinsics, when it has one (SplaTAM-S's densification resolution, splatam.py:781-794; see
    datasets.RGBDSequence; keyframes are stored without it) --, `prune_dict` prunes inside the mapping
    iterations (prune_gaussians' schedule keys), `select_keyframes` picks the mapping window by re-projection
    overlap (window-2 selected + the last keyframe + the current frame) instead of the last `window` keyframes,
    `checkpoint_dir` writes params<t>.npz per mapped frame and params.npz at the end; `first_frame_iters` mapping
    iterations run on frame 0 before tracking starts (needed when the map is a raw back-projection).
    `map_every` (default: keyframe_every) maps every map_every-th frame while only every keyframe_every-th frame joins
    the keyframe list, as the reference's two config keys do (splatam.py:777,912).  `graph`: each mapping phase is
    captured into a CUDA graph over the sync-free rasterizer (fused path only).  `densify_dict`: gradient-based
    densification inside the mapping iterations (the reference's `use_gaussian_splatting_densification` branch,
    splatam.py:863-864; eager steps only -- the map size changes).  `tracking_lrs`: the tracking learning rates of
    (cam_unnorm_rots, cam_trans); the default is Replica's.  `depth_loss_thres`: track_frame's rule that doubles a
    frame's tracking iterations while the depth loss stays high (ScanNet++: 20000).  `timing`: dict that receives the
    accumulated wall seconds of tracking / mapping (synchronised) and the tracking and mapping iteration counts."""
    import time
    map_every = keyframe_every if map_every is None else map_every
    timing = {} if timing is None else timing
    timing.update(tracking_s=0.0, mapping_s=0.0, mapping_iters=0, tracking_iters=0)
    dev = gauss_init["means3D"].device
    T = len(frames)
    rots = torch.zeros(1, 4, T, device=dev); rots[:, 0] = 1.0
    trans = torch.zeros(1, 3, T, device=dev)
    kw = {} if render is None else {"render": render}
    mapper = M.ShardedMapper(gauss_init, rots, trans, seed=seed, fused=fused, track_means2D=densify_dict is not None, **kw)
    keyframes = [dict(_without_densify(frames[0]), est_w2c=torch.eye(4, device=dev))]
    counts = [mapper.g.shapes["means3D"][0]]
    for it in range(first_frame_iters):       # the reference maps frame 0 before it tracks frame 1 (splatam.py:777)
        mapper.step([keyframes[0]])
        if prune_dict is not None:
            mapper.prune_gaussians(it, prune_dict, scene_radius)
    for t in range(1, T):
        with torch.no_grad():           # constant-velocity initialisation (splatam.py:423-444)
            if t > 1:
                r1, r2 = F.normalize(rots[0, :, t - 1], dim=0), F.normalize(rots[0, :, t - 2], dim=0)
                rots[0, :, t] = F.normalize(r1 + (r1 - r2), dim=0)
                trans[0, :, t] = trans[0, :, t - 1] + (trans[0, :, t - 1] - trans[0, :, t - 2])
            else:
                rots[0, :, t] = rots[0, :, t - 1]
                trans[0, :, t] = trans[0, :, t - 1]
        params = dict({k: v.detach() for k, v in mapper.g.params.items()}, cam_unnorm_rots=rots, cam_trans=trans)
        torch.cuda.synchronize(dev) if dev.type == "cuda" else None
        t0 = time.perf_counter()
        losses = M.track_frame(params, frames[t], render=render, num_iters=tracking_iters, lr_rot=tracking_lrs[0],
                               lr_trans=tracking_lrs[1], fused=fused, depth_loss_thres=depth_loss_thres)
        torch.cuda.synchronize(dev) if dev.type == "cuda" else None
        timing["tracking_s"] += time.perf_counter() - t0
        timing["tracking_iters"] += len(losses)
        rots, trans = params["cam_unnorm_rots"].detach(), params["cam_trans"].detach()
        mapper.cam = dict(cam_unnorm_rots=rots, cam_trans=trans)
        cam_now = mapper.sync_camera()            # multi-rank runs: rank 0's tracking result is the pose of record
        rots, trans = cam_now["cam_unnorm_rots"], cam_now["cam_trans"]
        frame = frames[t]
        cur = dict(_without_densify(frame), est_w2c=_curr_w2c(rots, trans, t))
        if t % map_every == 0:
            if add_new_gaussians:
                if "densify" in frame:            # SplaTAM-S: grow the map from the densification-size frame
                    mapper.add_new_gaussians(frame["densify"], t, frame["densify"]["intrinsics"], sil_thres)
                else:
                    mapper.add_new_gaussians(frame, t, intrinsics, sil_thres)
            if select_keyframes:
                from .keyframes import keyframe_selection_overlap
                if mapper.world > 1:      # the selection draws from the global RNGs: every rank must draw the same
                    import numpy as _np
                    torch.manual_seed(1000 * seed + t); _np.random.seed(1000 * seed + t)
                sel = keyframe_selection_overlap(frames[t]["depth"], cur["est_w2c"], torch.as_tensor(intrinsics).to(dev),
                                                 keyframes[:-1], max(window - 2, 0))
                win = [keyframes[int(i)] for i in sel] + [keyframes[-1], cur]
            else:
                win = (keyframes + [cur])[-window:]
            mapper.reset_optimizer()                          # splatam.py:822
            if graph and densify_dict is None:
                mapper.enable_graph(win)
            torch.cuda.synchronize(dev) if dev.type == "cuda" else None
            t0 = time.perf_counter()
            for it in range(mapping_iters):
                mapper.step(win)
                if prune_dict is not None:
                    mapper.prune_gaussians(it, prune_dict, scene_radius)
                if densify_dict is not None:
                    mapper.densify(it, densify_dict, scene_radius)
            mapper.poll_overflow(win, block=True)
            torch.cuda.synchronize(dev) if dev.type == "cuda" else None
            timing["mapping_s"] += time.perf_counter() - t0
            timing["mapping_iters"] += mapping_iters
            counts.append(mapper.g.shapes["means3D"][0])
        if t % keyframe_every == 0:
            keyframes.append(cur)
            if checkpoint_dir is not None:
                from . import formats
                formats.save_params_ckpt(dict(mapper.g.params, cam_unnorm_rots=rots, cam_trans=trans), checkpoint_dir, t)
    # PSNR of the keyframes re-rendered from the final map at the estimated poses
    final = {k: v.detach() for k, v in mapper.g.params.items()}
    vals = []
    for fr in keyframes:
        est = render_frame(final, rots, trans, fr["id"], cam, render)
        vals.append(psnr(est["im"].clamp(0, 1), fr["im"].clamp(0, 1)))
    if checkpoint_dir is not None:
        from . import formats
        formats.save_params(dict(final, cam_unnorm_rots=rots, cam_trans=trans), checkpoint_dir)
    return dict(rots=rots, trans=trans, psnr=sum(vals) / len(vals), gauss=final, counts=counts)


def w2c_list(rots, trans):
    """Per-frame 4x4 w2c matrices from the packed pose tensors (R/utils/eval_helpers.py:555-563)."""
    return [_curr_w2c(rots, trans, t) for t in range(rots.shape[-1])]


def ate_horn(gt_w2c, est_w2c):
    """The reference's trajectory metric, restated: evaluate_ate + align (R/utils/eval_helpers.py:23-77): the
    translation columns of the w2c matrices are aligned rigidly with Horn's closed form (SVD of the 3x3
    cross-covariance, reflection fix on the last singular direction) and the MEAN residual norm is returned -- the
    number the reference prints as "Final Average ATE RMSE" (:569-570)."""
    import numpy as np
    model = np.stack([m[:3, 3].detach().cpu().double().numpy() for m in gt_w2c], 1)       # 3 x n (gt)
    data = np.stack([m[:3, 3].detach().cpu().double().numpy() for m in est_w2c], 1)       # 3 x n (estimate)
    mz, dz = model - model.mean(1, keepdims=True), data - data.mean(1, keepdims=True)
    W = mz @ dz.T                                   # sum of outer(model_i, data_i)
    U, _, Vh = np.linalg.svd(W.T)
    S = np.eye(3)
    if np.linalg.det(U) * np.linalg.det(Vh) < 0:
        S[2, 2] = -1.0
    rot = U @ S @ Vh
    t = data.mean(1, keepdims=True) - rot @ model.mean(1, keepdims=True)
    err = rot @ model + t - data
    return float(np.sqrt((err * err).sum(0)).mean())


def ate_rmse(rots_est, trans_est, rots_gt, trans_gt):
    """RMSE of camera-centre positions (all poses share frame 0, so no alignment is needed)."""
    def centres(rots, trans):
        out = []
        for t in range(rots.shape[-1]):
            R = M.build_rotation(F.normalize(rots[..., t]))[0]
            out.append(-(R.T @ trans[0, :, t]))
        return torch.stack(out)
    d = centres(rots_est, trans_est) - centres(rots_gt, trans_gt)
    return float(torch.sqrt((d ** 2).sum(-1).mean()))
