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

import numpy as np
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


def keyframes_from_checkpoint(frames, ckpt):
    """The keyframe list of a checkpoint (formats.load_checkpoint): frames[k] for every stored id k, with est_w2c
    rebuilt from the stored camera column k (F.normalize + build_rotation, as R/scripts/splatam.py:619-638 does) -- or,
    when the checkpoint's sidecar holds `keyframe_est_w2c` (a run with keyframe-pose refinement, whose later mapping
    phases move a column after its keyframe stored its pose), the stored matrices themselves."""
    rots, trans = ckpt["cam_unnorm_rots"], ckpt["cam_trans"]
    ids = ckpt["keyframe_time_indices"]
    state = ckpt.get("state")
    if state is not None and "keyframe_est_w2c" in state:
        est = torch.from_numpy(np.array(state["keyframe_est_w2c"], dtype=np.float32)).to(rots.device)
        if est.shape != (len(ids), 4, 4):
            raise ValueError("the checkpoint's run state holds %s keyframe poses for %d keyframes"
                             % (tuple(est.shape), len(ids)))
        return [dict(_without_densify(frames[k]), est_w2c=est[i]) for i, k in enumerate(ids)]
    return [dict(_without_densify(frames[k]), est_w2c=_curr_w2c(rots, trans, k)) for k in ids]


EXPOSURE_DEFAULTS = dict(lr_log_gain=0.01, lr_bias=0.002)


def exposure_config(exposure):
    """run_slam's `exposure` dict with EXPOSURE_DEFAULTS filled in; ValueError for unknown keys or bad rates."""
    if not isinstance(exposure, dict):
        raise ValueError("exposure must be None or a dict of %s, got %r" % (sorted(EXPOSURE_DEFAULTS), exposure))
    unknown = sorted(set(exposure) - set(EXPOSURE_DEFAULTS))
    if unknown:
        raise ValueError("unknown exposure keys %s (known: %s)" % (unknown, sorted(EXPOSURE_DEFAULTS)))
    cfg = dict(EXPOSURE_DEFAULTS, **exposure)
    for k, v in cfg.items():
        if isinstance(v, bool) or not isinstance(v, (int, float)) or not math.isfinite(v) or v < 0:
            raise ValueError("exposure %s must be a finite rate >= 0, got %r" % (k, v))
    return {k: float(v) for k, v in cfg.items()}


def _run_state(mapper, counts, keyframes=None, pose_graph=None, reloc_frames=None, masks=None):
    """The sidecar of a checkpoint (formats.save_checkpoint's `run_state`): what continues a run exactly and the
    reference's params{t}.npz cannot carry -- the mapper's own state (ShardedMapper.run_state: the Gaussians'
    `timestep`, its schedule and device generators, the densification statistic), torch's CPU RNG and the CUDA RNG of
    the map's device (keyframe selection and densification draw from the global generators), NumPy's global RNG
    (keyframe_selection_overlap's permutation) and the Gaussian counts so far; with `keyframes` (runs with keyframe-pose
    refinement) also their stored est_w2c, which the refined camera columns no longer give; with `pose_graph` (runs
    with loop closure) also its edges and their measurements (loop.PoseGraph.state); with `reloc_frames` (runs with
    relocalisation: (lost ids, relocalised ids)) `reloc_lost` and `reloc_relocalised`; with a `cam_exposure` in the
    mapper's cameras (runs with exposure) also that table [1,6,T]; with `masks` (runs with motion masks: the
    keyframes' bool [H,W] masks) `keyframe_dynamic`, np.packbits of their [K,H,W] stack, and `keyframe_dynamic_shape`.
    Numeric arrays only."""
    dev = mapper.g.flat.device
    _, keys, pos, has_gauss, cached = np.random.get_state()
    st = dict(mapper.run_state(), torch_rng=torch.get_rng_state().numpy(),
              numpy_rng_keys=np.asarray(keys, dtype=np.uint32), numpy_rng_pos=np.array(pos, dtype=np.int64),
              numpy_rng_has_gauss=np.array(has_gauss, dtype=np.int64),
              numpy_rng_cached_gaussian=np.array(cached, dtype=np.float64), counts=np.array(counts, dtype=np.int64))
    if dev.type == "cuda":
        st["cuda_rng"] = torch.cuda.get_rng_state(dev).numpy()
    if keyframes is not None:
        st["keyframe_est_w2c"] = torch.stack([kf["est_w2c"].detach().float() for kf in keyframes]).cpu().numpy()
    if pose_graph is not None:
        st.update(pose_graph.state())
    if reloc_frames is not None:
        st["reloc_lost"] = np.array(sorted(reloc_frames[0]), dtype=np.int64)
        st["reloc_relocalised"] = np.array(sorted(reloc_frames[1]), dtype=np.int64)
    if "cam_exposure" in mapper.cam:
        st["cam_exposure"] = mapper.cam["cam_exposure"].detach().float().cpu().numpy()
    if masks is not None:
        m = torch.stack(masks).cpu().numpy()
        st["keyframe_dynamic"] = np.packbits(m.reshape(-1))
        st["keyframe_dynamic_shape"] = np.array(m.shape, dtype=np.int64)
    return st


def _keyframe_masks(state, n):
    """The keyframes' motion masks of a checkpoint's sidecar (_run_state's `masks`): a list of n bool [H,W] arrays."""
    if state is None or "keyframe_dynamic" not in state:
        raise ValueError("dynamic: the checkpoint holds no keyframe motion masks (it was written by a run without them)")
    shape = tuple(int(x) for x in np.asarray(state["keyframe_dynamic_shape"]).reshape(-1))
    if len(shape) != 3 or shape[0] != n:
        raise ValueError("the checkpoint's motion masks have shape %s for %d keyframes" % (shape, n))
    bits = np.unpackbits(np.asarray(state["keyframe_dynamic"], dtype=np.uint8))[:int(np.prod(shape))]
    return list(bits.reshape(shape).astype(bool))


def _restore_run_state(mapper, st):
    """Inverse of _run_state on a mapper built from the checkpoint's map; returns the Gaussian counts so far."""
    mapper.load_run_state(st)
    dev = mapper.g.flat.device
    torch.set_rng_state(torch.from_numpy(np.array(st["torch_rng"], dtype=np.uint8)))
    np.random.set_state(("MT19937", np.array(st["numpy_rng_keys"], dtype=np.uint32), int(st["numpy_rng_pos"]),
                         int(st["numpy_rng_has_gauss"]), float(st["numpy_rng_cached_gaussian"])))
    if dev.type == "cuda" and "cuda_rng" in st:
        torch.cuda.set_rng_state(torch.from_numpy(np.array(st["cuda_rng"], dtype=np.uint8)), dev)
    return [int(c) for c in st["counts"]]


def _check_resume(gauss_init, resume, T, checkpoint_every, checkpoint_dir):
    import numbers
    if checkpoint_every is not None:
        if (isinstance(checkpoint_every, bool) or not isinstance(checkpoint_every, numbers.Integral)
                or checkpoint_every <= 0):
            raise ValueError("checkpoint_every must be a positive integer, got %r" % (checkpoint_every,))
        if checkpoint_dir is None:
            raise ValueError("checkpoint_every needs a checkpoint_dir")
    if resume is None:
        if gauss_init is None:
            raise ValueError("run_slam needs gauss_init or resume")
        return
    if gauss_init is not None:
        raise ValueError("give gauss_init or resume, not both")
    n = resume["cam_unnorm_rots"].shape[-1]
    if n != T or resume["cam_trans"].shape[-1] != T:
        raise ValueError("the checkpoint's cameras cover %d frames, the sequence has %d" % (n, T))
    if not 0 <= int(resume["time_idx"]) <= T - 1:
        raise ValueError("checkpoint frame %d is outside [0, %d]" % (int(resume["time_idx"]), T - 1))


def run_slam(gauss_init, frames, cam, render=None, tracking_iters=20, mapping_iters=8, keyframe_every=2,
             window=4, fused=None, seed=0, intrinsics=None, add_new_gaussians=False, sil_thres=0.5, prune_dict=None,
             scene_radius=None, select_keyframes=False, checkpoint_dir=None, first_frame_iters=0, map_every=None,
             graph=False, timing=None, densify_dict=None, tracking_lrs=(0.0004, 0.002), depth_loss_thres=None,
             checkpoint_every=None, resume=None, mapping_cam_lrs=(0.0, 0.0), pose_init="constant_velocity",
             loop_closure=None, relocalise=None, exposure=None, dynamic=None):
    """Tracks every frame and maps on keyframes.  gauss_init: dict of the five Gaussian tensors (the map's
    starting point); frames: list of dict(id, cam, w2c, im, depth).  Returns dict(rots, trans, psnr, gauss, counts,
    timestep, keyframe_time_indices, keyframe_est_w2c): `timestep` is the frame that created each Gaussian of the final
    map, `keyframe_est_w2c` the pose each keyframe stored when it joined the list.

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
    frame's tracking iterations while the depth loss stays high (ScanNet++: 20000).  `mapping_cam_lrs`: the mapping
    learning rates of (cam_unnorm_rots, cam_trans); non-zero turns on keyframe-pose refinement (the reference's
    do_ba=True, `ShardedMapper`): each mapping iteration also steps its keyframe's pose, and a keyframe joins the
    keyframe list with its pose after its own mapping phase, as the reference stores it.  `timing`: dict that receives
    the accumulated wall seconds of tracking / mapping (synchronised), the tracking and mapping iteration counts, and
    `setup_s`, the wall seconds from the call to the start of the frame loop.
    `pose_init`: how each frame's tracking starts.  "constant_velocity" (the default) is the reference's guess
    (splatam.py:423-444).  "icp" follows that guess with icp.init_pose: the map's depth rendered at frame t-1's pose is
    aligned with frame t's depth by point-to-plane ICP on the GPU (needs CUDA tensors and `intrinsics`), and the ICP
    pose replaces the guess when it passes its acceptance test.  "rgbd_icp" aligns with icp.align_rgbd instead: the
    map's RGB render and frame t's colour add a photometric term at icp.DEFAULT_WEIGHT, and the records also hold
    `photo_rms`.  Every rank computes the same pose.  With "icp",
    `timing` also receives `pose_init_s` (synchronised wall seconds) and the result holds `icp`: per tracked frame
    dict(frame, accepted, inlier_frac, rms), read from the device once at the end.  `pose_init` is not stored in
    checkpoints: a resumed run passes it again.
    `loop_closure`: None (the default: off, and nothing of it runs) or a dict of loop.DEFAULTS keys (needs CUDA tensors
    and `intrinsics`).  Every keyframe frame t > 0 becomes a node of a keyframe pose graph, with an odometry edge from
    the previous node measured from the camera columns after tracking; then, before new Gaussians are added,
    loop.close_loop looks for an old keyframe frame t sees again, measures the loop by ICP against that keyframe's
    depth, solves the graph and, if every edge fits, moves every camera column, every keyframe's est_w2c and every
    Gaussian (by its `timestep`) with the correction of its node; frame t's mapping window then holds the loop keyframe
    in place of its first entry.  `timing` also receives `loop_closure_s` and the result holds `loops`: one dict(frame,
    keyframe, accepted, inlier_frac, rms, correction_m, correction_deg) per measured candidate.  Checkpoints then also
    hold the graph and every keyframe's est_w2c; `loop_closure` itself is not stored: a resumed run passes it again.
    `relocalise`: None (the default: off, and nothing of it runs) or a dict of reloc.DEFAULTS keys (`photometric`: the
    health check also compares the map's RGB render with the frame's by colour NCC, and candidates are verified with
    icp.align_rgbd; needs CUDA tensors
    and `intrinsics`; one rank only -- with several ranks it raises ValueError).  Each keyframe's frame adds its
    descriptor to a reloc.Database when it joins the keyframe list.  After tracking, reloc.health checks every frame
    against the map's depth/silhouette render at its pose (one render and one small host read per frame); a lost frame
    calls reloc.relocalise against the keyframe database.  A relocalised frame continues as a normal frame, and the
    next frame starts with zero velocity.  A frame that stays lost takes column t - 1 (so the next guess has zero
    velocity) and is not mapped, adds no Gaussians, joins no keyframe list and adds no pose-graph node.  `timing` also
    receives `health_s` and `reloc_s`, and the result holds `reloc`: per lost frame dict(frame, relocalised, candidate
    (camera column or None), score, coverage, inlier_frac, rms (the final health), candidates, scores, icp),
    `reloc_lost` (the ids of frames that stayed lost) and `reloc_database`.  Checkpoints also hold the lost and
    relocalised ids; on resume the database is rebuilt from the restored keyframes.  `relocalise` itself is not
    stored: a resumed run passes it again.
    `exposure`: None (the default: off, and nothing of it runs) or a dict of EXPOSURE_DEFAULTS keys (the tracking rates
    lr_log_gain, lr_bias).  Each frame t gets a colour correction, column t of a [1,6,T] table (log-gains a_r, a_g,
    a_b, biases b_r, b_g, b_b): its renders are compared with it through exp(a) * render + b (train_ops.exposure).
    Frame 0 keeps the identity, so the map holds frame 0's appearance; frame t starts from column t - 1 and tracking
    optimises it with the pose (track_frame's lr_exposure); mapping applies each keyframe's column without stepping
    it; new Gaussians take the frame's colour mapped back, (c - b) exp(-a); `pose_init="rgbd_icp"` corrects the map's
    RGB render by column t - 1; the final PSNR is of the corrected renders.  The result holds `exposure` [1,6,T] and
    checkpoints hold the table in their sidecar (not in params{t}.npz); resuming with `exposure` from a checkpoint
    without it raises ValueError, and so does `exposure` together with `relocalise`.
    `dynamic`: None (the default: off, and nothing of it runs) or a dict of dynamic.DEFAULTS keys.  Each tracked frame
    gets a motion mask from the residual between its depth and the map's depth render (dynamic.py states the rule):
    tracking leaves out the `dynamic | inconsistent` pixels, recomputing them every `refresh_every` iterations from that
    iteration's render (track_frame's `dynamic`); after tracking, one render at the pose of record gives the frame's
    masks; its keyframe stores `dynamic`, which mapping leaves out of its loss and `add_new_gaussians` out of map
    growth (max-pooled to the densification frame's size for SplaTAM-S).  Frame 0 has an empty mask.  The result holds
    `dynamic`: per tracked frame dict(frame, scale, dynamic_frac, inconsistent_frac), read from the device once at the
    end; checkpoints hold the keyframes' masks in their sidecar, and `dynamic` together with `relocalise` raises
    ValueError.

    Checkpoints and resume (R/scripts/splatam.py:604-643,927-931).  With `checkpoint_dir` and `checkpoint_every` = N,
    after frame t's mapping and keyframe step, for every t % N == 0 (frame 0 included, after `first_frame_iters`),
    rank 0 writes formats.save_checkpoint's three files: the reference's params{t}.npz and keyframe_time_indices{t}.npy,
    and the run_state{t}.npz sidecar (`_run_state`); the per-keyframe params<t>.npz are then not written, and the final
    params.npz is written by rank 0 only.  Without `checkpoint_every`, `checkpoint_dir` writes params<t>.npz per
    keyframe and params.npz at the end.
    `resume` = formats.load_checkpoint(dir, t, device), with gauss_init None: the map, the cameras and the keyframe list
    come from the checkpoint (keyframe k is frames[k] with est_w2c rebuilt from the stored camera column, as
    splatam.py:619-638 does); with a sidecar every RNG, the schedule generator, the densification statistic, `timestep`
    and `counts` are restored -- with refinement also the keyframes' stored est_w2c, since later mapping phases move
    a keyframe's column after it stored its pose --, without one (a checkpoint the reference wrote) `timestep` is
    zeros, `counts` starts at the loaded map and the RNGs are left as they are.  `first_frame_iters` does not run.
    The loop continues at frame t + 1, unlike the reference, which restarts at t: it tracks and maps frame t a second
    time and appends it to its keyframe list twice.  Continuing at t + 1 is what makes a resumed run equal the
    uninterrupted one."""
    import time
    t_setup = time.perf_counter()
    map_every = keyframe_every if map_every is None else map_every
    timing = {} if timing is None else timing
    timing.update(tracking_s=0.0, mapping_s=0.0, mapping_iters=0, tracking_iters=0, setup_s=0.0)
    T = len(frames)
    _check_resume(gauss_init, resume, T, checkpoint_every, checkpoint_dir)
    if pose_init not in ("constant_velocity", "icp", "rgbd_icp"):
        raise ValueError("pose_init must be 'constant_velocity', 'icp' or 'rgbd_icp', got %r" % (pose_init,))
    use_expo = exposure is not None
    if use_expo:
        expo_cfg = exposure_config(exposure)
        if relocalise is not None:
            raise ValueError("exposure and relocalise cannot be combined: relocalisation's candidate tracking does not "
                             "estimate exposure")
        if resume is not None and (resume["state"] is None or "cam_exposure" not in resume["state"]):
            raise ValueError("exposure: the checkpoint holds no exposure table (it was written by a run without it)")
        lr_expo = (expo_cfg["lr_log_gain"], expo_cfg["lr_bias"])
    use_dyn = dynamic is not None
    if use_dyn:
        from . import dynamic as _dynamic
        dyn_cfg = _dynamic.config(dynamic)
        if relocalise is not None:
            raise ValueError("dynamic and relocalise cannot be combined: relocalisation's health check does not use the "
                             "motion mask")
        dyn_stats = []
    use_icp = pose_init != "constant_velocity"
    if use_icp:
        if intrinsics is None:
            raise ValueError("pose_init=%r needs the intrinsics" % (pose_init,))
        from . import _lib, icp
        _lib.need_cuda("run_slam(pose_init=%r)" % (pose_init,), (gauss_init or resume["gauss"])["means3D"])
        K_icp = np.asarray(torch.as_tensor(intrinsics).detach().cpu(), dtype=np.float64)
        timing["pose_init_s"] = 0.0
        icp_stats = []
    use_loop = loop_closure is not None
    if use_loop:
        from . import _lib, loop
        loop_cfg = loop.config(loop_closure)
        if intrinsics is None:
            raise ValueError("loop_closure needs the intrinsics")
        _lib.need_cuda("run_slam(loop_closure=...)", (gauss_init or resume["gauss"])["means3D"])
        timing["loop_closure_s"] = 0.0
        loops = []
    use_reloc = relocalise is not None
    if use_reloc:
        from . import _lib, reloc
        reloc_cfg = reloc.config(relocalise)
        if intrinsics is None:
            raise ValueError("relocalise needs the intrinsics")
        import torch.distributed as dist
        if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
            raise ValueError("relocalise runs on one rank only, got a world of %d" % dist.get_world_size())
        _lib.need_cuda("run_slam(relocalise=...)", (gauss_init or resume["gauss"])["means3D"])
        timing.update(health_s=0.0, reloc_s=0.0)
        reloc_recs, reloc_lost, reloc_done = [], set(), set()
    kw = {} if render is None else {"render": render}
    track_m2d = densify_dict is not None
    kw["lrs"] = dict(cam_unnorm_rots=float(mapping_cam_lrs[0]), cam_trans=float(mapping_cam_lrs[1]))
    refine = any(v != 0.0 for v in kw["lrs"].values())
    if resume is None:
        dev = gauss_init["means3D"].device
        rots = torch.zeros(1, 4, T, device=dev); rots[:, 0] = 1.0
        trans = torch.zeros(1, 3, T, device=dev)
        if use_expo:
            kw["cam_exposure"] = torch.zeros(1, 6, T, device=dev)
        mapper = M.ShardedMapper(gauss_init, rots, trans, seed=seed, fused=fused, track_means2D=track_m2d, **kw)
        keyframes = [dict(_without_densify(frames[0]), est_w2c=torch.eye(4, device=dev))]
        counts = [mapper.g.shapes["means3D"][0]]
        start = 1
        if use_dyn:
            keyframes[0]["dynamic"] = torch.zeros(frames[0]["depth"].shape[-2:], dtype=torch.bool, device=dev)
    else:
        dev = resume["gauss"]["means3D"].device
        rots = resume["cam_unnorm_rots"].detach().clone().to(dev)
        trans = resume["cam_trans"].detach().clone().to(dev)
        if use_expo:
            kw["cam_exposure"] = torch.from_numpy(np.array(resume["state"]["cam_exposure"], dtype=np.float32)).to(dev)
            if tuple(kw["cam_exposure"].shape) != (1, 6, T):
                raise ValueError("the checkpoint's exposure table has shape %s, expected (1, 6, %d)"
                                 % (tuple(kw["cam_exposure"].shape), T))
        mapper = M.ShardedMapper(resume["gauss"], rots, trans, seed=seed, fused=fused, track_means2D=track_m2d, **kw)
        keyframes = keyframes_from_checkpoint(frames, dict(resume, cam_unnorm_rots=rots, cam_trans=trans))
        if resume["state"] is not None:
            counts = _restore_run_state(mapper, resume["state"])
        else:
            counts = [mapper.g.shapes["means3D"][0]]
        start = int(resume["time_idx"]) + 1
        first_frame_iters = 0
        if use_dyn:
            for kf, m in zip(keyframes, _keyframe_masks(resume["state"], len(keyframes))):
                kf["dynamic"] = torch.from_numpy(m).to(dev)
    if use_loop:
        st = resume["state"] if resume is not None else None
        if st is not None and "loop_graph_edges" in st:
            pose_graph = loop.PoseGraph.from_state(st, dev)
        else:
            pose_graph = loop.PoseGraph.chain([int(kf["id"]) for kf in keyframes], rots, trans)
    if use_reloc:
        st = resume["state"] if resume is not None else None
        if st is not None and "reloc_lost" in st:
            reloc_lost = {int(i) for i in np.asarray(st["reloc_lost"]).reshape(-1)}
            reloc_done = {int(i) for i in np.asarray(st["reloc_relocalised"]).reshape(-1)}
        reloc_db = reloc.Database()
        for kf in keyframes:
            reloc_db.add(kf, int(kf["id"]))

    def checkpoint(t):
        if checkpoint_every is None or t % checkpoint_every != 0 or mapper.rank != 0:
            return
        from . import formats
        formats.save_checkpoint(checkpoint_dir, t, dict(mapper.g.params, cam_unnorm_rots=rots, cam_trans=trans),
                                [kf["id"] for kf in keyframes],
                                _run_state(mapper, counts, keyframes if (refine or use_loop) else None,
                                           pose_graph if use_loop else None,
                                           (reloc_lost, reloc_done) if use_reloc else None,
                                           [kf["dynamic"] for kf in keyframes] if use_dyn else None))

    def refined_cameras():
        """Refinement: copies of the mapper's cameras after a mapping phase (tracking then works on its own tensors)."""
        return tuple(mapper.cam[k].detach().clone() for k in M.CAM_KEYS)

    for it in range(first_frame_iters):       # the reference maps frame 0 before it tracks frame 1 (splatam.py:777)
        mapper.step([keyframes[0]])
        if prune_dict is not None:
            mapper.prune_gaussians(it, prune_dict, scene_radius)
    if refine and first_frame_iters > 0:
        rots, trans = refined_cameras()
        keyframes[0]["est_w2c"] = _curr_w2c(rots, trans, 0)
    if resume is None:
        checkpoint(0)
    torch.cuda.synchronize(dev) if dev.type == "cuda" else None
    timing["setup_s"] = time.perf_counter() - t_setup
    for t in range(start, T):
        with torch.no_grad():           # constant-velocity initialisation (splatam.py:423-444)
            if t > 1 and not (use_reloc and (t - 1) in reloc_done):
                r1, r2 = F.normalize(rots[0, :, t - 1], dim=0), F.normalize(rots[0, :, t - 2], dim=0)
                rots[0, :, t] = F.normalize(r1 + (r1 - r2), dim=0)
                trans[0, :, t] = trans[0, :, t - 1] + (trans[0, :, t - 1] - trans[0, :, t - 2])
            else:
                rots[0, :, t] = rots[0, :, t - 1]
                trans[0, :, t] = trans[0, :, t - 1]
        params = dict({k: v.detach() for k, v in mapper.g.params.items()}, cam_unnorm_rots=rots, cam_trans=trans)
        if use_expo:
            expo = mapper.cam["cam_exposure"]
            with torch.no_grad():
                expo[..., t] = expo[..., t - 1]               # zero velocity
            params["cam_exposure"] = expo
        torch.cuda.synchronize(dev) if dev.type == "cuda" else None
        if use_icp:
            t0 = time.perf_counter()
            icp_stats.append(icp.init_pose(params, frames[t], t, K_icp, render=render, fused=fused,
                                           photometric=pose_init == "rgbd_icp"))
            torch.cuda.synchronize(dev)
            timing["pose_init_s"] += time.perf_counter() - t0
        t0 = time.perf_counter()
        losses = M.track_frame(params, frames[t], render=render, num_iters=tracking_iters, lr_rot=tracking_lrs[0],
                               lr_trans=tracking_lrs[1], fused=fused, depth_loss_thres=depth_loss_thres,
                               lr_exposure=lr_expo if use_expo else None, dynamic=dyn_cfg if use_dyn else None)
        torch.cuda.synchronize(dev) if dev.type == "cuda" else None
        timing["tracking_s"] += time.perf_counter() - t0
        timing["tracking_iters"] += len(losses)
        rots, trans = params["cam_unnorm_rots"].detach(), params["cam_trans"].detach()
        mapper.cam = dict(mapper.cam, cam_unnorm_rots=rots, cam_trans=trans)
        cam_now = mapper.sync_camera()            # multi-rank runs: rank 0's tracking result is the pose of record
        rots, trans = cam_now["cam_unnorm_rots"], cam_now["cam_trans"]
        frame = frames[t]
        if use_reloc:
            t0 = time.perf_counter()
            now = dict(params, cam_unnorm_rots=rots, cam_trans=trans)
            healthy = reloc.read_health(reloc.health(now, frame, t, reloc_cfg, render, fused))["ok"]
            timing["health_s"] += time.perf_counter() - t0
            if not healthy:
                t0 = time.perf_counter()
                rec = reloc.relocalise(now, frame, t, reloc_db, intrinsics, reloc_cfg, render=render, fused=fused,
                                       tracking=dict(num_iters=tracking_iters, lr_rot=tracking_lrs[0],
                                                     lr_trans=tracking_lrs[1], depth_loss_thres=depth_loss_thres))
                rots, trans = now["cam_unnorm_rots"].detach(), now["cam_trans"].detach()
                h = rec["health"] or {}
                reloc_recs.append(dict(frame=t, relocalised=rec["accepted"], candidate=(
                    reloc_db.columns[rec["chosen"]] if rec["chosen"] is not None else None),
                    score=(rec["scores"][rec["candidates"].index(rec["chosen"])] if rec["chosen"] is not None
                           else None), coverage=h.get("coverage"), inlier_frac=h.get("inlier_frac"), rms=h.get("rms"),
                    candidates=rec["columns"], scores=rec["scores"], icp=rec["icp"],
                    **({"ncc": h.get("ncc")} if reloc_cfg["photometric"] else {})))
                if not rec["accepted"]:
                    with torch.no_grad():
                        rots[..., t] = rots[..., t - 1]
                        trans[..., t] = trans[..., t - 1]
                mapper.cam = dict(cam_unnorm_rots=rots, cam_trans=trans)
                cam_now = mapper.sync_camera()
                rots, trans = cam_now["cam_unnorm_rots"], cam_now["cam_trans"]
                torch.cuda.synchronize(dev)
                timing["reloc_s"] += time.perf_counter() - t0
                if not rec["accepted"]:
                    reloc_lost.add(t)
                    checkpoint(t)
                    continue
                reloc_done.add(t)
        loop_kf = None
        if use_loop and t % keyframe_every == 0:
            t0 = time.perf_counter()
            pose_graph.add_odometry(pose_graph.nodes()[-1], t, pose_graph.odometry_from(rots, trans, t))
            recs, loop_kf = loop.close_loop(t, frame, keyframes, rots, trans, pose_graph, intrinsics, loop_cfg, seed,
                                            mapper)
            loops += recs
            rots, trans = mapper.cam["cam_unnorm_rots"], mapper.cam["cam_trans"]    # sync_camera may replace them
            torch.cuda.synchronize(dev)
            timing["loop_closure_s"] += time.perf_counter() - t0
        cur = dict(_without_densify(frame), est_w2c=_curr_w2c(rots, trans, t))
        grow_kw = {}
        if use_dyn:       # the frame's masks at its pose of record: identical on every rank (same replica, same kernels)
            now = dict({k: v.detach() for k, v in mapper.g.params.items()}, cam_unnorm_rots=rots, cam_trans=trans,
                       **({"cam_exposure": mapper.cam["cam_exposure"]} if use_expo else {}))
            trk_fused = (dev.type == "cuda" and render is None) if fused is None else bool(fused)
            with torch.no_grad():
                _, depth_sil, _, _ = M._render_pair(now, frame, render or M.default_render, trk_fused,
                                                    camera_grad=False)
                dyn_now, _, st_now = _dynamic.masks(depth_sil, frame["depth"], dyn_cfg, 0.99, trk_fused)
            cur["dynamic"] = dyn_now.clone()
            grow_kw = dict(exclude=cur["dynamic"])
            dyn_stats.append(st_now)
        if t % map_every == 0:
            if add_new_gaussians:
                if "densify" in frame:            # SplaTAM-S: grow the map from the densification-size frame
                    mapper.add_new_gaussians(frame["densify"], t, frame["densify"]["intrinsics"], sil_thres, **grow_kw)
                else:
                    mapper.add_new_gaussians(frame, t, intrinsics, sil_thres, **grow_kw)
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
            if loop_kf is not None and len(win) >= 2 and all(w is not keyframes[loop_kf] for w in win):
                win[0] = keyframes[loop_kf]               # the seam between the loop's two ends gets optimised
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
            if refine:
                rots, trans = refined_cameras()
                cur["est_w2c"] = _curr_w2c(rots, trans, t)
        if t % keyframe_every == 0:
            keyframes.append(cur)
            if use_reloc:
                reloc_db.add(frame, t)
            if checkpoint_dir is not None and checkpoint_every is None:
                from . import formats
                formats.save_params_ckpt(dict(mapper.g.params, cam_unnorm_rots=rots, cam_trans=trans), checkpoint_dir, t)
        checkpoint(t)
    # PSNR of the keyframes re-rendered from the final map at the estimated poses
    final = {k: v.detach() for k, v in mapper.g.params.items()}
    vals = []
    for fr in keyframes:
        est = render_frame(final, rots, trans, fr["id"], cam, render)
        if use_expo:
            from .train_ops import exposure as _exposure, exposure_torch
            ab = mapper.cam["cam_exposure"][0, :, fr["id"]]
            est["im"] = _exposure(est["im"], ab) if mapper.fused else exposure_torch(est["im"], ab)
        vals.append(psnr(est["im"].clamp(0, 1), fr["im"].clamp(0, 1)))
    if checkpoint_dir is not None and (checkpoint_every is None or mapper.rank == 0):
        from . import formats
        formats.save_params(dict(final, cam_unnorm_rots=rots, cam_trans=trans), checkpoint_dir)
    out = dict(rots=rots, trans=trans, psnr=sum(vals) / len(vals), gauss=final, counts=counts,
               timestep=mapper.timestep.detach().clone(), keyframe_time_indices=[int(kf["id"]) for kf in keyframes],
               keyframe_est_w2c=[kf["est_w2c"] for kf in keyframes])
    if use_expo:
        out["exposure"] = mapper.cam["cam_exposure"].detach().clone()
    if use_dyn:
        st = torch.stack(dyn_stats).cpu().numpy() if dyn_stats else np.zeros((0, _dynamic.STATS), np.float32)
        npx = float(frames[0]["depth"].shape[-2] * frames[0]["depth"].shape[-1])
        out["dynamic"] = [dict(frame=start + i, scale=float(s[1]), dynamic_frac=float(s[4]) / npx,
                               inconsistent_frac=float(s[5]) / npx) for i, s in enumerate(st)]
        out["keyframe_dynamic"] = [kf["dynamic"] for kf in keyframes]
    if use_icp:
        st = torch.stack(icp_stats).cpu().numpy() if icp_stats else np.zeros((0, icp.STATS))
        out["icp"] = [dict(frame=start + i, accepted=bool(s[0]), inlier_frac=float(s[1]), rms=float(s[2]),
                           **({"photo_rms": float(s[37])} if pose_init == "rgbd_icp" else {}))
                      for i, s in enumerate(st)]
    if use_loop:
        out["loops"] = loops
    if use_reloc:
        out.update(reloc=reloc_recs, reloc_lost=sorted(reloc_lost), reloc_database=reloc_db)
    return out


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
