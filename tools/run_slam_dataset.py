#!/usr/bin/env python
"""SplaTAM on a recorded sequence: reads Replica, TUM-RGBD, ScanNet, ScanNet++, ReplicaV2 or a NeRFCapture iPhone
capture (rgb/, depth/, transforms.json; --dataset nerfcapture, evaluated against its ARKit poses) from disk
(splatam_b200.datasets), runs the SLAM loop (splatam_b200.slam.run_slam) from the back-projection of frame 0 with the
shipped hyper-parameters of R/configs/{replica,tum,scannet,scannetpp,replica_v2}/splatam.py, then the final evaluation
(splatam_b200.evaluate) against the dataset's ground-truth poses.  ScanNet++ and ReplicaV2 run on their train split;
with --nvs the test split is read too and the novel-view evaluation (evaluate.evaluate_nvs) is reported as well.
--variant splatam_s runs SplaTAM-S (R/configs/replica/splatam_s.py, Replica only): 10 tracking and 15 mapping
iterations, a window of 32, and new Gaussians -- the initial map included -- from each frame read at 340x600.
One GPU.

  python tools/run_slam_dataset.py --dataset replica --basedir data/Replica --sequence room0
  python tools/run_slam_dataset.py --dataset replica --basedir data/Replica --sequence room0 --variant splatam_s
  python tools/run_slam_dataset.py --dataset tum --basedir data/TUM_RGBD --sequence rgbd_dataset_freiburg1_desk
  python tools/run_slam_dataset.py --dataset scannetpp --basedir data/ScanNet++/data --sequence 8b5caf3398 --nvs

--config takes a data YAML of the reference's shape (default: the shipped camera of the dataset); --start / --end /
--stride select frames as the reference does; --frames caps the number of frames; --tracking-iters / --mapping-iters
override the shipped iteration counts; --pose-init icp starts each frame's tracking from a point-to-plane ICP
alignment of its depth with the map's (splatam_b200.icp; default constant_velocity, the reference's guess), and
--pose-init rgbd_icp from a joint alignment of its depth and colour with the map's renders;
--loop-closure closes loops against old keyframes with splatam_b200.loop's defaults and prints every closure attempt.
--relocalise checks every tracked frame against the map and relocalises lost ones against the keyframes
(splatam_b200.reloc's defaults) and prints every lost frame; --relocalise-photometric does so with the photometric
health check and RGB-D ICP verification.  Prints one JSON line: ATE, PSNR, MS-SSIM, depth L1, initial and final
Gaussian counts, tracking
and mapping wall times, and the load time per frame that the SLAM loop waited for (decode + upload not hidden by the
prefetch).  --out DIR writes the reference's psnr.txt / rmse.txt / l1.txt / ssim.txt and its full params.npz record
(formats.save_run_record: the Gaussians, the cameras, `timestep`, `intrinsics`, `w2c`, `org_width` / `org_height`,
`gt_w2c_all_frames` and `keyframe_time_indices`), which the reference's viewers and post_splatam_opt.py open.
--lpips-alexnet PATH --lpips-lin PATH (both or neither: torchvision's alexnet-owt-7be5be79.pth and LPIPS v0.1's
alex.pth, read from disk, never downloaded) add LPIPS to the evaluation: `lpips` (and `nvs_lpips` with --nvs) in the
JSON line and lpips.txt under --out.
--save-frames (needs --out) also saves the final evaluation's rendered and ground-truth colour and depth PNGs under
--out (rendered_rgb/, rendered_depth/, rgb/, depth/), and with --nvs those of the novel views under --out/eval_nvs.
--dynamic (not with --relocalise) gives each frame a motion mask from the map's depth residual and keeps its pixels
out of tracking, mapping and map growth (slam.run_slam's `dynamic`); the JSON line gains the median and largest
flagged share of a frame, and --out receives dynamic.npz (formats.save_dynamic: per-frame stats, keyframe masks).
--checkpoint-every N writes the reference's params{t}.npz / keyframe_time_indices{t}.npy, and a run_state{t}.npz
sidecar, under --out every N frames; --resume T continues the run from the checkpoint of frame T under --out (one
written here, or the reference's own, which then continues without the sidecar's RNG states):

  python tools/run_slam_dataset.py --dataset replica --basedir data/Replica --sequence room0 --out runs/room0 \\
      --checkpoint-every 100
  python tools/run_slam_dataset.py --dataset replica --basedir data/Replica --sequence room0 --out runs/room0 \\
      --checkpoint-every 100 --resume 1500"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402
import torch  # noqa: E402

_PRUNE = dict(start_after=0, remove_big_after=0, stop_after=20, prune_every=20, removal_opacity_threshold=0.005,
              final_removal_opacity_threshold=0.005, reset_opacities=False, reset_opacities_every=500)
# R/configs/<dataset>/splatam.py: image size, iterations, keyframe / map period, window, radius ratio, eval period
HYPER = {
    "replica": dict(height=680, width=1200, tracking_iters=40, mapping_iters=60, keyframe_every=5, map_every=1,
                    window=24, scene_radius_depth_ratio=3, eval_every=5),
    "tum": dict(height=480, width=640, tracking_iters=200, mapping_iters=30, keyframe_every=5, map_every=1, window=20,
                scene_radius_depth_ratio=2, eval_every=500),
    "scannet": dict(height=480, width=640, tracking_iters=100, mapping_iters=30, keyframe_every=5, map_every=1,
                    window=10, scene_radius_depth_ratio=3, eval_every=500),
    "scannetpp": dict(height=584, width=876, tracking_iters=200, mapping_iters=60, keyframe_every=5, map_every=1,
                      window=24, scene_radius_depth_ratio=3, eval_every=1, tracking_lrs=(0.001, 0.004),
                      depth_loss_thres=20000),
    "replicav2": dict(height=680, width=1200, tracking_iters=40, mapping_iters=60, keyframe_every=5, map_every=1,
                      window=24, scene_radius_depth_ratio=3, eval_every=5),
    # R/configs/iphone/splatam.py: half the phone's 1920x1440, new Gaussians from the quarter-size frame;
    # keyframe_every depends on the frame count (nerfcapture_keyframe_every)
    "nerfcapture": dict(height=720, width=960, densify_height=360, densify_width=480, tracking_iters=60,
                        mapping_iters=60, keyframe_every=None, map_every=1, window=32, scene_radius_depth_ratio=3,
                        eval_every=1, tracking_lrs=(0.001, 0.004), depth_loss_thres=20000),
}
# R/configs/replica/splatam_s.py: SplaTAM-S, the fast variant; new Gaussians come from the frame read at the
# densification size (340x600) while tracking and mapping use 680x1200
VARIANTS = ("splatam", "splatam_s")
HYPER_S = {
    "replica": dict(height=680, width=1200, densify_height=340, densify_width=600, tracking_iters=10,
                    mapping_iters=15, keyframe_every=5, map_every=1, window=32, scene_radius_depth_ratio=3,
                    eval_every=5),
}
# rows without these keys track with Replica's rates and without the depth-loss rule
# (follow-up: the shipped TUM and ScanNet configs have their own tracking rates)
_TRACKING_DEFAULTS = dict(tracking_lrs=(0.0004, 0.002), depth_loss_thres=None)
SIL_THRES = 0.5          # mapping: add_new_gaussians' silhouette threshold


def nerfcapture_keyframe_every(frames):
    """R/configs/iphone/*.py: frames // 5 below 25 frames, else 5; fewer than 5 frames would make it 0 (the reference
    then divides by zero), so they are rejected."""
    if frames < 5:
        raise ValueError("a NeRFCapture run needs at least 5 frames, got %d" % frames)
    return frames // 5 if frames < 25 else 5


class _Capped:
    """The first n frames of a sequence (the loop and the evaluation only use len() and [t])."""

    def __init__(self, seq, n):
        self.seq, self.n = seq, min(n, len(seq)) if n else len(seq)

    def __len__(self):
        return self.n

    def __getitem__(self, t):
        if not 0 <= t < self.n:
            raise IndexError(t)
        return self.seq[t]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--dataset", required=True, choices=sorted(HYPER))
    ap.add_argument("--basedir", required=True)
    ap.add_argument("--sequence", required=True)
    ap.add_argument("--config", default=None, help="data YAML (camera_params); default: the shipped camera")
    ap.add_argument("--start", type=int, default=0)
    ap.add_argument("--end", type=int, default=-1)
    ap.add_argument("--stride", type=int, default=1)
    ap.add_argument("--frames", type=int, default=0, help="use only the first N selected frames (0: all)")
    ap.add_argument("--tracking-iters", type=int, default=0)
    ap.add_argument("--mapping-iters", type=int, default=0)
    ap.add_argument("--prefetch", type=int, default=2)
    ap.add_argument("--out", default=None)
    ap.add_argument("--nvs", action="store_true", help="also evaluate novel views on the test split "
                                                       "(scannetpp, replicav2)")
    ap.add_argument("--variant", default="splatam", choices=VARIANTS,
                    help="splatam_s: SplaTAM-S, the fast variant (replica only)")
    ap.add_argument("--lpips-alexnet", default=None, help="torchvision AlexNet weights (alexnet-owt-7be5be79.pth)")
    ap.add_argument("--lpips-lin", default=None, help="LPIPS v0.1 linear heads (alex.pth)")
    ap.add_argument("--checkpoint-every", type=int, default=0,
                    help="write a checkpoint under --out every N frames (0: off); the reference's shipped "
                         "checkpoint_interval is 100 for Replica, TUM, ScanNet and ReplicaV2 and 5 for ScanNet++")
    ap.add_argument("--resume", type=int, default=None, metavar="T",
                    help="continue from the checkpoint of frame T under --out")
    ap.add_argument("--save-frames", action="store_true",
                    help="save the evaluation's rendered and ground-truth frames under --out")
    ap.add_argument("--mapping-cam-lrs", type=float, nargs=2, default=(0.0, 0.0), metavar=("ROT", "TRANS"),
                    help="mapping learning rates of cam_unnorm_rots and cam_trans; non-zero refines each mapping "
                         "iteration's keyframe pose (the reference's do_ba=True); default 0 0, as every shipped config")
    ap.add_argument("--pose-init", default="constant_velocity", choices=("constant_velocity", "icp", "rgbd_icp"),
                    help="tracking start: the reference's constant-velocity guess, or that guess refined by ICP "
                         "(rgbd_icp: depth and colour)")
    ap.add_argument("--loop-closure", action="store_true",
                    help="close loops against old keyframes (splatam_b200.loop, its DEFAULTS); off by default")
    ap.add_argument("--relocalise", action="store_true",
                    help="health-check every frame and relocalise lost ones (splatam_b200.reloc, its DEFAULTS); off by "
                         "default")
    ap.add_argument("--relocalise-photometric", action="store_true",
                    help="--relocalise with the photometric health check and RGB-D ICP verification (implies "
                         "--relocalise)")
    ap.add_argument("--exposure", action="store_true",
                    help="estimate each frame's exposure and white balance while tracking, and map and evaluate "
                         "through it (slam.run_slam's `exposure`, its EXPOSURE_DEFAULTS); with --out also writes "
                         "exposure.npz; off by default")
    ap.add_argument("--dynamic", action="store_true",
                    help="estimate a motion mask per frame and keep its pixels out of tracking, mapping and map "
                         "growth (slam.run_slam's `dynamic`, dynamic.DEFAULTS); with --out also writes dynamic.npz; "
                         "off by default")
    a = ap.parse_args()
    a.relocalise = a.relocalise or a.relocalise_photometric
    if a.exposure and a.relocalise:
        ap.error("--exposure cannot be combined with --relocalise")
    if a.dynamic and a.relocalise:
        ap.error("--dynamic cannot be combined with --relocalise")
    if (a.lpips_alexnet is None) != (a.lpips_lin is None):
        ap.error("--lpips-alexnet and --lpips-lin go together")
    if a.checkpoint_every < 0:
        ap.error("--checkpoint-every must be 0 (off) or positive")
    if (a.checkpoint_every or a.resume is not None) and a.out is None:
        ap.error("--checkpoint-every and --resume need --out")
    if a.save_frames and a.out is None:
        ap.error("--save-frames needs --out")
    if a.nvs and a.dataset not in ("scannetpp", "replicav2"):
        ap.error("--nvs needs a dataset with a test split (scannetpp, replicav2)")
    if a.variant == "splatam_s" and a.dataset not in HYPER_S:
        ap.error("--variant splatam_s has a shipped config for %s only" % ", ".join(sorted(HYPER_S)))
    from splatam_b200 import datasets, evaluate, slam
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    torch.manual_seed(0); np.random.seed(0)
    h = dict(_TRACKING_DEFAULTS, **(HYPER_S if a.variant == "splatam_s" else HYPER)[a.dataset])
    h["tracking_iters"] = a.tracking_iters or h["tracking_iters"]
    h["mapping_iters"] = a.mapping_iters or h["mapping_iters"]
    cfg = datasets.load_config(a.config) if a.config else None
    net = None if a.lpips_alexnet is None else evaluate.LpipsAlex.load(a.lpips_alexnet, a.lpips_lin, dev)
    seq = datasets.RGBDSequence(a.dataset, a.basedir, a.sequence, cfg, start=a.start, end=a.end, stride=a.stride,
                                desired_height=h["height"], desired_width=h["width"], device=dev, prefetch=a.prefetch,
                                densify_height=h.get("densify_height"), densify_width=h.get("densify_width"))
    frames = _Capped(seq, a.frames)
    T = len(frames)
    if a.dataset == "nerfcapture":
        try:
            h["keyframe_every"] = nerfcapture_keyframe_every(T)
        except ValueError as e:
            ap.error(str(e))
    K = seq.intrinsics.cpu()
    from splatam_b200 import formats
    t_resume = time.perf_counter()
    # the initial map and the scene radius come from the densification-size frame 0 when there is one
    # (splatam.py:185-206): its max depth can be below the full-size one; a resumed run reads frame 0 for the radius
    # only, as the reference still computes it there
    first = frames[0].get("densify", frames[0])
    radius = float(first["depth"].max()) / h["scene_radius_depth_ratio"]
    if a.resume is None:
        init, _ = slam.initialize_map(first, first["intrinsics"].cpu())
        ckpt = None
    else:
        init, ckpt = None, formats.load_checkpoint(a.out, a.resume, dev)
    initial_gaussians = int((init if ckpt is None else ckpt["gauss"])["means3D"].shape[0])
    timing = {}
    wait0 = seq.load_wait_s
    torch.cuda.synchronize(dev)
    t0 = time.perf_counter()
    out = slam.run_slam(init, frames, seq.cam, seed=0, timing=timing, tracking_iters=h["tracking_iters"],
                        mapping_iters=h["mapping_iters"], keyframe_every=h["keyframe_every"], map_every=h["map_every"],
                        window=h["window"], sil_thres=SIL_THRES, intrinsics=K, add_new_gaussians=True, prune_dict=_PRUNE,
                        scene_radius=radius, select_keyframes=True, first_frame_iters=h["mapping_iters"],
                        checkpoint_dir=a.out if a.checkpoint_every else None,
                        checkpoint_every=a.checkpoint_every or None, resume=ckpt,
                        tracking_lrs=h["tracking_lrs"], depth_loss_thres=h["depth_loss_thres"],
                        mapping_cam_lrs=tuple(a.mapping_cam_lrs), pose_init=a.pose_init,
                        loop_closure={} if a.loop_closure else None,
                        relocalise=((dict(photometric=True) if a.relocalise_photometric else {}) if a.relocalise
                                    else None),
                        exposure={} if a.exposure else None, dynamic={} if a.dynamic else None)
    torch.cuda.synchronize(dev)
    wall = time.perf_counter() - t0
    # --resume: wall time from reading the checkpoint to the first tracked frame (frame-0 read, load, keyframe rebuild)
    resume_s = None if ckpt is None else t0 - t_resume + timing["setup_s"]
    load_wait = seq.load_wait_s - wait0
    gt = [seq.files.poses[t] for t in range(T)]
    gt_w2c = [torch.linalg.inv(p.to(dev)) for p in gt]
    gt_w2c_all = seq.gt_w2c[:T]                  # the record's gt_w2c_all_frames: NaN where a pose is invalid
    params = dict(out["gauss"], cam_unnorm_rots=out["rots"], cam_trans=out["trans"])
    if a.exposure:                               # scored through each frame's estimated colour correction
        params["cam_exposure"] = out["exposure"]
    res = evaluate.evaluate(params, frames, seq.cam, SIL_THRES, h["mapping_iters"], True, eval_every=h["eval_every"],
                            gt_w2c=gt_w2c, out_dir=a.out, lpips=net, save_frames=a.save_frames)
    seq.close()
    nvs = {}
    if a.nvs:
        with datasets.RGBDSequence(a.dataset, a.basedir, a.sequence, cfg, desired_height=h["height"],
                                   desired_width=h["width"], device=dev, prefetch=a.prefetch, split="test") as test:
            r = evaluate.evaluate_nvs(out["gauss"], test, test.cam, SIL_THRES, h["mapping_iters"], True,
                                      eval_every=h["eval_every"],
                                      out_dir=None if a.out is None else os.path.join(a.out, "eval_nvs"), lpips=net,
                                      save_frames=a.save_frames)
        nvs = dict(nvs_psnr_db=r["psnr"], nvs_ms_ssim=r["ms_ssim"], nvs_depth_rmse_m=r["depth_rmse"],
                   nvs_depth_l1_m=r["depth_l1"], nvs_evaluated_frames=len(r["frame_ids"]),
                   nvs_valid_frames=int(r["valid_nvs_frames"].sum()))
        if net is not None:
            nvs["nvs_lpips"] = r["lpips"]
    if a.out is not None:
        formats.save_run_record(a.out, out["gauss"], out["rots"], out["trans"], out["timestep"], K, seq.w2c, seq.width,
                                seq.height, gt_w2c_all, out["keyframe_time_indices"])
        if a.exposure:
            formats.save_exposure(a.out, out["exposure"])
        if a.dynamic:
            formats.save_dynamic(a.out, out["dynamic"], out["keyframe_time_indices"], out["keyframe_dynamic"])
    dyn = {}
    if a.dynamic:
        fr = [r["dynamic_frac"] for r in out["dynamic"]]
        dyn = dict(dynamic_frac_median=float(np.median(fr)) if fr else 0.0, dynamic_frac_max=max(fr, default=0.0))
    print(json.dumps(dict(
        dataset=a.dataset, sequence=a.sequence, variant=a.variant, frames=T, width=seq.width, height=seq.height,
        densify_height=seq.densify_height, densify_width=seq.densify_width, hyper=h,
        initial_gaussians=initial_gaussians, resumed_from=a.resume, resume_s=resume_s,
        mapping_cam_lrs=list(a.mapping_cam_lrs), pose_init=a.pose_init, exposure=a.exposure, dynamic=a.dynamic, **dyn,
        **({} if a.pose_init == "constant_velocity" else dict(pose_init_s=timing["pose_init_s"],
                                                icp_accepted=sum(s["accepted"] for s in out["icp"]))),
        **({} if not a.loop_closure else dict(loop_closure_s=timing["loop_closure_s"], loops=out["loops"])),
        **({} if not a.relocalise else dict(health_s=timing["health_s"], reloc_s=timing["reloc_s"], reloc=out["reloc"],
                                            reloc_lost=out["reloc_lost"])),
        ate_m=res["ate"], psnr_db=res["psnr"], ms_ssim=res["ms_ssim"], depth_l1_m=res["depth_l1"],
        gaussians=int(out["counts"][-1]), wall_s=wall, tracking_s=timing["tracking_s"], mapping_s=timing["mapping_s"],
        load_wait_ms_per_frame=1e3 * load_wait / max(T - 1, 1), evaluated_frames=len(res["frame_ids"]),
        tracking_iters=timing["tracking_iters"], **({} if net is None else dict(lpips=res["lpips"])), **nvs,
        metric_note="ate_m = the reference's Final Average ATE RMSE (mean Horn-aligned residual); load_wait = host "
                    "time run_slam spent in the reader for frames 1..T-1")))


if __name__ == "__main__":
    main()
