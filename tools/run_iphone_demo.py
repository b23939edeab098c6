#!/usr/bin/env python
"""SplaTAM's online iPhone demo (R/scripts/iphone_demo.py with R/configs/iphone/online_demo.py): tracks and maps each
frame as it arrives from the NeRFCapture app and writes the capture as it goes.

  python tools/run_iphone_demo.py --source dds --out captures/splatam_demo          # a phone on DDS domain 0
  python tools/run_iphone_demo.py --source synthetic --frames 10 --out /tmp/demo    # rendered packets, no phone
  python tools/run_iphone_demo.py --source dds --capture-only --frames 50 --out captures/scan   # record only

Packets become frames through capture.LiveCapture: 720x960 (downscale_factor 2) for tracking and mapping and 360x480
(densify_downscale_factor 4) for new Gaussians; the initial map is frame 0's back-projection at 360x480.  Then
slam.run_slam with the demo's hyper-parameters: 60 tracking and 60 mapping iterations, a window of 32, mapping every
frame, keyframe_every = frames // 5 below 25 frames (else 5), tracking rates (0.001, 0.004) with the depth-loss rule at
20000, scene radius = max depth / 3.  --out receives rgb/N.png, depth/N.png and transforms.json (which
`run_slam_dataset.py --dataset nerfcapture` reads back) and the reference's params.npz (formats.save_run_record;
org_width / org_height the tracking size, gt_w2c_all_frames the ARKit poses), which eval_record.py and
render_record.py open.  --pose-init icp starts each frame's tracking from a point-to-plane ICP alignment of its
depth with the map's (splatam_b200.icp; default constant_velocity, the reference's guess).  --exposure estimates each
frame's exposure and white balance while tracking (slam.run_slam's `exposure`) and writes exposure.npz beside
params.npz.  --dynamic keeps each frame's motion mask (moving people, slam.run_slam's `dynamic`) out of tracking,
mapping and map growth and writes dynamic.npz beside params.npz.  --capture-only writes the capture without SLAM, as nerfcapture2dataset.py does.  Prints one
JSON line: ATE against the ARKit poses (the reference's Horn-aligned mean), Gaussian count, wall times, frames/s."""
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
HYPER = dict(height=720, width=960, densify_height=360, densify_width=480, downscale_factor=2.0,
             densify_downscale_factor=4.0, tracking_iters=60, mapping_iters=60, map_every=1, window=32,
             scene_radius_depth_ratio=3, tracking_lrs=(0.001, 0.004), depth_loss_thres=20000, depth_scale=10.0)
SIL_THRES = 0.5


def run(packets, frames, out, capture_only=False, device="cuda:0", tracking_iters=None, mapping_iters=None,
        pose_init="constant_velocity", exposure=False, dynamic=False):
    """The demo over an iterable of CaptureFrame packets; returns the JSON-able result dict."""
    from splatam_b200 import capture, formats, slam
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    from run_slam_dataset import nerfcapture_keyframe_every
    h = dict(HYPER)
    h["tracking_iters"] = tracking_iters or h["tracking_iters"]
    h["mapping_iters"] = mapping_iters or h["mapping_iters"]
    dev = torch.device(device)
    if not capture_only:
        h["keyframe_every"] = nerfcapture_keyframe_every(frames)
    writer = capture.CaptureWriter(out, h["depth_scale"])
    seq = capture.LiveCapture(packets, frames, h["height"], h["width"], h["densify_height"], h["densify_width"],
                              h["downscale_factor"], h["densify_downscale_factor"], device=dev, writer=writer)
    t0 = time.perf_counter()
    res = dict(frames=frames, out=out, hyper=h)
    with seq:
        if capture_only:
            for t in range(frames):
                seq[t]
        else:
            first = seq[0]["densify"]
            radius = float(first["depth"].max()) / h["scene_radius_depth_ratio"]
            init, _ = slam.initialize_map(first, first["intrinsics"].cpu())
            res["initial_gaussians"] = int(init["means3D"].shape[0])
            timing = {}
            K = seq.intrinsics.cpu()
            o = slam.run_slam(init, seq, seq.cam, seed=0, timing=timing, tracking_iters=h["tracking_iters"],
                              mapping_iters=h["mapping_iters"], keyframe_every=h["keyframe_every"],
                              map_every=h["map_every"], window=h["window"], sil_thres=SIL_THRES, intrinsics=K,
                              add_new_gaussians=True, prune_dict=_PRUNE, scene_radius=radius, select_keyframes=True,
                              first_frame_iters=h["mapping_iters"], tracking_lrs=h["tracking_lrs"],
                              depth_loss_thres=h["depth_loss_thres"], pose_init=pose_init,
                              exposure={} if exposure else None, dynamic={} if dynamic else None)
            torch.cuda.synchronize(dev)
            est = slam.w2c_list(o["rots"], o["trans"])
            res.update(ate_m=slam.ate_horn(seq.gt_w2c, est), gaussians=int(o["counts"][-1]),
                       tracking_s=timing["tracking_s"], mapping_s=timing["mapping_s"],
                       tracking_iters=timing["tracking_iters"], pose_init=pose_init, exposure=bool(exposure),
                       dynamic=bool(dynamic))
            if pose_init == "icp":
                res.update(pose_init_s=timing["pose_init_s"], icp_accepted=sum(s["accepted"] for s in o["icp"]))
            formats.save_run_record(out, o["gauss"], o["rots"], o["trans"], o["timestep"], K, seq.w2c, seq.width,
                                    seq.height, seq.gt_w2c, o["keyframe_time_indices"])
            if exposure:
                formats.save_exposure(out, o["exposure"])
            if dynamic:
                formats.save_dynamic(out, o["dynamic"], o["keyframe_time_indices"], o["keyframe_dynamic"])
    torch.cuda.synchronize(dev)
    wall = time.perf_counter() - t0
    res.update(wall_s=wall, frames_per_s=frames / wall, dropped_packets=seq.dropped,
               load_wait_ms_per_frame=1e3 * seq.load_wait_s / frames)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--source", required=True, choices=("dds", "synthetic"))
    ap.add_argument("--out", required=True, help="capture directory (must not hold a capture yet)")
    ap.add_argument("--frames", type=int, default=10, help="frames to capture (online_demo.py: 10)")
    ap.add_argument("--domain-id", type=int, default=0, help="DDS domain of the app (--source dds)")
    ap.add_argument("--capture-only", action="store_true", help="write the capture without running SLAM")
    ap.add_argument("--tracking-iters", type=int, default=0)
    ap.add_argument("--mapping-iters", type=int, default=0)
    ap.add_argument("--seed", type=int, default=14, help="generating scene of --source synthetic")
    ap.add_argument("--pose-init", default="constant_velocity", choices=("constant_velocity", "icp"),
                    help="tracking start: the reference's constant-velocity guess, or that guess refined by ICP")
    ap.add_argument("--exposure", action="store_true",
                    help="estimate each frame's exposure and white balance while tracking; writes exposure.npz")
    ap.add_argument("--dynamic", action="store_true",
                    help="keep each frame's motion mask out of tracking, mapping and map growth; writes dynamic.npz")
    a = ap.parse_args()
    if a.dynamic and a.capture_only:
        ap.error("--dynamic needs SLAM (not --capture-only)")
    if not a.capture_only and a.frames < 5:
        ap.error("SLAM needs at least 5 frames (keyframe_every = frames // 5)")
    from splatam_b200 import capture
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    torch.manual_seed(0); np.random.seed(0)
    if a.source == "dds":
        packets = capture.dds_frames(a.domain_id)
    else:
        packets = capture.synthetic_frames(a.frames, dev, seed=a.seed)
    res = run(packets, a.frames, a.out, a.capture_only, dev, a.tracking_iters, a.mapping_iters, a.pose_init,
              a.exposure, a.dynamic)
    res["source"] = a.source
    print(json.dumps(res))


if __name__ == "__main__":
    main()
