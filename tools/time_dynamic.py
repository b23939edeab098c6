"""Measures the motion masks (csrc/dynamic.cu, splatam_b200/dynamic.py, slam.run_slam's `dynamic`) on the GPU and
prints one JSON line with the card's name and power limit, read in the same call:

  kernels   the five kernels' time per frame at 320x192 and 1200x680 with the default options (CUDA events over 200
            calls of dynamic.motion_masks on scenes.motion_mask_frame)
  runs      with --runs: tools/run_slam_dataset.py (Replica's settings, --pose-init icp) with and without --dynamic on
            scenes.write_dynamic_sequence (the box enters; and with present_at_start, the box leaves) and on the static
            scenes.write_loop_sequence, all at Replica's 1200x680 and --frames frames (`end_to_end`): ATE, tracking
            and whole-run wall time, ghost Gaussians (final-map centres inside the box's swept volume grown by 5 cm),
            motion-mask recall on the ground-truth masks and the flagged share of static pixels over the keyframes,
            and the keyframes' PSNR over ground-truth static pixels

  python tools/time_dynamic.py --runs --frames 81"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402
import torch  # noqa: E402

import scenes  # noqa: E402
from splatam_b200 import dynamic as D  # noqa: E402


def _events(fn, n):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(n):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / n


def _run_tool(base, name, dynamic, frames):
    out_dir = os.path.join(base, "out_%s_%s" % (name, "on" if dynamic else "off"))
    cmd = [sys.executable, os.path.join(ROOT, "tools", "run_slam_dataset.py"), "--dataset", "replica", "--basedir",
           base, "--sequence", name, "--frames", str(frames), "--out", out_dir, "--pose-init", "icp"] + (
               ["--dynamic"] if dynamic else [])
    res = json.loads(subprocess.run(cmd, check=True, capture_output=True, text=True).stdout.strip().splitlines()[-1])
    res.pop("hyper", None)
    return res, out_dir


def _keyframe_scores(base, name, out_dir, box_track=None):
    """(ghost Gaussians, keyframe PSNR over ground-truth static pixels, mask recall, flagged static share) of a run
    record under out_dir; the last two only when dynamic.npz exists, the first only with a `box_track`."""
    from PIL import Image
    import splatam_b200 as S
    from splatam_b200 import formats, slam
    dev = torch.device("cuda", 0)
    with np.load(os.path.join(out_dir, "params.npz")) as z:
        p = {k: torch.from_numpy(np.asarray(z[k])).float().to(dev) for k in
             ("means3D", "rgb_colors", "unnorm_rotations", "logit_opacities", "log_scales", "cam_unnorm_rots",
              "cam_trans")}
        kf = [int(i) for i in np.asarray(z["keyframe_time_indices"]).reshape(-1)]
    out = {}
    if box_track is not None:
        half = np.array(scenes.DYNAMIC_BOX) / 2 + 0.05
        lo, hi = box_track.min(0) - half, box_track.max(0) + half
        m = p["means3D"].cpu().numpy()
        out["ghosts"] = int(((m >= lo) & (m <= hi)).all(1).sum())
    cam = scenes.loop_room(cam=scenes.REPLICA, P=16).settings(S.GaussianRasterizationSettings, dev)
    gauss = {k: p[k] for k in ("means3D", "rgb_colors", "unnorm_rotations", "logit_opacities", "log_scales")}
    se, n = 0.0, 0
    for t in kf:
        est = slam.render_frame(gauss, p["cam_unnorm_rots"], p["cam_trans"], t, cam)["im"].clamp(0, 1)
        gt = torch.from_numpy(np.asarray(Image.open(os.path.join(base, name, "results", "frame%06d.jpg" % t)),
                                         np.float32) / 255.0).permute(2, 0, 1).to(dev)
        mpath = os.path.join(base, name, "masks", "mask%06d.png" % t)
        static = torch.ones(gt.shape[1:], dtype=torch.bool, device=dev) if not os.path.exists(mpath) else \
            torch.from_numpy(np.asarray(Image.open(mpath)) < 128).to(dev)
        d = (est - gt)[:, static]
        se += float((d * d).sum())
        n += d.numel()
    out["static_psnr_db"] = -10.0 * np.log10(se / max(n, 1))
    path = os.path.join(out_dir, "dynamic.npz")
    if os.path.exists(path) and os.path.exists(os.path.join(base, name, "masks")):
        rec = formats.load_dynamic(path)
        tp = fn = fp = tn = 0
        for t, m in zip(rec["keyframe_ids"], rec["keyframe_masks"]):
            if t == 0:
                continue                      # frame 0 initialises the map and has no mask
            gtm = np.asarray(Image.open(os.path.join(base, name, "masks", "mask%06d.png" % t))) >= 128
            tp += int((m & gtm).sum()); fn += int((~m & gtm).sum())
            fp += int((m & ~gtm).sum()); tn += int((~m & ~gtm).sum())
        out.update(mask_recall=tp / max(tp + fn, 1), static_flagged=fp / max(fp + tn, 1))
    return out


def end_to_end(base, frames):
    """Writes the three sequences under `base` and runs the tool on each with and without --dynamic; returns a list of
    dicts (case, dynamic, the tool's JSON numbers and `_keyframe_scores`)."""
    dev = torch.device("cuda", 0)
    tracks = {}
    for name, present in (("enters", False), ("leaves", True)):
        _, poses = scenes.write_dynamic_sequence(os.path.join(base, name), frames, dev, cam=scenes.REPLICA,
                                                 present_at_start=present)
        tracks[name] = poses[:, :3, 3]
    scenes.write_loop_sequence(os.path.join(base, "static"), frames, dev, cam=scenes.REPLICA)
    rows = []
    for name in ("enters", "leaves", "static"):
        for dyn in (False, True):
            res, out_dir = _run_tool(base, name, dyn, frames)
            row = dict(case=name, dynamic=dyn, ate_m=res["ate_m"], psnr_db=res["psnr_db"],
                       gaussians=res["gaussians"], wall_s=res["wall_s"], tracking_s=res["tracking_s"],
                       mapping_s=res["mapping_s"], tracking_ms_per_frame=1e3 * res["tracking_s"] / max(frames - 1, 1),
                       **{k: res[k] for k in ("dynamic_frac_median", "dynamic_frac_max") if k in res})
            row.update(_keyframe_scores(base, name, out_dir, tracks.get(name)))
            rows.append(row)
            print(json.dumps(row), file=sys.stderr, flush=True)         # progress: one line per run
    return rows


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--runs", action="store_true", help="also the end-to-end runs")
    ap.add_argument("--frames", type=int, default=81)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "time_dynamic needs a CUDA device"
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    out = dict(card=card, defaults=D.DEFAULTS, kernels_ms={})
    for H, W in ((192, 320), (680, 1200)):
        ds, g = scenes.motion_mask_frame(H, W, seed=1, objects=4)
        ds, g = torch.from_numpy(ds).cuda(), torch.from_numpy(g).cuda()
        out["kernels_ms"]["%dx%d" % (W, H)] = round(_events(lambda: D.motion_masks(ds, g, D.DEFAULTS), 200), 4)
    if a.runs:
        with tempfile.TemporaryDirectory() as base:
            out["runs"] = end_to_end(base, a.frames)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
