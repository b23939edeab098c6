"""Measures per-frame exposure (csrc/exposure.cu, slam.run_slam's `exposure`) on the GPU and prints one JSON line:

  kernels          sb_exposure_apply and sb_exposure_backward at 1200x680 and 1920x1440 (CUDA events over 200 calls),
                   with the byte bound (apply: 24 B per pixel, x read and y written; backward: 36 B per pixel, x and gy
                   read, gx written) at 3.35 TB/s and its share
  runs             SLAM on two scenes.write_replica_sequence sequences of --frames frames at 1200x680 (Replica's
                   settings with --tracking-iters / --mapping-iters): one whose frames change exposure and white
                   balance (scenes.exposure_profile) and one of constant exposure; exposure off and on alternated
                   --reps times: ATE (the reference's Horn-aligned mean), PSNR of the evaluation (through the estimated
                   corrections when on), tracking ms per frame, and the largest log-gain and bias errors of the
                   estimates against the table
  sweep            the varying sequence at each (lr_log_gain, lr_bias) of --sweep

The card's name and power limit are read in the same call.

  python tools/time_exposure.py --frames 16 --sweep 0.005,0.001 0.01,0.002 0.02,0.004"""
import argparse
import json
import os
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import numpy as np  # noqa: E402
import torch  # noqa: E402


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


def kernels(dev):
    from splatam_b200 import _lib
    out = {}
    g = torch.Generator().manual_seed(0)
    for W, H in ((1200, 680), (1920, 1440)):
        x, gy = torch.rand(3, H, W, generator=g).to(dev), torch.randn(3, H, W, generator=g).to(dev)
        ab = (torch.rand(6, generator=g) * 0.2 - 0.1).to(dev)
        y, gx = torch.empty_like(x), torch.empty_like(x)
        g_ab = torch.empty(6, dtype=torch.float64, device=dev)
        ws = torch.empty(_lib.nbytes("sb_exposure_workspace_bytes", H, W), dtype=torch.uint8, device=dev)
        apply_ms = _events(lambda: _lib.call("sb_exposure_apply", H, W, x, ab, 0, y, device=dev), 200)
        back_ms = _events(lambda: _lib.call("sb_exposure_backward", H, W, x, ab, gy, gx, g_ab, ws, ws.numel(),
                                            device=dev), 200)
        row = {}
        for name, ms, bpp in (("apply", apply_ms, 24), ("backward", back_ms, 36)):
            bound_us = H * W * bpp / 3.35e12 * 1e6
            row[name] = dict(us=round(1e3 * ms, 2), bound_us=round(bound_us, 2), share=round(bound_us / (1e3 * ms), 3))
        out["%dx%d" % (W, H)] = row
    return out


def slam_run(basedir, frames, tracking_iters, mapping_iters, exposure, table):
    """Replica's run_slam_dataset settings on a written sequence -> ATE, PSNR, tracking ms per frame, estimate errors."""
    import run_slam_dataset as RSD
    from splatam_b200 import datasets, evaluate, slam
    dev = torch.device("cuda", 0)
    h = dict(RSD._TRACKING_DEFAULTS, **RSD.HYPER["replica"])
    torch.manual_seed(0); np.random.seed(0)
    with datasets.RGBDSequence("replica", basedir, "room0", desired_height=h["height"], desired_width=h["width"],
                               device=dev) as seq:
        fr = RSD._Capped(seq, frames)
        T = len(fr)
        first = fr[0]
        init, _ = slam.initialize_map(first, first["intrinsics"].cpu())
        timing = {}
        out = slam.run_slam(init, fr, seq.cam, seed=0, timing=timing, tracking_iters=tracking_iters,
                            mapping_iters=mapping_iters, keyframe_every=h["keyframe_every"], map_every=h["map_every"],
                            window=h["window"], sil_thres=RSD.SIL_THRES, intrinsics=seq.intrinsics.cpu(),
                            add_new_gaussians=True, prune_dict=RSD._PRUNE,
                            scene_radius=float(first["depth"].max()) / h["scene_radius_depth_ratio"],
                            select_keyframes=True, first_frame_iters=mapping_iters, tracking_lrs=h["tracking_lrs"],
                            exposure=exposure)
        params = dict(out["gauss"], cam_unnorm_rots=out["rots"], cam_trans=out["trans"])
        if exposure is not None:
            params["cam_exposure"] = out["exposure"]
        gt_w2c = [torch.linalg.inv(seq.files.poses[t].to(dev)) for t in range(T)]
        res = evaluate.evaluate(params, fr, seq.cam, RSD.SIL_THRES, mapping_iters, True, eval_every=1, gt_w2c=gt_w2c)
    row = dict(ate_mm=round(1e3 * res["ate"], 3), psnr_db=round(res["psnr"], 3),
               tracking_ms_per_frame=round(1e3 * timing["tracking_s"] / max(T - 1, 1), 2))
    if exposure is not None:
        est = out["exposure"][0].cpu().numpy()
        ref = np.zeros((T, 6), np.float32) if table is None else table[:T]
        row.update(gain_err_max=round(float(np.abs(est[:3].T - ref[:, :3]).max()), 4),
                   bias_err_max=round(float(np.abs(est[3:].T - ref[:, 3:]).max()), 4))
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=16)
    ap.add_argument("--tracking-iters", type=int, default=40)
    ap.add_argument("--mapping-iters", type=int, default=30)
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--sweep", nargs="*", default=[], metavar="LR_LOG_GAIN,LR_BIAS")
    ap.add_argument("--no-kernels", action="store_true")
    a = ap.parse_args()
    import scenes
    from gpu_info import gpu_info
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    line = dict(gpu=gpu_info(), frames=a.frames, tracking_iters=a.tracking_iters, mapping_iters=a.mapping_iters)
    if not a.no_kernels:
        line["kernels"] = kernels(dev)
    table = scenes.exposure_profile(a.frames)
    with tempfile.TemporaryDirectory() as tmp:
        clip = {}
        for name, tab in (("varying", table), ("constant", None)):
            scenes.write_replica_sequence(os.path.join(tmp, name, "room0"), a.frames, dev, exposure=tab)
        # the share of colour values the profile pushes past [0, 1] (clipped before quantisation)
        import splatam_b200 as S
        from splatam_b200 import slam
        gen = scenes.view_filling(seed=14, cam=scenes.REPLICA, margin=48, opacity=(0.85, 0.95))
        rs = gen.settings(S.GaussianRasterizationSettings, dev)
        gt = dict(means3D=gen.means3D, rgb_colors=gen.colors, unnorm_rotations=gen.rotations,
                  logit_opacities=torch.logit(gen.opacities.clamp(0.02, 0.98)), log_scales=torch.log(gen.scales[:, :1]))
        gt = {k: v.to(dev).contiguous() for k, v in gt.items()}
        rots, trans = slam.look_trajectory(a.frames, dev)
        n_clip = n_all = 0
        for t in range(a.frames):
            im = slam.render_frame(gt, rots, trans, t, rs)["im"]
            row = torch.from_numpy(table[t]).to(dev)
            y = torch.exp(row[:3, None, None]) * im + row[3:, None, None]
            n_clip += int(((y < 0) | (y > 1)).sum() - ((im < 0) | (im > 1)).sum())
            n_all += y.numel()
        clip["varying_extra_clipped_frac"] = n_clip / n_all
        line.update(clip)
        runs = {"varying": [], "constant": []}
        for rep in range(a.reps):
            for name in ("varying", "constant"):
                for expo in ((None, {}) if rep % 2 == 0 else ({}, None)):
                    r = slam_run(os.path.join(tmp, name), a.frames, a.tracking_iters, a.mapping_iters, expo,
                                 table if name == "varying" else None)
                    r["exposure"] = expo is not None
                    runs[name].append(r)
                    print(name, r, file=sys.stderr, flush=True)
        line["runs"] = runs
        sweep = []
        for pair in a.sweep:
            lg, lb = (float(v) for v in pair.split(","))
            r = slam_run(os.path.join(tmp, "varying"), a.frames, a.tracking_iters, a.mapping_iters,
                         dict(lr_log_gain=lg, lr_bias=lb), table)
            r.update(lr_log_gain=lg, lr_bias=lb)
            sweep.append(r)
            print("sweep", r, file=sys.stderr, flush=True)
        line["sweep"] = sweep
    print(json.dumps(line))


if __name__ == "__main__":
    main()
