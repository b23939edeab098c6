#!/usr/bin/env python
"""Measures ICP pose initialisation (splatam_b200/icp.py, csrc/icp.cu) on one GPU, and prints the card's name and
power limit first:

(a) icp.align's device time per frame at 1200x680 and 960x720 (CUDA events over `--launches` back-to-back calls,
    default iterations 10 / 5 / 4), and the depth/silhouette render of the map it needs (scenes.room, `--gaussians`);
    then icp.align and icp.align_rgbd alternated three times;
(b) tools/run_slam_dataset.py on a synthetic Replica-layout sequence (scenes.write_replica_sequence, `--frames`
    frames) at each `--strides` value, for constant velocity with 40 tracking iterations, ICP with 40 and ICP with 10:
    ATE, tracking and pose-initialisation wall time per frame and the accepted ICP poses.  One JSON line per run.

Run:  python tools/time_icp.py [--frames 40] [--strides 1 4] [--launches 50]
      python tools/time_icp.py --sizes 97x45 --launches 2 --skip-slam      (a quick check at a tiny size)"""
import argparse
import json
import math
import os
import subprocess
import sys
import tempfile
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import scenes  # noqa: E402
from gpu_info import gpu_info  # noqa: E402

RUNS = (("constant_velocity", 40), ("icp", 40), ("icp", 10), ("rgbd_icp", 40))


def _size(s):
    w, h = (int(x) for x in s.lower().split("x"))
    return w, h


def align_time(dev, w, h, gaussians, launches):
    """(align ms, render ms, stats) per frame at w x h: the map seen from two poses 6 cm and 3 degrees apart."""
    import splatam_b200 as S
    from splatam_b200 import icp, mapping as M
    f = 0.5 * w
    sc = scenes.room(seed=31, P=gaussians, cam=dict(w=w, h=h, fx=f, fy=f, cx=(w - 1) / 2, cy=(h - 1) / 2))
    cam = sc.settings(S.GaussianRasterizationSettings, dev)
    gt = {k: v.to(dev) for k, v in sc.splatam_params().items()}
    rots = torch.zeros(1, 4, 2, device=dev)
    rots[0, 0] = 1.0
    a = math.radians(3.0) / 2
    rots[0, :, 1] = torch.tensor([math.cos(a), 0.0, math.sin(a), 0.0])
    trans = torch.zeros(1, 3, 2, device=dev)
    trans[0, :, 1] = torch.tensor([0.06, 0.0, 0.0])
    params = dict(gt, cam_unnorm_rots=rots, cam_trans=trans)
    frame = dict(cam=cam, w2c=torch.eye(4, device=dev))
    K = [[f, 0, (w - 1) / 2], [0, f, (h - 1) / 2], [0, 0, 1]]
    ds1 = icp.model_depth_sil(params, 1, frame)
    data = torch.where(ds1[1] > 0.99, ds1[0] / ds1[1], torch.zeros_like(ds1[0]))
    eye = torch.eye(4, device=dev)
    ds0 = icp.model_depth_sil(params, 0, frame)
    _, st = icp.align(ds0, data, K, eye, eye)                                  # warm-up, workspace
    e0, e1, e2 = (torch.cuda.Event(enable_timing=True) for _ in range(3))
    e0.record()
    for _ in range(launches):
        icp.model_depth_sil(params, 0, frame)
    e1.record()
    for _ in range(launches):
        icp.align(ds0, data, K, eye, eye)
    e2.record()
    torch.cuda.synchronize(dev)
    truth = M.camera_w2c(rots[..., 1], trans[..., 1])[0]
    w2c, st = icp.align(ds0, data, K, eye, eye)
    err = (w2c @ torch.linalg.inv(truth)).double().cpu()
    # sb_rgbd_icp_align against sb_icp_align, alternated three times on the same inputs
    im0, _ = icp.model_render(params, 0, frame)
    im1, _ = icp.model_render(params, 1, frame)
    icp.align_rgbd(ds0, im0, data, im1, K, eye, eye)
    geo, rgbd = [], []
    for _ in range(3):
        for fn, acc in ((lambda: icp.align(ds0, data, K, eye, eye), geo),
                        (lambda: icp.align_rgbd(ds0, im0, data, im1, K, eye, eye), rgbd)):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(launches):
                fn()
            b.record()
            torch.cuda.synchronize(dev)
            acc.append(round(a.elapsed_time(b) / launches, 4))
    w2c_r, st_r = icp.align_rgbd(ds0, im0, data, im1, K, eye, eye)
    err_r = (w2c_r @ torch.linalg.inv(truth)).double().cpu()
    return dict(render_ms=e0.elapsed_time(e1) / launches, align_ms=e1.elapsed_time(e2) / launches,
                stats=icp.read_stats(st), trans_err_mm=1e3 * float(err[:3, 3].abs().max()),
                rot_err_deg=math.degrees(math.acos(max(-1.0, min(1.0, (float(err[:3, :3].trace()) - 1) / 2)))),
                alternated_align_ms=geo, alternated_rgbd_align_ms=rgbd, rgbd_stats=icp.read_stats(st_r),
                rgbd_trans_err_mm=1e3 * float(err_r[:3, 3].abs().max()))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", nargs="+", default=["1200x680", "960x720"])
    ap.add_argument("--gaussians", type=int, default=200_000)
    ap.add_argument("--launches", type=int, default=50)
    ap.add_argument("--frames", type=int, default=40)
    ap.add_argument("--strides", type=int, nargs="+", default=[1, 4])
    ap.add_argument("--skip-slam", action="store_true")
    a = ap.parse_args()
    sizes = [_size(s) for s in a.sizes]
    if not torch.cuda.is_available():
        raise SystemExit("time_icp.py measures on a CUDA device; none is visible")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    print(json.dumps(dict(part="gpu", gpu=gpu_info())), flush=True)
    for w, h in sizes:
        r = align_time(dev, w, h, a.gaussians, a.launches)
        print(json.dumps(dict(part="align", width=w, height=h, gaussians=a.gaussians, launches=a.launches, **r)),
              flush=True)
    if a.skip_slam:
        return
    with tempfile.TemporaryDirectory() as base:
        scenes.write_replica_sequence(os.path.join(base, "room0"), a.frames, dev)
        torch.cuda.empty_cache()
        for stride in a.strides:
            for mode, iters in RUNS:
                t0 = time.perf_counter()
                out = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "run_slam_dataset.py"), "--dataset",
                                      "replica", "--basedir", base, "--sequence", "room0", "--stride", str(stride),
                                      "--tracking-iters", str(iters), "--pose-init", mode],
                                     capture_output=True, text=True)
                head = dict(part="slam", stride=stride, pose_init=mode, tracking_iters=iters)
                if out.returncode != 0:
                    print(json.dumps(dict(head, error=out.stderr[-2000:])), flush=True)
                    continue
                r = json.loads(out.stdout.strip().splitlines()[-1])
                n = r["frames"]
                print(json.dumps(dict(head, frames=n, ate_mm=1e3 * r["ate_m"], psnr_db=r["psnr_db"],
                                      tracking_ms_per_frame=1e3 * r["tracking_s"] / n,
                                      pose_init_ms_per_frame=1e3 * r.get("pose_init_s", 0.0) / n,
                                      icp_accepted=r.get("icp_accepted"), wall_s=r["wall_s"],
                                      process_s=time.perf_counter() - t0)), flush=True)


if __name__ == "__main__":
    main()
