#!/usr/bin/env python
"""Times the saved evaluation frames (csrc/eval_frames.cu and evaluate(..., save_frames=True)) on one GPU.  Prints the
GPU name and power limit of the run and one JSON line:
  kernel_us             sb_eval_frames_u8 per call at 1200x680 and 876x584, CUDA events over --reps calls, and the
                        bandwidth its 44 bytes per pixel (32 read, 12 written) imply
  png_encode_ms         host time per 1200x680 RGB image to encode with Pillow at the level evaluate uses
                        (evaluate.PNG_COMPRESS_LEVEL) and at Pillow's default (6), median over the four images of a frame
  evaluate_frames_per_s evaluate() over --frames frames of a 1200x680 view-filling map without save_frames, then with
                        it at 1, 2, 4 and 8 writer threads (evaluate.FRAME_WRITER_THREADS); PNGs go to a temporary
                        directory
Run:  python tools/time_eval_frames.py [--frames 100] [--reps 200]"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

import scenes  # noqa: E402

BYTES_PER_PIXEL = 4 * (3 + 1 + 3 + 1) + 4 * 3


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, check=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:          # the name still comes from torch
        return "%s, power limit unknown (%s)" % (torch.cuda.get_device_name(0), e)


def time_kernel(reps):
    from splatam_b200 import evaluate as EV
    dev = torch.device("cuda:0")
    out = {}
    for w, h in ((1200, 680), (876, 584)):
        g = torch.Generator().manual_seed(w)
        im, gt = torch.rand(3, h, w, generator=g).to(dev), torch.rand(3, h, w, generator=g).to(dev)
        ds, gd = (8 * torch.rand(3, h, w, generator=g)).to(dev), (8 * torch.rand(1, h, w, generator=g)).to(dev)
        lut, buf = EV.jet_lut(dev), torch.empty(4, h, w, 3, dtype=torch.uint8, device=dev)
        for _ in range(20):
            EV.eval_frames_u8(im, ds, gt, gd, lut, buf)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            EV.eval_frames_u8(im, ds, gt, gd, lut, buf)
        e1.record()
        torch.cuda.synchronize()
        us = 1e3 * e0.elapsed_time(e1) / reps
        out["%dx%d" % (w, h)] = dict(us=round(us, 2), gb_per_s=round(BYTES_PER_PIXEL * w * h / (us * 1e3), 1))
    return out


def time_encode(px, d):
    from PIL import Image
    from splatam_b200 import evaluate as EV
    out = {}
    for level in (EV.PNG_COMPRESS_LEVEL, 6):
        ms = []
        for k in range(4):
            for rep in range(3):
                t0 = time.perf_counter()
                Image.fromarray(px[k]).save(os.path.join(d, "enc_%d_%d.png" % (k, rep)), compress_level=level)
                ms.append(1e3 * (time.perf_counter() - t0))
        out["level_%d" % level] = round(statistics.median(ms), 2)
    return out


def time_evaluate(frames_n, d):
    import splatam_b200 as S
    from splatam_b200 import evaluate as EV, slam
    dev = torch.device("cuda:0")
    sc = scenes.view_filling(margin=100)
    cam = sc.settings(S.GaussianRasterizationSettings, dev)
    gt = dict(means3D=sc.means3D, rgb_colors=sc.colors, unnorm_rotations=sc.rotations,
              logit_opacities=torch.logit(sc.opacities.reshape(-1, 1)), log_scales=torch.log(sc.scales[:, :1]))
    gt = {k: v.to(dev).contiguous() for k, v in gt.items()}
    rots, trans = slam.look_trajectory(frames_n, dev, step=(0.002, -0.001, 0.001), rot_step=(0.0005, -0.0004, 0.0003))
    frames = [slam.render_frame(gt, rots, trans, t, cam) for t in range(frames_n)]
    params = dict(gt, cam_unnorm_rots=rots, cam_trans=trans)

    def run(save, tag):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        res = EV.evaluate(params, frames, cam, 0.5, 60, True, out_dir=os.path.join(d, tag), save_frames=save)
        torch.cuda.synchronize()
        return len(res["frame_ids"]) / (time.perf_counter() - t0), res
    run(False, "warm")
    run(True, "warm_frames")
    out = {}
    rate, ref = run(False, "plain")
    out["no_save_frames"] = round(rate, 2)
    default = EV.FRAME_WRITER_THREADS
    try:
        for n in (1, 2, 4, 8):
            EV.FRAME_WRITER_THREADS = n
            rate, res = run(True, "threads%d" % n)
            assert res["psnr_per_frame"].tolist() == ref["psnr_per_frame"].tolist()
            out["save_frames_%d_threads" % n] = round(rate, 2)
    finally:
        EV.FRAME_WRITER_THREADS = default
    px = EV.eval_frames_u8(*(t for t in _frame_inputs(params, frames[0], cam))).cpu().numpy()
    return out, px, sc.P


def _frame_inputs(params, fr, cam):
    from splatam_b200 import mapping as M
    with torch.no_grad():
        im, ds, _, _ = M._render_pair(params, dict(fr, cam=cam), M.default_render, True, False)
    return im, ds, fr["im"], fr["depth"]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=100)
    ap.add_argument("--reps", type=int, default=200)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_eval_frames.py needs a CUDA device")
    gpu = gpu_info()
    print("GPU:", gpu, "| host CPUs:", os.cpu_count())
    kernel = time_kernel(a.reps)
    with tempfile.TemporaryDirectory() as d:
        rates, px, P = time_evaluate(a.frames, d)
        encode = time_encode(px, d)
    print(json.dumps(dict(gpu=gpu, host_cpus=os.cpu_count(), kernel_us=kernel, png_encode_ms=encode,
                          evaluate_frames_per_s=rates, frames=a.frames, gaussians=P, width=1200, height=680)))


if __name__ == "__main__":
    main()
