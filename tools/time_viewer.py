#!/usr/bin/env python
"""Times the headless viewer (splatam_b200/viewer.py, csrc/viewer.cu) on one GPU at user sizes: a seeded synthetic
record of --gaussians Gaussians (default 1M) with a non-decreasing timestep over --frames timesteps (default 2000),
viewed at 600x340 with view_scale 2 (a 1200x680 frame).  Prints the GPU name and power limit of the run and one JSON
line:
  kernel_us        per call, CUDA events over --reps calls after warm-up: sb_viewer_points over all centres,
                   sb_viewer_compose in colour and depth mode, sb_viewer_lines over every frustum edge and trajectory
                   segment (the final view's 9T - 1 segments)
  render_ms        the viewer's colour render and silhouette render of the whole map, per call
  frames_per_s     online_frames end to end (colour and centres modes, frames kept on the device), and
                   render_record online with PNG writing, over --online-frames frames spread over the run; PNGs go to
                   a temporary directory
Run:  python tools/time_viewer.py [--gaussians 1000000] [--frames 2000] [--reps 200] [--online-frames 100]"""
import argparse
import json
import os
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import numpy as np  # noqa: E402
import torch  # noqa: E402
from gpu_info import gpu_info  # noqa: E402


def synthetic_record(path, P, T, seed=0):
    """A room-sized map seen from a camera walking along z: Gaussians spread in a 4 x 3 x (2 + T/100) m box, each
    with the timestep of the first frame that is near it (sorted, so non-decreasing), isotropic log-scales around
    1 cm, and a smooth trajectory."""
    from splatam_b200 import formats
    g = np.random.default_rng(seed)
    depth = 2.0 + T / 100.0
    means = np.c_[g.uniform(-2, 2, P), g.uniform(-1.5, 1.5, P), g.uniform(0.5, depth + 2, P)].astype(np.float32)
    ts = np.clip(np.floor((means[:, 2] - 0.5) / (depth + 1.5) * T), 0, T - 1).astype(np.float32)
    order = np.argsort(ts, kind="stable")
    means, ts = means[order], ts[order]
    gauss = dict(means3D=means, rgb_colors=g.uniform(0, 1, (P, 3)).astype(np.float32),
                 unnorm_rotations=g.normal(size=(P, 4)).astype(np.float32),
                 logit_opacities=g.normal(1.0, 1.0, (P, 1)).astype(np.float32),
                 log_scales=np.log(g.uniform(0.005, 0.02, (P, 1))).astype(np.float32))
    t = np.arange(T)
    rots = np.zeros((1, 4, T), np.float32)
    rots[0, 0] = 1.0
    rots[0, 2] = 0.05 * np.sin(t / 50.0)
    trans = np.zeros((1, 3, T), np.float32)
    trans[0, 0] = 0.2 * np.sin(t / 80.0)
    trans[0, 2] = -t / 100.0                       # w2c translation: the camera moves to +z
    K = np.array([[600.0, 0, 599.5], [0, 600.0, 339.5], [0, 0, 1]], np.float32)
    return formats.save_run_record(path, gauss, rots, trans, ts, K, np.eye(4), 1200, 680, [np.eye(4)] * T, [0])


def events_us(fn, reps):
    for _ in range(3):
        fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) * 1e3 / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gaussians", type=int, default=1_000_000)
    ap.add_argument("--frames", type=int, default=2000)
    ap.add_argument("--reps", type=int, default=200)
    ap.add_argument("--online-frames", type=int, default=100)
    a = ap.parse_args()
    from splatam_b200 import viewer as V
    dev = torch.device("cuda:0")
    gpu = gpu_info()
    print(gpu, flush=True)
    out = dict(gpu=gpu, gaussians=a.gaussians, timesteps=a.frames)
    with tempfile.TemporaryDirectory() as tmp:
        rec = V.load_record(synthetic_record(tmp, a.gaussians, a.frames), dev)
        assert rec.monotone
        cfg = V.ViewerConfig()
        views = V._Views(rec, cfg, online=False)
        frame = torch.empty(views.H, views.W, 3, dtype=torch.uint8, device=dev)
        im, depth, _ = V.render_view(rec, views, 0, None)
        sil_views = V._Views(rec, V.ViewerConfig(show_sil=True), online=False)
        k = {}
        k["points"] = events_us(lambda: V.draw_points(rec.means3D, rec.colors, None, 0.0, views.w2c[0], views.k_out,
                                                      views.W, views.H, 2, cfg.viz_near, cfg.viz_far, views.keys,
                                                      frame, views.zbuf), a.reps)
        k["compose_color"] = events_us(lambda: V.compose(im, depth, None, 0, 2, views.lut, frame, views.zbuf,
                                                         views.vmax), a.reps)
        k["compose_depth"] = events_us(lambda: V.compose(im, depth, None, 1, 2, views.lut, frame, views.zbuf,
                                                         views.vmax), a.reps)
        k["lines"] = events_us(lambda: V.draw_lines(views.segs, views.seg_cols, views.w2c[0], views.k_out, views.W,
                                                    views.H, cfg.viz_near, views.zbuf, views.keys, frame), a.reps)
        out["kernel_us"] = {n: round(v, 1) for n, v in k.items()}
        out["line_segments"] = int(views.segs.shape[0])
        out["points_GBps"] = round((a.gaussians * 12 + views.H * views.W * (8 + 8 + 3 + 4)) / (k["points"] * 1e3), 1)
        nr = max(10, a.reps // 10)
        out["render_ms"] = dict(color=round(events_us(lambda: V.render_view(rec, views, 0, None), nr) / 1e3, 3),
                                color_and_sil=round(events_us(lambda: V.render_view(rec, sil_views, 0, None), nr)
                                                    / 1e3, 3))
        every = max(1, a.frames // a.online_frames)
        fps = {}
        for mode in ("color", "centers"):
            c = V.ViewerConfig(render_mode=mode)
            for _ in V.online_frames(rec, c, every=a.frames):          # warm-up
                pass
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            n = sum(1 for _ in V.online_frames(rec, c, every=every))
            torch.cuda.synchronize()
            fps[mode] = round(n / (time.perf_counter() - t0), 2)
        d = os.path.join(tmp, "png")
        t0 = time.perf_counter()
        n = len(V.render_record(rec, cfg, d, "online", every=every))
        fps["color_png"] = round(n / (time.perf_counter() - t0), 2)
        out["frames_per_s"] = fps
        out["png_writer_threads"] = V.EV.FRAME_WRITER_THREADS
        out["online_frames"] = n
    print(json.dumps(out))


if __name__ == "__main__":
    main()
