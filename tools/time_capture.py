#!/usr/bin/env python
"""Times the live-capture path on one GPU and prints one JSON line with the card's name and power limit:
* kernel time per 1920x1440 packet (256x192 depth) of each entry point, CUDA events over --launches launches:
  sb_ingest_capture at 720x960 plus 360x480 (the two launches of a frame), sb_capture_depth_u16 at 1920x1440;
* host time per packet of the reference's conversion (iphone_demo.py:218-243 and 177-182: four cv2.resize calls, the
  uint16 cast, pageable .cuda() uploads and the float / 255 on the device, synchronised) against capture.LiveCapture's
  (pinned upload, both ingest launches, synchronised), over the same packets;
* online frames/s of tools/run_iphone_demo.py on --frames synthetic packets with the shipped 60 / 60 iterations.

  python tools/time_capture.py --out /tmp/time_capture"""
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


def event_ms(fn, n):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(n):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=500)
    ap.add_argument("--packets", type=int, default=30)
    ap.add_argument("--frames", type=int, default=10)
    ap.add_argument("--out", default=None, help="directory for the online run's capture (default: a temporary one)")
    a = ap.parse_args()
    from splatam_b200 import capture as C
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    g = np.random.default_rng(0)
    rgb = g.integers(0, 256, (1440, 1920, 3), dtype=np.uint8)
    depth = g.uniform(0.2, 6.0, (192, 256)).astype(np.float32)
    dr, dd = torch.from_numpy(rgb).to(dev), torch.from_numpy(depth).to(dev)
    res = dict(gpu=gpu_info(), packet="1920x1440 rgb, 256x192 depth")
    res["ingest_capture_us"] = 1e3 * event_ms(lambda: (C.ingest_capture(dr, dd, 720, 960),
                                                      C.ingest_capture(dr, dd, 360, 480)), a.launches)
    res["capture_depth_u16_us"] = 1e3 * event_ms(lambda: C.capture_depth_u16(dd, 10.0, 1440, 1920), a.launches)

    frames = [C.CaptureFrame(id=t, timestamp=0.0, fl_x=1450.0, fl_y=1450.0, cx=959.5, cy=719.5,
                             transform_matrix=tuple(np.eye(4).reshape(-1)), width=1920, height=1440,
                             image=rgb.tobytes(), has_depth=True, depth_width=256, depth_height=192, depth_scale=10.0,
                             depth_image=depth.tobytes()) for t in range(a.packets)]
    try:
        import cv2
    except ImportError:
        cv2 = None
    if cv2 is not None:
        def reference_style(fr):
            image, d = fr.rgb(), fr.depth()
            q = cv2.resize((d * 65535 / float(10.0)).astype(np.uint16), (1920, 1440), interpolation=cv2.INTER_NEAREST)
            out = []
            for (H, W) in ((720, 960), (360, 480)):
                c = cv2.resize(image, (W, H), interpolation=cv2.INTER_LINEAR)
                dd_ = np.expand_dims(cv2.resize(d, (W, H), interpolation=cv2.INTER_NEAREST), -1)
                out.append((torch.from_numpy(c).cuda().float().permute(2, 0, 1) / 255,
                            torch.from_numpy(dd_).cuda().float().permute(2, 0, 1)))
            torch.cuda.synchronize()
            return q, out
        reference_style(frames[0])
        t0 = time.perf_counter()
        for fr in frames:
            reference_style(fr)
        res["reference_style_host_ms_per_packet"] = 1e3 * (time.perf_counter() - t0) / len(frames)
    else:
        res["reference_style_host_ms_per_packet"] = "not measured: cv2 is not installed"
    seq = C.LiveCapture(iter(frames), len(frames), device=dev)
    seq[0]
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for t in range(1, len(frames)):
        seq[t]
        torch.cuda.synchronize()
    res["live_capture_host_ms_per_packet"] = 1e3 * (time.perf_counter() - t0) / (len(frames) - 1)
    del seq

    import run_iphone_demo
    with tempfile.TemporaryDirectory() as tmp:
        out = os.path.join(a.out or tmp, "online")
        torch.manual_seed(0); np.random.seed(0)
        packets = list(C.synthetic_frames(a.frames, dev))
        r = run_iphone_demo.run(iter(packets), a.frames, out, device=dev)
    res.update(online_frames=a.frames, online_frames_per_s=r["frames_per_s"], online_wall_s=r["wall_s"],
               online_ate_m=r["ate_m"], online_tracking_s=r["tracking_s"], online_mapping_s=r["mapping_s"],
               online_note="packets rendered before the run; wall time covers ingest, SLAM and writing the capture")
    print(json.dumps(res))


if __name__ == "__main__":
    main()
