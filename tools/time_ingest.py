#!/usr/bin/env python
"""Times frame loading on one GPU over a synthetic 1200x680 Replica-layout sequence (scenes.write_replica_sequence:
JPEG colour, 16-bit PNG depth at scale 6553.5) written to a temporary directory, or to --dir, where it is kept (for
tools/run_slam_dataset.py --dataset replica --basedir <dir> --sequence room0).  Prints the GPU name and power limit of
the run and one JSON line, per frame:
  reference_sync_ms     the reference loader's path: Pillow decode, float64 arrays, cv2.resize (INTER_LINEAR colour,
                        INTER_NEAREST depth), depth / png_depth_scale, torch.from_numpy(...).to(cuda).float() from
                        pageable memory (float64 colour and depth: 32 B per pixel), permute(2, 0, 1) / 255 (R/datasets/gradslam_datasets/basedataset.py:224-341);
                        synchronised
  reader_sync_ms        datasets.RGBDSequence with prefetch=0 (decode, uint8 / uint16 upload, ingest kernel);
                        synchronised
  track_only_ms         40 track_frame iterations on frames already in memory
  track_prefetch_ms     the same 40 iterations with each frame read from disk by RGBDSequence(prefetch=2) first
  exposed_load_ms       track_prefetch_ms - track_only_ms: what loading adds to a tracked frame
  kernel_us             sb_ingest_rgbd on one 1200x680 frame, CUDA events over --reps launches
Run:  python tools/time_ingest.py [--frames 40] [--reps 200] [--dir DIR]"""
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

import scenes  # noqa: E402
from gpu_info import gpu_info  # noqa: E402


def reference_frame(files, t, dev):
    """One frame the way the reference's loader and splatam.py produce it."""
    import cv2
    from PIL import Image
    H, W = files.height, files.width
    color = np.asarray(np.asarray(Image.open(files.color_paths[t])), dtype=float)
    color = cv2.resize(color, (W, H), interpolation=cv2.INTER_LINEAR)
    depth = np.asarray(np.asarray(Image.open(files.depth_paths[t])), dtype=np.int64)
    depth = np.expand_dims(cv2.resize(depth.astype(float), (W, H), interpolation=cv2.INTER_NEAREST), -1)
    depth = depth / files.png_depth_scale
    color = torch.from_numpy(color).to(dev).type(torch.float)
    depth = torch.from_numpy(depth).to(dev).type(torch.float)
    return color.permute(2, 0, 1) / 255, depth.permute(2, 0, 1)


def per_frame_ms(fn, n, dev):
    torch.cuda.synchronize(dev)
    t0 = time.perf_counter()
    for t in range(n):
        fn(t)
    torch.cuda.synchronize(dev)
    return 1e3 * (time.perf_counter() - t0) / n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=40)
    ap.add_argument("--reps", type=int, default=200)
    ap.add_argument("--iters", type=int, default=40, help="track_frame iterations per frame in the prefetch timing")
    ap.add_argument("--dir", default=None, help="write the sequence under DIR/room0 and keep it")
    a = ap.parse_args()
    from splatam_b200 import datasets, mapping as M, slam
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    info = gpu_info()
    print("gpu:", info)
    tmp = None if a.dir else tempfile.TemporaryDirectory()
    base = a.dir or tmp.name
    try:
        scenes.write_replica_sequence(os.path.join(base, "room0"), a.frames, dev)
        files = datasets.SequenceFiles("replica", base, "room0")
        n = len(files)
        warm = 3
        # (a) the reference's synchronous path
        for t in range(warm):
            reference_frame(files, t, dev)
        ref_ms = per_frame_ms(lambda t: reference_frame(files, t, dev), n, dev)
        # (b) this reader, synchronous
        sync_seq = datasets.RGBDSequence("replica", base, "room0", device=dev, prefetch=0, cache=1)
        for t in range(warm):
            sync_seq[t]
        reader_ms = per_frame_ms(lambda t: sync_seq[t], n, dev)
        # (c) prefetching reader while the GPU tracks every frame for a fixed number of iterations
        with datasets.RGBDSequence("replica", base, "room0", device=dev, prefetch=0) as seq0:
            held = [seq0[t] for t in range(n)]
        init, _ = slam.initialize_map(held[0], seq0.intrinsics.cpu())
        rots = torch.zeros(1, 4, n, device=dev)
        rots[:, 0] = 1.0
        trans = torch.zeros(1, 3, n, device=dev)
        params = dict({k: v.detach() for k, v in init.items()}, cam_unnorm_rots=rots, cam_trans=trans)

        def track(fr):
            M.track_frame(params, fr, num_iters=a.iters)
        for t in range(warm):
            track(dict(held[t], cam=seq0.cam))
        track_ms = per_frame_ms(lambda t: track(dict(held[warm + t], cam=seq0.cam)), n - warm, dev)
        del held
        with datasets.RGBDSequence("replica", base, "room0", device=dev, prefetch=2) as seq:
            for t in range(warm):
                track(seq[t])
            seq.load_wait_s = 0.0
            both_ms = per_frame_ms(lambda t: track(seq[warm + t]), n - warm, dev)
            wait_ms = 1e3 * seq.load_wait_s / (n - warm)
        # (d) the kernel alone
        from PIL import Image
        rgb = torch.from_numpy(np.asarray(Image.open(files.color_paths[0])).copy()).to(dev)
        raw = torch.from_numpy(datasets.decode_depth(files.depth_paths[0])).to(dev)
        color, depth = datasets.ingest_rgbd(rgb, raw, files.height, files.width, files.png_depth_scale)
        for _ in range(20):
            datasets.ingest_rgbd(rgb, raw, files.height, files.width, files.png_depth_scale, color, depth)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(a.reps):
            datasets.ingest_rgbd(rgb, raw, files.height, files.width, files.png_depth_scale, color, depth)
        e1.record()
        torch.cuda.synchronize(dev)
        kernel_us = 1e3 * e0.elapsed_time(e1) / a.reps
    finally:
        if tmp is not None:
            tmp.cleanup()
    hw = files.height * files.width
    print(json.dumps(dict(
        gpu=info, frames=n, width=files.width, height=files.height, reference_sync_ms=ref_ms, reader_sync_ms=reader_ms,
        track_iters=a.iters, track_only_ms=track_ms, track_prefetch_ms=both_ms, exposed_load_ms=both_ms - track_ms,
        reader_wait_ms=wait_ms, kernel_us=kernel_us, kernel_bytes_per_pixel=(3 + 2 + 16),
        kernel_gb_per_s=(3 + 2 + 16) * hw / (kernel_us * 1e-6) / 1e9,
        upload_bytes_per_pixel=dict(reference=32, reader=5))))


if __name__ == "__main__":
    main()
