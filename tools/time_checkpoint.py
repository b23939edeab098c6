#!/usr/bin/env python
"""Wall time of one SLAM checkpoint (formats.save_checkpoint of params{t}.npz, keyframe_time_indices{t}.npy and the
run_state{t}.npz sidecar, device-to-host copies included) at given map sizes, on one GPU.  The map is a random
isotropic one held by a ShardedMapper on cuda:0, with a 2000-frame camera track and 400 keyframe ids, as a Replica run
has them; files go to a temporary directory that is removed afterwards.  Prints one JSON line per size.

  python tools/time_checkpoint.py --gaussians 873000 1000000 3000000 --reps 5"""
import argparse
import json
import os
import shutil
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import torch  # noqa: E402
from gpu_info import gpu_info  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gaussians", type=int, nargs="+", default=[873_000, 1_000_000, 3_000_000])
    ap.add_argument("--frames", type=int, default=2000)
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    from splatam_b200 import formats, mapping as M, slam
    dev = torch.device("cuda", 0)
    g = torch.Generator(device=dev).manual_seed(0)
    name = gpu_info()
    for P in a.gaussians:
        gauss = dict(means3D=torch.randn(P, 3, device=dev, generator=g), rgb_colors=torch.rand(P, 3, device=dev, generator=g),
                     unnorm_rotations=torch.randn(P, 4, device=dev, generator=g),
                     logit_opacities=torch.randn(P, 1, device=dev, generator=g),
                     log_scales=torch.randn(P, 1, device=dev, generator=g) - 4.0)
        rots = torch.randn(1, 4, a.frames, device=dev, generator=g)
        trans = torch.randn(1, 3, a.frames, device=dev, generator=g)
        mapper = M.ShardedMapper(gauss, rots, trans, fused=True,
                                 timestep=torch.randint(0, a.frames, (P,), device=dev, generator=g))
        counts = list(range(P - a.frames, P))
        kti = list(range(0, a.frames, 5))
        tmp = tempfile.mkdtemp(prefix="sb_ckpt_")
        times, size = [], 0
        try:
            for r in range(a.reps + 1):                    # the first write warms the page cache and the allocator
                torch.cuda.synchronize(dev)
                t0 = time.perf_counter()
                paths = formats.save_checkpoint(tmp, r, dict(mapper.g.params, cam_unnorm_rots=rots, cam_trans=trans),
                                                kti, slam._run_state(mapper, counts))
                times.append(time.perf_counter() - t0)
                size = sum(os.path.getsize(p) for p in paths)
                for p in paths:
                    os.remove(p)
        finally:
            shutil.rmtree(tmp, ignore_errors=True)
        times = times[1:]
        print(json.dumps(dict(gaussians=P, frames=a.frames, bytes=size, write_s_min=min(times),
                              write_s_median=sorted(times)[len(times) // 2], write_s_max=max(times), reps=len(times),
                              gpu=name)))


if __name__ == "__main__":
    main()
