#!/usr/bin/env python
"""Speed of the offline all-frame loop (splatam_b200.offline.optimize_map, eager, fused path) on one GPU, and of the
densification statistic it runs every iteration: sb_densify_accumulate against the torch statement it replaces
(`accum[seen] += norm(g[seen, :2]); denom[seen] += 1`), in the same process.

The map is synthetic (scenes.config3: isotropic Gaussians in front of the camera), `--gaussians` of them (default
873,000, the map size of a Replica run), at 1200x680 with Replica's camera and at 876x584 with a camera of the same
field of view.  Four target frames are rendered from it along slam.look_trajectory, and the loop starts from a
perturbed copy with the shipped learning rates and densify schedule.  The timed iterations lie before the schedule's
first densify event (iteration 500), so they measure the per-iteration cost (render, loss, backward, statistic, Adam),
not the map edits every 100 iterations.  The GPU name and power limit are read (nvidia-smi query, read-only) in the same
call.  Prints one JSON line per image size and one for the statistic.

  python tools/time_offline.py --gaussians 873000 --iters 200"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

import scenes  # noqa: E402

SIZES = {"1200x680": scenes.REPLICA,
         "876x584": dict(w=876, h=584, fx=438.0, fy=438.0, cx=437.5, cy=291.5)}


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, check=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:          # the name still comes from torch
        return "%s, power limit unknown (%s)" % (torch.cuda.get_device_name(0), e)


def time_loop(P, cam, iters, warmup, dev):
    import splatam_b200 as S
    from splatam_b200 import mapping as M, offline, slam
    sc = scenes.config3(P=P, cam=cam)
    settings = sc.settings(S.GaussianRasterizationSettings, dev)
    gt = dict(means3D=sc.means3D, rgb_colors=sc.colors, unnorm_rotations=sc.rotations,
              logit_opacities=torch.logit(sc.opacities), log_scales=torch.log(sc.scales[:, :1]))
    gt = {k: v.to(dev).contiguous() for k, v in gt.items()}
    rots, trans = slam.look_trajectory(4, dev)
    frames = [slam.render_frame(gt, rots, trans, t, settings) for t in range(4)]
    train = [dict(fr, pose=M.camera_w2c(rots[..., t], trans[..., t])) for t, fr in enumerate(frames)]
    g = torch.Generator(device=dev).manual_seed(1)
    init = {k: v + 0.01 * torch.randn(v.shape, device=dev, generator=g) for k, v in gt.items()}
    mapper = M.ShardedMapper(init, rots, trans, lrs=offline.LRS, fused=True)
    radius = float(frames[0]["depth"].max()) / 2.0
    assert warmup + iters < offline.DENSIFY["start_after"]
    run = lambda n: offline.optimize_map(mapper, train, n, offline.MEANS3D_LR_FINAL, offline.DENSIFY, radius)
    run(warmup)
    torch.cuda.synchronize(dev)
    t0 = time.perf_counter()
    run(iters)
    torch.cuda.synchronize(dev)
    dt = time.perf_counter() - t0
    return dict(gaussians=P, width=cam["w"], height=cam["h"], iters=iters, iters_per_s=iters / dt,
                ms_per_iter=1e3 * dt / iters)


def time_statistic(P, reps, dev):
    from splatam_b200 import map_ops
    g = torch.Generator(device=dev).manual_seed(2)
    grad = 1e-3 * torch.randn(P, 3, device=dev, generator=g)
    seen = torch.rand(P, device=dev, generator=g) < 0.6
    accum, denom = torch.zeros(P, device=dev), torch.zeros(P, device=dev)

    def torch_statement():
        accum[seen] += torch.norm(grad[seen, :2], dim=-1)
        denom[seen] += 1

    def kernel():
        map_ops.densify_accumulate(grad, seen, accum, denom)
    out = dict(gaussians=P, seen_fraction=float(seen.float().mean()), reps=reps)
    for name, fn in (("torch", torch_statement), ("kernel", kernel), ("torch", torch_statement), ("kernel", kernel)):
        for _ in range(10):
            fn()
        torch.cuda.synchronize(dev)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0 = time.perf_counter()
        e0.record()
        for _ in range(reps):
            fn()
        e1.record()
        torch.cuda.synchronize(dev)
        host = time.perf_counter() - t0
        # second round of each overwrites the first: the first round also warms the allocator and the launch path
        out[name + "_us_per_call_events"] = 1e3 * e0.elapsed_time(e1) / reps
        out[name + "_us_per_call_host"] = 1e6 * host / reps
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gaussians", type=int, default=873_000)
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--stat-reps", type=int, default=500)
    a = ap.parse_args()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    gpu = gpu_info()
    for name, cam in SIZES.items():
        print(json.dumps(dict(what="offline loop, eager, fused", size=name, gpu=gpu,
                              **time_loop(a.gaussians, cam, a.iters, a.warmup, dev))), flush=True)
        torch.cuda.empty_cache()
    print(json.dumps(dict(what="densification statistic", gpu=gpu, **time_statistic(a.gaussians, a.stat_reps, dev))))


if __name__ == "__main__":
    main()
