"""Measures keyframe-pose refinement (ShardedMapper with non-zero camera rates, run_slam's `mapping_cam_lrs`) on one
GPU, and prints the card's name and power limit first:

(a) mapping keyframe-iterations/s on bench.py's mapping workload (1M-Gaussian view-filling map, 1200x680, eight
    keyframes), in graph mode and eagerly, refinement off and on, run alternately `--reps` times each;
(b) SplaTAM and SplaTAM-S through tools/run_slam_dataset.py on a synthetic Replica-layout sequence
    (scenes.write_replica_sequence, `--frames` frames) without refinement and with each `--cam-lrs` pair, run
    alternately: ATE, PSNR and wall time per frame.  One JSON line per run.

Run:  python tools/time_ba.py [--frames 40] [--reps 2] [--cam-lrs 0.0004 0.002 0.0001 0.0005]"""
import argparse
import json
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

CAM_LRS = dict(cam_unnorm_rots=0.0004, cam_trans=0.002)


def mapping_rate(dev, gauss, rots, trans, frames, refine, steps, warmup, graph=True):
    from splatam_b200 import mapping as M
    mapper = M.ShardedMapper(gauss, rots, trans, seed=11, fused=True, lrs=CAM_LRS if refine else None)
    if graph:
        mapper.enable_graph(frames)
    for _ in range(warmup):
        mapper.step(frames)
    torch.cuda.synchronize(dev)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        mapper.step(frames)
    e1.record()
    torch.cuda.synchronize(dev)
    _, overflow = mapper.check_capacity()
    assert not overflow and mapper.effective_steps()[1] == 0, "a step overflowed: the rate would be invalid"
    return 1e3 * steps / e0.elapsed_time(e1)


def profile_eager(dev, gauss, rots, trans, frames, steps=20):
    """Prints the CUDA ops that take the most device time over `steps` eager steps, refinement off, then on."""
    from torch.profiler import ProfilerActivity, profile
    from splatam_b200 import mapping as M
    for refine in (False, True):
        mapper = M.ShardedMapper(gauss, rots, trans, seed=11, fused=True, lrs=CAM_LRS if refine else None)
        for _ in range(5):
            mapper.step(frames)
        torch.cuda.synchronize(dev)
        with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
            for _ in range(steps):
                mapper.step(frames)
            torch.cuda.synchronize(dev)
        print("profile refine=%s (%d eager steps)" % (refine, steps), flush=True)
        print(prof.key_averages().table(sort_by="cuda_time_total", row_limit=14, max_name_column_width=60), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=40)
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--cam-lrs", type=float, nargs="+", default=[0.0004, 0.002, 0.0001, 0.0005],
                    help="camera-rate pairs ROT TRANS ... of part (b)")
    ap.add_argument("--variants", nargs="+", default=["splatam", "splatam_s"])
    ap.add_argument("--skip-rate", action="store_true")
    ap.add_argument("--skip-slam", action="store_true")
    ap.add_argument("--profile", action="store_true", help="torch.profiler's top CUDA ops of 20 eager steps, off / on")
    a = ap.parse_args()
    if len(a.cam_lrs) % 2:
        ap.error("--cam-lrs takes pairs")
    import splatam_b200 as S
    import bench
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    print("gpu:", gpu_info(), flush=True)
    if not a.skip_rate:
        _, gauss, rots, trans, frames = bench.mapping_problem(dev, S.GaussianRasterizationSettings, 1_000_000)
        for graph in (True, False):
            for rep in range(a.reps):
                for refine in (False, True):
                    r = mapping_rate(dev, gauss, rots, trans, frames, refine, a.steps, 10, graph)
                    print(json.dumps(dict(part="mapping_rate", graph=graph, rep=rep, refine=refine,
                                          keyframe_iters_per_s=r)), flush=True)
        if a.profile:
            profile_eager(dev, gauss, rots, trans, frames)
        del gauss, frames
        torch.cuda.empty_cache()
    if a.skip_slam:
        return
    pairs = [(0.0, 0.0)] + [(a.cam_lrs[i], a.cam_lrs[i + 1]) for i in range(0, len(a.cam_lrs), 2)]
    with tempfile.TemporaryDirectory() as base:
        scenes.write_replica_sequence(os.path.join(base, "room0"), a.frames, dev)
        torch.cuda.empty_cache()
        for variant in a.variants:
            for rot, tr in pairs:
                t0 = time.perf_counter()
                out = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "run_slam_dataset.py"), "--dataset",
                                      "replica", "--basedir", base, "--sequence", "room0", "--variant", variant,
                                      "--mapping-cam-lrs", str(rot), str(tr)], capture_output=True, text=True)
                if out.returncode != 0:
                    print(json.dumps(dict(part="slam", variant=variant, mapping_cam_lrs=[rot, tr],
                                          error=out.stderr[-2000:])), flush=True)
                    continue
                r = json.loads(out.stdout.strip().splitlines()[-1])
                print(json.dumps(dict(part="slam", variant=variant, mapping_cam_lrs=[rot, tr], ate_mm=1e3 * r["ate_m"],
                                      psnr_db=r["psnr_db"], wall_s_per_frame=r["wall_s"] / r["frames"],
                                      mapping_ms_per_frame=1e3 * r["mapping_s"] / r["frames"],
                                      tracking_ms_per_frame=1e3 * r["tracking_s"] / r["frames"],
                                      gaussians=r["gaussians"], process_s=time.perf_counter() - t0)), flush=True)


if __name__ == "__main__":
    main()
