#!/usr/bin/env python
"""Measures loop closure (splatam_b200/loop.py, csrc/loop.cu) on one GPU, and prints the card's name and power limit
first; one JSON line per measurement:

(a) sb_deform_gaussians' device time at `--gaussians` (CUDA events over `--launches` launches, every Gaussian moved)
    and its share of the HBM bound: 60 B per Gaussian (12 + 16 + 4 read, 28 written) over 3.35 TB/s;
(b) one pose-graph solve (PoseGraph.solve: normal equations, Cholesky, update, to convergence) at `--keyframes` nodes
    with 1 and 10 loop edges (oracle/loop_numpy.random_graph), wall time with a device synchronisation;
(c) close_loop at the last keyframe of scenes.drifted_loop: with no keyframe old enough (an early return), with a
    candidate that is scored and measured by ICP but rejected (min_inlier_frac 1), and when the loop closes;
(d) with --runs: tools/run_slam_dataset.py --pose-init icp on the loop sequence (scenes.write_loop_sequence at the
    Replica camera, `--frames` frames, read from disk with Replica's shipped hyper-parameters), without and with
    --loop-closure, alternated, `--repeats` each: its JSON line (ATE, PSNR, wall and loop-closure seconds, loops).

Run:  python tools/time_loop_closure.py [--gaussians 1000000 3000000] [--keyframes 100 400]
      python tools/time_loop_closure.py --runs --skip-parts [--frames 81] [--repeats 2]"""
import argparse
import json
import math
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import scenes  # noqa: E402
from gpu_info import gpu_info  # noqa: E402
from oracle import loop_numpy as O  # noqa: E402

HBM_BYTES_PER_S = 3.35e12          # H100 SXM data sheet


def deform_time(dev, P, launches):
    from splatam_b200 import loop
    g = torch.Generator().manual_seed(1)
    means = (torch.randn(P, 3, generator=g)).to(dev)
    rots = torch.randn(P, 4, generator=g).to(dev)
    T = 400
    ts = torch.randint(1, T, (P,), generator=g).float().to(dev)
    table = torch.zeros(T, 12, device=dev)
    table[:, 0] = table[:, 5] = table[:, 10] = math.cos(0.01)
    table[:, 2], table[:, 8], table[:, 3] = math.sin(0.01), -math.sin(0.01), 0.001
    flag = torch.ones(1, dtype=torch.int32, device=dev)
    for _ in range(3):
        loop.deform_gaussians(means, rots, ts, table, flag)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(launches):
        loop.deform_gaussians(means, rots, ts, table, flag)
    e1.record()
    torch.cuda.synchronize(dev)
    us = 1e3 * e0.elapsed_time(e1) / launches
    bound_us = 1e6 * 60 * P / HBM_BYTES_PER_S
    return dict(measurement="deform", gaussians=P, us=us, hbm_bound_us=bound_us, share_of_hbm_bound=bound_us / us)


def solve_time(dev, N, loops, reps=3):
    from splatam_b200 import loop
    est, edges, Z = O.random_graph(N, loops, N + loops)
    g = loop.PoseGraph(0)
    for (i, j), z in zip(edges[:N - 1], Z[:N - 1]):
        g.add_odometry(i, j, torch.from_numpy(z).to(dev))
    for (i, j), z in zip(edges[N - 1:], Z[N - 1:]):
        g.add_loop(i, j, torch.from_numpy(z).to(dev))
    cfg = loop.config({})
    w2c = torch.from_numpy(np.stack(est)).to(dev)
    g.solve(w2c, N, N - 1, cfg)
    ts = []
    for _ in range(reps):
        torch.cuda.synchronize(dev)
        t0 = time.perf_counter()
        sol = g.solve(w2c, N, N - 1, cfg)
        torch.cuda.synchronize(dev)
        ts.append(time.perf_counter() - t0)
    return dict(measurement="solve", keyframes=N, loops=loops, ms=1e3 * min(ts), steps=sol["steps"],
                accepted=bool(int(sol["flag"])))


def close_loop_cost(dev):
    from splatam_b200 import loop
    st = scenes.drifted_loop(dev)
    t = st["T"] - 1
    c = scenes.LOOP_CAM
    K = torch.tensor([[c["fx"], 0.0, c["cx"]], [0.0, c["fy"], c["cy"]], [0.0, 0.0, 1.0]])
    out = []
    for label, kw in (("no keyframe old enough (early return)", dict(min_gap=1000)),
                      ("candidate scored, measured by ICP and rejected", dict(min_inlier_frac=1.0)),
                      ("loop closes", {})):
        ts = []
        for _ in range(3):
            mapper, kfs, graph, rots, trans = scenes.drifted_loop_at(st, t)
            mapper.cam = dict(cam_unnorm_rots=rots, cam_trans=trans)
            cfg = loop.config(kw)
            torch.cuda.synchronize(dev)
            t0 = time.perf_counter()
            recs, j = loop.close_loop(t, st["frames"][t], kfs, rots, trans, graph, K, cfg, mapper=mapper)
            torch.cuda.synchronize(dev)
            ts.append(time.perf_counter() - t0)
        out.append(dict(measurement="close_loop", case=label, keyframes=len(kfs),
                        gaussians=int(mapper.timestep.numel()), ms=1e3 * min(ts), closed=j is not None, records=recs))
    return out


def whole_runs(T, repeats, base):
    """tools/run_slam_dataset.py's JSON line per run, the two settings alternated."""
    import subprocess
    dev = torch.device("cuda", 0)
    scenes.write_loop_sequence(os.path.join(base, "loop"), T, dev, cam=scenes.REPLICA)
    out = []
    for r in range(repeats):
        for lc in (False, True):
            cmd = [sys.executable, os.path.join(ROOT, "tools", "run_slam_dataset.py"), "--dataset", "replica",
                   "--basedir", base, "--sequence", "loop", "--pose-init", "icp"] + (["--loop-closure"] if lc else [])
            res = json.loads(subprocess.run(cmd, check=True, capture_output=True, text=True).stdout.strip()
                             .splitlines()[-1])
            res.pop("hyper", None)
            out.append(dict(res, measurement="run", loop_closure=lc, repeat=r,
                            ms_per_frame=1e3 * res["wall_s"] / res["frames"]))
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--gaussians", type=int, nargs="+", default=[1_000_000, 3_000_000])
    ap.add_argument("--keyframes", type=int, nargs="+", default=[100, 400])
    ap.add_argument("--launches", type=int, default=50)
    ap.add_argument("--skip-parts", action="store_true", help="skip (a)-(c)")
    ap.add_argument("--runs", action="store_true", help="(d): whole runs on the loop sequence")
    ap.add_argument("--frames", type=int, default=81)
    ap.add_argument("--repeats", type=int, default=2)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_loop_closure.py measures on a GPU; none is visible")
    dev = torch.device("cuda", 0)
    print(json.dumps(dict(gpu=gpu_info())), flush=True)
    if not a.skip_parts:
        for P in a.gaussians:
            print(json.dumps(deform_time(dev, P, a.launches)), flush=True)
        for N in a.keyframes:
            for loops in (1, 10):
                print(json.dumps(solve_time(dev, N, loops)), flush=True)
        for r in close_loop_cost(dev):
            print(json.dumps(r), flush=True)
    if a.runs:
        import tempfile
        with tempfile.TemporaryDirectory() as base:
            for r in whole_runs(a.frames, a.repeats, base):
                print(json.dumps(r), flush=True)


if __name__ == "__main__":
    main()
