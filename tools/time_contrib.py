"""Measures map compaction (splatam_b200.contrib) on one GPU, and prints the card's name and power limit first.  One
JSON line per measurement:

(a) stats_pass: device time of one blend-statistics pass (sb_blend_stats) against one blend_forward of the same render,
    on bench.py's flagship scene (scenes.config3: 1M Gaussians, 1200x680), CUDA events over `--reps` launches each;
(b) compact_record: wall time of contrib.compact_record on a 2,000-view record of a 1M-Gaussian view-filling map
    (`--views`), statistics and compaction apart;
(c) slam: SplaTAM and SplaTAM-S through tools/run_slam_dataset.py --out on the `--frames`-frame synthetic Replica-layout
    sequence (scenes.write_replica_sequence); then, for the lossless rule and each `--min-weights` value, the fraction
    of Gaussians removed and tools/eval_record.py's PSNR against the ground-truth frames on the compacted record, next
    to the original record's.

Run:  python tools/time_contrib.py [--frames 40] [--views 2000] [--min-weights 0.01 0.05 0.2]"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import scenes  # noqa: E402
from gpu_info import gpu_info  # noqa: E402


def stats_pass(dev, reps):
    import ctypes
    import splatam_b200 as S
    from splatam_b200 import _lib, contrib
    from splatam_b200.rasterizer import forward_states
    sc = scenes.config3()
    rs = sc.settings(S.GaussianRasterizationSettings, dev)
    inp = sc.inputs(dev)
    with torch.no_grad(), forward_states() as states:
        color, _, depth = S.GaussianRasterizer(rs)(**inp)
    st = states[-1]
    acc = contrib.BlendStats(sc.P, dev)
    e = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
    stats_ms = []
    for _ in range(reps):
        e[0].record()
        _lib.call("sb_forward_render", ctypes.byref(st.settings.c), sc.P, st.num_rendered, inp["colors_precomp"], None,
                  st.geom, st.geom.numel(), st.binning, st.binning.numel(), st.image, st.image.numel(), color, None,
                  depth, device=dev)
        e[1].record()
        acc.pixels = 0
        acc.add(st)
        e[2].record()
        torch.cuda.synchronize(dev)
        stats_ms.append(e[1].elapsed_time(e[2]))
    # blend_forward alone: the stage profiler brackets each stage of the render above
    buf_ms, buf_n = (ctypes.c_float * 10)(), (ctypes.c_int * 10)()
    _lib.load().sb_profile_begin()
    for _ in range(reps):
        _lib.call("sb_forward_render", ctypes.byref(st.settings.c), sc.P, st.num_rendered, inp["colors_precomp"], None,
                  st.geom, st.geom.numel(), st.binning, st.binning.numel(), st.image, st.image.numel(), color, None,
                  depth, device=dev)
    _lib.load().sb_profile_end(buf_ms, buf_n)
    fwd = buf_ms[6] / max(buf_n[6], 1)
    print(json.dumps(dict(part="stats_pass", gaussians=sc.P, width=sc.w, height=sc.h, num_rendered=st.num_rendered,
                          blend_forward_ms=fwd, stats_ms_median=float(np.median(stats_ms)),
                          stats_over_forward=float(np.median(stats_ms)) / fwd)), flush=True)


def compact_timing(dev, views, base):
    from splatam_b200 import formats, slam
    sc = scenes.view_filling(P=1_000_000)
    r40, t40 = slam.look_trajectory(40, "cpu")             # the views cycle through 40 poses that keep the map in view
    idx = torch.arange(views) % 40
    rots, trans = r40[..., idx].contiguous(), t40[..., idx].contiguous()
    K = np.array([[sc.fx, 0, sc.cx], [0, sc.fy, sc.cy], [0, 0, 1]], np.float32)
    gauss = sc.splatam_params(opacity_clamp=(1e-4, 1 - 1e-4))
    path = formats.save_run_record(os.path.join(base, "big"), gauss, rots, trans, torch.zeros(sc.P), K, np.eye(4),
                                   sc.w, sc.h, [np.eye(4, dtype=np.float32)] * views, list(range(views)))
    out = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "compact_record.py"), "--record", path, "--out",
                          os.path.join(base, "big_compact.npz")], capture_output=True, text=True)
    if out.returncode != 0:
        print(json.dumps(dict(part="compact_record", error=out.stderr[-2000:])), flush=True)
        return
    r = json.loads(out.stdout.strip().splitlines()[-1])
    print(json.dumps(dict(part="compact_record", **r)), flush=True)


def _tool(name, *args):
    out = subprocess.run([sys.executable, os.path.join(ROOT, "tools", name)] + [str(a) for a in args],
                         capture_output=True, text=True)
    if out.returncode != 0:
        raise RuntimeError("%s failed: %s" % (name, out.stderr[-2000:]))
    return json.loads(out.stdout.strip().splitlines()[-1])


def slam_fractions(dev, frames, min_weights, base):
    scenes.write_replica_sequence(os.path.join(base, "room0"), frames, dev)
    torch.cuda.empty_cache()
    data = ["--dataset", "replica", "--basedir", base, "--sequence", "room0"]
    for variant in ("splatam", "splatam_s"):
        run_dir = os.path.join(base, "run_" + variant)
        try:
            _tool("run_slam_dataset.py", *data, "--variant", variant, "--out", run_dir)
            rec = os.path.join(run_dir, "params.npz")
            orig = _tool("eval_record.py", *data, "--record", rec, "--no-frames", "--out", os.path.join(run_dir, "e0"))
            for w in [0.0] + list(min_weights):
                dst = os.path.join(run_dir, "compact_%g.npz" % w)
                c = _tool("compact_record.py", "--record", rec, "--out", dst, "--min-weight", w)
                e = _tool("eval_record.py", *data, "--record", dst, "--no-frames", "--out",
                          os.path.join(run_dir, "e_%g" % w))
                print(json.dumps(dict(part="slam", variant=variant, frames=frames, min_weight=w,
                                      gaussians_before=c["gaussians_before"], gaussians_after=c["gaussians_after"],
                                      removed_fraction=c["removed_fraction"], views=c["views"],
                                      psnr_gt_original_db=orig["psnr_db"], psnr_gt_compacted_db=e["psnr_db"],
                                      depth_l1_gt_original_m=orig["depth_l1_m"], depth_l1_gt_compacted_m=e["depth_l1_m"],
                                      psnr_vs_original_db=c.get("psnr_db"), stats_s=c["stats_s"])), flush=True)
        except RuntimeError as err:
            print(json.dumps(dict(part="slam", variant=variant, error=str(err))), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--views", type=int, default=2000)
    ap.add_argument("--frames", type=int, default=40)
    ap.add_argument("--min-weights", type=float, nargs="*", default=[0.01, 0.05, 0.2])
    ap.add_argument("--skip-slam", action="store_true")
    a = ap.parse_args()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    print(json.dumps(dict(part="card", gpu=gpu_info())), flush=True)
    stats_pass(dev, a.reps)
    torch.cuda.empty_cache()
    with tempfile.TemporaryDirectory() as base:
        compact_timing(dev, a.views, base)
        torch.cuda.empty_cache()
        if not a.skip_slam:
            slam_fractions(dev, a.frames, a.min_weights, base)


if __name__ == "__main__":
    main()
