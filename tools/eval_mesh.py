#!/usr/bin/env python
"""Scores a reconstructed mesh against the scene's ground-truth mesh on the GPU (splatam_b200/mesh_eval.py): accuracy
and completion (mean distances, cm), precision, recall (the completion ratio: the share of ground-truth samples within
--threshold of the reconstruction) and F-score, from --samples area-weighted samples of each mesh.  Prints one JSON
line with those scores, the sample counts and the device time of culling, grid build and queries.

  python tools/extract_mesh.py --record runs/room0/params.npz --out runs/room0/mesh.ply
  python tools/eval_mesh.py --mesh runs/room0/mesh.ply --gt-mesh data/Replica/room0_mesh.ply \
      --dataset replica --basedir data/Replica --sequence room0

The dataset flags are run_slam_dataset.py's (--dataset, --basedir, --sequence, --config, --start, --end, --stride) and
should select the run's frames.  The ground-truth mesh is moved from the dataset's world frame into the map's frame
(datasets.SequenceFiles.world_to_map: the first selected camera is the map's origin), and only the ground-truth samples
that some --every-th selected frame observed, by its depth at the native image size and its ground-truth pose, are
kept.  --no-cull keeps every sample; with --no-cull and no dataset flags the two meshes are scored as they are, for a
ground truth that is already in the map's frame and culled.

--depth-views N also renders both meshes from N random views (mesh_eval.depth_l1: 500x500, fx = fy = 300, centres in
the box of the kept ground-truth samples) and adds depth_l1_cm, depth_l1_surface_cm, hole_ratio, depth_views_used,
depth_views_drawn and render_ms to the line; with culling only pixels whose ground-truth surface was observed count.
One GPU."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402
import torch  # noqa: E402


def parse_args(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--mesh", required=True, help="the reconstructed mesh (PLY), in the map's frame")
    ap.add_argument("--gt-mesh", required=True, help="the ground-truth mesh (PLY), in the dataset's world frame")
    ap.add_argument("--dataset", default=None, help="dataset name, as for run_slam_dataset.py")
    ap.add_argument("--basedir", default=None)
    ap.add_argument("--sequence", default=None)
    ap.add_argument("--config", default=None, help="data YAML (camera_params); default: the shipped camera")
    ap.add_argument("--start", type=int, default=0)
    ap.add_argument("--end", type=int, default=-1)
    ap.add_argument("--stride", type=int, default=1)
    ap.add_argument("--every", type=int, default=1, help="cull with every N-th selected frame")
    ap.add_argument("--samples", type=int, default=200_000, help="points sampled on each mesh")
    ap.add_argument("--threshold", type=float, default=0.05, help="precision / recall distance (metres)")
    ap.add_argument("--occlusion-eps", type=float, default=0.03,
                    help="a sample is observed when its depth is at most the frame's depth plus this (metres)")
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--batch", type=int, default=8, help="frames per culling launch")
    ap.add_argument("--no-cull", action="store_true", help="keep every ground-truth sample")
    ap.add_argument("--depth-views", type=int, default=0,
                    help="also score depth L1 over this many accepted random views (0: off)")
    a = ap.parse_args(argv)
    for flag, path in (("--mesh", a.mesh), ("--gt-mesh", a.gt_mesh)):
        if not os.path.isfile(path):
            ap.error("%s %s: no such file" % (flag, path))
    core = [a.dataset, a.basedir, a.sequence]
    selection = [f for f, v, d in (("--config", a.config, None), ("--start", a.start, 0), ("--end", a.end, -1),
                                   ("--stride", a.stride, 1), ("--every", a.every, 1)) if v != d]
    if any(core) and not all(core):
        ap.error("--dataset, --basedir and --sequence go together")
    if not any(core):
        if not a.no_cull:
            ap.error("culling needs the sequence: pass --dataset, --basedir and --sequence, or --no-cull")
        if selection:
            ap.error("%s select frames: they need --dataset, --basedir and --sequence" % ", ".join(selection))
    if a.depth_views < 0:
        ap.error("--depth-views must be >= 0")
    if a.every < 1 or a.batch < 1 or a.samples < 1:
        ap.error("--every, --batch and --samples must be positive")
    if not (np.isfinite(a.threshold) and a.threshold > 0):
        ap.error("--threshold must be positive")
    if not (np.isfinite(a.occlusion_eps) and a.occlusion_eps >= 0):
        ap.error("--occlusion-eps must be >= 0")
    return a


def to_map(vertices, world_to_map):
    """vertices [V,3] of the world frame -> the map's frame, in float64, returned as float32."""
    M = np.asarray(world_to_map, np.float64)
    return (np.asarray(vertices, np.float64) @ M[:3, :3].T + M[:3, 3]).astype(np.float32)


def main(argv=None):
    a = parse_args(argv)
    from splatam_b200 import datasets, formats, mesh_eval
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    pv, _, pf = formats.load_mesh_ply(a.mesh)
    gv, _, gf = formats.load_mesh_ply(a.gt_mesh)
    seq = frames = K = None
    try:
        if a.dataset:
            cfg = datasets.load_config(a.config) if a.config else None
            seq = datasets.RGBDSequence(a.dataset, a.basedir, a.sequence, cfg, start=a.start, end=a.end,
                                        stride=a.stride, device=dev, prefetch=2 if a.every == 1 else 0)
            gv = to_map(gv, seq.files.world_to_map)
            if not a.no_cull:
                K = seq.intrinsics.cpu().numpy()
                frames = (seq[t] for t in range(0, len(seq), a.every))
        out = mesh_eval.evaluate_mesh((pv, pf), (gv, gf), frames, K, samples=a.samples, threshold=a.threshold,
                                      occlusion_eps=a.occlusion_eps, seed=a.seed, device=dev, batch=a.batch,
                                      depth_views=a.depth_views)
    finally:
        if seq is not None:
            seq.close()
    line = dict(mesh=a.mesh, gt_mesh=a.gt_mesh, culled=frames is not None,
                frames=0 if frames is None else len(range(0, len(seq), a.every)),
                accuracy_cm=100 * out["accuracy"], completion_cm=100 * out["completion"],
                precision=out["precision"], recall=out["recall"], fscore=out["fscore"], threshold_cm=100 * a.threshold,
                pred_samples=out["pred_samples"], gt_samples=out["gt_samples"],
                gt_samples_kept=out["gt_samples_kept"], cull_ms=out["cull_ms"], grid_ms=out["grid_ms"],
                query_ms=out["query_ms"])
    if a.depth_views:
        line.update(depth_l1_cm=100 * out["depth_l1"], depth_l1_surface_cm=100 * out["depth_l1_surface"],
                    hole_ratio=out["hole_ratio"], depth_views_used=out["depth_views_used"],
                    depth_views_drawn=out["depth_views_drawn"], render_ms=out["depth_render_ms"])
    print(json.dumps(line))
    return line


if __name__ == "__main__":
    main()
