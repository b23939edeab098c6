#!/usr/bin/env python
"""Builds a navigation map from a finished SplaTAM run record: the map's depth, fused into a TSDF volume as
extract_mesh.py fuses it, labelled free / occupied / unknown, and an exact Euclidean signed distance field over it, on
the GPU (splatam_b200/navmap.py).  Writes the map as one npz (formats.save_nav_map; NavMap.load reads it) and prints
one JSON line: dims, voxels, frames, the free / occupied / unknown counts, the clearance at the record's camera
centres, the device times and the wall time.

  python tools/nav_map.py --record runs/room0/params.npz --out runs/room0/navmap.npz --voxel 0.05

--unknown obstacle (the default) treats unobserved space as an obstacle, the conservative choice for planning;
--unknown free measures clearance to observed surfaces only (the labels still mark the unknown samples).  --occ-dist:
samples with T * trunc <= this are occupied (default half a voxel).  Every fusion flag of extract_mesh.py applies,
--source input with its dataset flags included.  One GPU."""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import numpy as np  # noqa: E402
import torch  # noqa: E402
import extract_mesh  # noqa: E402


def parse_args(argv=None):
    """This tool's own flags, then extract_mesh.parse_args (and its checks) on the rest."""
    ap = argparse.ArgumentParser(allow_abbrev=False, add_help=False)
    ap.add_argument("--unknown", default="obstacle", choices=("obstacle", "free"),
                    help="whether unobserved space counts as an obstacle")
    ap.add_argument("--occ-dist", type=float, default=None, help="occupied where T * trunc <= this (default voxel/2)")
    own, rest = ap.parse_known_args(argv)
    if own.occ_dist is not None and not np.isfinite(own.occ_dist):
        ap.error("--occ-dist must be finite")
    a = extract_mesh.parse_args(rest)
    a.unknown, a.occ_dist = own.unknown, own.occ_dist
    return a


def main(argv=None):
    a = parse_args(argv)
    from splatam_b200 import navmap
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    seq = frames = None
    if a.source == "input":
        seq, frames = extract_mesh.open_input(a, a.record, dev)
    t0 = time.perf_counter()
    try:
        nm, info = navmap.nav_record(
            a.record, a.voxel, every=a.every, sil_thres=a.sil_thres, depth_max=a.depth_max, bounds=a.bounds,
            batch=a.batch, trunc=a.trunc, min_weight=a.min_weight, occ_dist=a.occ_dist,
            unknown_is_obstacle=a.unknown == "obstacle", device=dev, source=frames)
        counts = nm.counts()
        nm.save(a.out)
    finally:
        if seq is not None:
            seq.close()
    wall = time.perf_counter() - t0
    c = np.asarray(info["clearance"], np.float64)
    line = dict(record=a.record, out=a.out, source=a.source, unknown_as=a.unknown, voxel=info["voxel_size"],
                trunc=info["trunc"], occ_dist=float(nm.occ_dist), dims=list(info["dims"]), voxels=info["voxels"],
                frames=info["frames"], **counts,
                clearance_min=float(c.min()) if len(c) else None,
                clearance_median=float(np.median(c)) if len(c) else None,
                render_ms=info["render_ms"], integrate_ms=info["integrate_ms"], labels_ms=info["labels_ms"],
                esdf_ms=info["esdf_ms"], wall_s=wall)
    print(json.dumps(line))
    return line


if __name__ == "__main__":
    main()
