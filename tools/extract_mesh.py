#!/usr/bin/env python
"""Extracts a coloured triangle mesh from a finished SplaTAM run record: the map's depth and colour, rendered at every
--every-th estimated pose, fused into a TSDF volume and meshed by marching cubes on the GPU (splatam_b200/mesh.py).
Writes a binary PLY that MeshLab and Blender open and prints one JSON line: voxels, frames, V, F and the device time
of rendering, integration and extraction.

  python tools/extract_mesh.py --record runs/room0/params.npz --out runs/room0/mesh.ply --voxel 0.01

--source input fuses the sequence's own depth and colour at the record's poses instead of the renders: a baseline for
the map's mesh.  The dataset flags are run_slam_dataset.py's (--dataset, --basedir, --sequence, --config, --start,
--end, --stride, --frames) and must select the frames the run used: frame t is fused at the record's pose t, so the
selected frame count must equal the record's camera count (a ValueError otherwise).  The sequence is read at the
record's image size.  One GPU.

  python tools/extract_mesh.py --record runs/room0/params.npz --out runs/room0/mesh_input.ply --source input \
      --dataset replica --basedir data/Replica --sequence room0 --stride 2"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import torch  # noqa: E402


def parse_args(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--record", required=True, help="params.npz of a finished run")
    ap.add_argument("--out", required=True, help="the mesh PLY to write")
    ap.add_argument("--voxel", type=float, default=0.01, help="voxel size in metres")
    ap.add_argument("--trunc", type=float, default=None, help="truncation in metres (default 4 voxels)")
    ap.add_argument("--every", type=int, default=1, help="fuse every N-th pose")
    ap.add_argument("--sil-thres", type=float, default=0.99, help="fuse rendered depth where silhouette > this")
    ap.add_argument("--depth-max", type=float, default=None, help="ignore depth beyond this (metres)")
    ap.add_argument("--bounds", type=float, nargs=6, default=None, metavar=("X0", "Y0", "Z0", "X1", "Y1", "Z1"),
                    help="volume box (default: 0.1/99.9 %% quantiles of the Gaussian centres, padded by 2 trunc)")
    ap.add_argument("--batch", type=int, default=8, help="frames per integration launch")
    ap.add_argument("--min-weight", type=float, default=1.0, help="cells need this weight at every corner")
    ap.add_argument("--source", default="render", choices=("render", "input"))
    ap.add_argument("--dataset", default=None, help="--source input: dataset name, as for run_slam_dataset.py")
    ap.add_argument("--basedir", default=None)
    ap.add_argument("--sequence", default=None)
    ap.add_argument("--config", default=None, help="data YAML (camera_params); default: the shipped camera")
    ap.add_argument("--start", type=int, default=0)
    ap.add_argument("--end", type=int, default=-1)
    ap.add_argument("--stride", type=int, default=1)
    ap.add_argument("--frames", type=int, default=0, help="use only the first N selected frames (0: all)")
    a = ap.parse_args(argv)
    if not os.path.isfile(a.record):
        ap.error("--record %s: no such file" % a.record)
    if a.every < 1 or a.batch < 1:
        ap.error("--every and --batch must be positive")
    if a.source == "input" and not (a.dataset and a.basedir and a.sequence):
        ap.error("--source input needs --dataset, --basedir and --sequence")
    given = [f for f, v, d in (("--dataset", a.dataset, None), ("--basedir", a.basedir, None),
                               ("--sequence", a.sequence, None), ("--config", a.config, None), ("--start", a.start, 0),
                               ("--end", a.end, -1), ("--stride", a.stride, 1), ("--frames", a.frames, 0)) if v != d]
    if a.source == "render" and given:
        ap.error("%s select input frames: they need --source input" % ", ".join(given))
    if a.frames < 0:
        ap.error("--frames must be 0 (all) or positive")
    return a


def open_input(a, record, device):
    """--source input: the run's frames as run_slam_dataset.py selects them -- datasets.RGBDSequence with the same
    config, start, end and stride, capped at --frames -- read at the record's image size.  Returns (sequence, frames);
    ValueError, with the sequence closed, when the selected frame count differs from the record's camera count."""
    from splatam_b200 import datasets, formats
    import run_slam_dataset as rsd
    raw = formats.read_record(record, formats.CHECKPOINT_KEYS + formats.CAMERA_KEYS)
    T = raw["cam_unnorm_rots"].shape[-1]
    height, width = int(raw["org_height"]), int(raw["org_width"])
    cfg = datasets.load_config(a.config) if a.config else None
    seq = datasets.RGBDSequence(a.dataset, a.basedir, a.sequence, cfg, start=a.start, end=a.end, stride=a.stride,
                                desired_height=height, desired_width=width, device=device)
    frames = rsd._Capped(seq, a.frames)
    if len(frames) != T:
        seq.close()
        raise ValueError("%s has %d cameras but --start %d --end %d --stride %d --frames %d select %d frames of %s: pass "
                         "the flags of the run" % (record, T, a.start, a.end, a.stride, a.frames, len(frames),
                                                   a.sequence))
    return seq, frames


def main(argv=None):
    a = parse_args(argv)
    from splatam_b200 import formats, mesh
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    seq = frames = None
    if a.source == "input":
        seq, frames = open_input(a, a.record, dev)
    t0 = time.perf_counter()
    try:
        verts, cols, faces, info = mesh.mesh_record(
            a.record, a.voxel, every=a.every, sil_thres=a.sil_thres, depth_max=a.depth_max, bounds=a.bounds,
            batch=a.batch, trunc=a.trunc, min_weight=a.min_weight, device=dev, source=frames)
    finally:
        if seq is not None:
            seq.close()
    wall = time.perf_counter() - t0
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    formats.save_mesh_ply(a.out, verts, cols, faces)
    line = dict(record=a.record, out=a.out, source=a.source, voxel=info["voxel_size"], trunc=info["trunc"],
                voxels=info["voxels"], dims=list(info["dims"]), frames=info["frames"], V=int(verts.shape[0]),
                F=int(faces.shape[0]), render_ms=info["render_ms"], integrate_ms=info["integrate_ms"],
                extract_ms=info["extract_ms"], wall_s=wall)
    print(json.dumps(line))
    return line


if __name__ == "__main__":
    main()
