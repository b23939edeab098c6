#!/usr/bin/env python
"""Renders a saved run record as the reference's viewers show it (viz_scripts/final_recon.py, online_recon.py), with
no display: the final view as DIR/final.png, or the online reconstruction as DIR/online/%06d.png, one frame per
timestep (every --every-th).  The record is a params.npz from formats.save_run_record or the reference, an offline
record, or a checkpoint params{t}.npz together with --camera-from (a run record whose intrinsics, w2c and image size
are used).  The viz settings default to the shipped configs' and can be set one by one.

--raw FILE also writes the frames as one raw RGB24 stream, which an external encoder can turn into a video, e.g.
  ffmpeg -f rawvideo -pix_fmt rgb24 -s 1200x680 -r 5 -i FILE -pix_fmt yuv420p online.mp4
(-s is viz_w * view_scale x viz_h * view_scale; ffmpeg is not needed by this tool).  Prints one JSON line.  One GPU.

  python tools/render_record.py --record runs/room0/params.npz --out runs/room0/viz --view online --render-mode depth"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402


def parse(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--record", required=True)
    ap.add_argument("--out", required=True)
    ap.add_argument("--view", choices=("final", "online"), default="final")
    ap.add_argument("--render-mode", choices=("color", "depth", "centers"), default="color")
    ap.add_argument("--show-sil", action="store_true")
    ap.add_argument("--no-cams", action="store_true", help="no camera frustums and trajectory")
    ap.add_argument("--no-offset", action="store_true", help="final view: no +0.5 offset of the first camera")
    ap.add_argument("--every", type=int, default=1)
    ap.add_argument("--viz-w", type=int, default=600)
    ap.add_argument("--viz-h", type=int, default=340)
    ap.add_argument("--viz-near", type=float, default=0.01)
    ap.add_argument("--viz-far", type=float, default=100.0)
    ap.add_argument("--view-scale", type=int, default=2)
    ap.add_argument("--camera-from", default=None, help="run record that supplies a checkpoint's camera")
    ap.add_argument("--raw", default=None)
    ap.add_argument("--device", default="cuda:0")
    return ap.parse_args(argv)


def main(argv=None):
    a = parse(argv)
    from splatam_b200 import formats, viewer as V
    cfg = V.ViewerConfig(render_mode=a.render_mode, show_sil=a.show_sil, visualize_cams=not a.no_cams,
                         offset_first_viz_cam=not a.no_offset, viz_w=a.viz_w, viz_h=a.viz_h, viz_near=a.viz_near,
                         viz_far=a.viz_far, view_scale=a.view_scale)
    camera = None
    if a.camera_from:
        src = formats.read_record(a.camera_from, formats.CAMERA_KEYS)
        camera = {k: src[k] for k in formats.CAMERA_KEYS}
    rec = V.load_record(a.record, torch.device(a.device), cfg, camera=camera)
    t0 = time.perf_counter()
    paths = V.render_record(rec, cfg, a.out, a.view, every=a.every, raw=a.raw)
    dt = time.perf_counter() - t0
    print(json.dumps(dict(record=os.path.abspath(a.record), view=a.view, frames=len(paths), gaussians=rec.P,
                          timesteps=rec.T, size=[cfg.viz_w * cfg.view_scale, cfg.viz_h * cfg.view_scale],
                          out=os.path.abspath(a.out), raw=a.raw, seconds=round(dt, 3))))


if __name__ == "__main__":
    main()
