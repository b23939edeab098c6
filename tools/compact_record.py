#!/usr/bin/env python
"""Compacts a finished SplaTAM run record to the Gaussians its views use (splatam_b200.contrib.compact_record):
renders the frames evaluate.select_frames(T, --every) picks, each at the record's camera column and as `evaluate`
renders it, gathers per-Gaussian blend statistics on the GPU, and writes --out without the Gaussians the keep rule
drops.  Every other entry of the record is copied as it is, so the viewers, export_ply, render_record.py,
extract_mesh.py, eval_record.py and the offline optimiser open the output.

  --min-weight 0  (default) lossless: keeps the Gaussians that blended into or ended the walk of some pixel of some
                  view; the compacted map renders bit-identically at those views
  --min-weight W  lossy: keeps the Gaussians whose largest blend weight alpha * T reached W; also reports the PSNR and
                  depth L1 of the compacted map's renders against the original's at the same views

Takes this project's or the reference's params.npz (14 keys) or the offline record (13 keys); a checkpoint has no
camera and is refused.  The input is never written.  Prints one JSON line.  One GPU.

  python tools/compact_record.py --record runs/room0/params.npz --out runs/room0/params_compact.npz --every 5"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def parse_args(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--record", required=True, help="params.npz of a finished run")
    ap.add_argument("--out", required=True, help="where to write the compacted record (not --record)")
    ap.add_argument("--every", type=int, default=1, help="the views: frame 0 and every frame t with (t + 1) %% N == 0")
    ap.add_argument("--min-weight", type=float, default=0.0, help="0: lossless rule; > 0: max_weight >= W")
    a = ap.parse_args(argv)
    if a.every < 1:
        ap.error("--every must be >= 1")
    if not a.min_weight >= 0.0:
        ap.error("--min-weight must be >= 0")
    if not os.path.isfile(a.record):
        ap.error("--record %s: no such file" % a.record)
    if os.path.abspath(a.out) == os.path.abspath(a.record) or \
            (os.path.exists(a.out) and os.path.samefile(a.out, a.record)):
        ap.error("--out must differ from --record: the input record is never written")
    return a


def main(argv=None):
    a = parse_args(argv)
    import torch
    from splatam_b200 import contrib
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    res = contrib.compact_record(a.record, a.out, every=a.every, min_weight=a.min_weight, device=dev)
    line = dict(record=a.record, out=res["path"], every=a.every, min_weight=a.min_weight,
                gaussians_before=res["gaussians_before"], gaussians_after=res["gaussians_after"],
                removed_fraction=1.0 - res["gaussians_after"] / max(res["gaussians_before"], 1), views=res["views"],
                width=res["width"], height=res["height"], stats_s=res["stats_s"], compact_s=res["compact_s"])
    if "psnr_db" in res:
        line.update(psnr_db=res["psnr_db"], depth_l1_m=res["depth_l1_m"])
    print(json.dumps(line))
    return line


if __name__ == "__main__":
    main()
