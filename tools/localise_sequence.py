"""Localise a new RGB-D sequence in a saved SplaTAM map (reloc.localise_sequence): the map stays frozen, frame 0 is
relocalised with no prior, every later frame is tracked from the constant-velocity guess (or ICP), health-checked and
relocalised when lost.  The relocalisation database holds the record's renders at its keyframe columns
(`keyframe_time_indices`), or at every --every-th column when the record has none.

    tools/localise_sequence.py --record D/params.npz --dataset replica --basedir B --sequence S [--every N] [--out DIR]

The query is read at the record's image size (org_height x org_width) with the dataset's camera; the database renders
use that camera too.  Writes DIR/localised.npz (cam_unnorm_rots / cam_trans in the map's frame, per-frame lost,
relocalised and health [T,5]: valid, covered, inliers, rms, healthy) and prints one JSON line with the lost and
relocalised counts.  With --map-dataset / --map-basedir / --map-sequence (the sequence the map was built from), the
ground truth of both sequences is put in the map's frame -- the query's poses through the map sequence's world_to_map
and the inverse of the query's own -- and the line also holds the absolute ATE in the map frame (RMSE of camera
centres; a global offset is what localisation must get right) and the Horn-aligned ATE (slam.ate_horn)."""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402
import torch  # noqa: E402


def parse_args(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--record", required=True, help="params.npz of a run (formats.save_run_record)")
    ap.add_argument("--dataset", required=True)
    ap.add_argument("--basedir", required=True)
    ap.add_argument("--sequence", required=True)
    ap.add_argument("--config", default=None, help="data YAML (camera_params) of the query; default: the shipped camera")
    ap.add_argument("--frames", type=int, default=0, help="use only the first N frames (0: all)")
    ap.add_argument("--every", type=int, default=5, help="database columns when the record has no keyframe list")
    ap.add_argument("--pose-init", default="constant_velocity", choices=("constant_velocity", "icp", "rgbd_icp"))
    ap.add_argument("--photometric", action="store_true",
                    help="photometric health check (colour NCC of the map's render against the frame) and RGB-D ICP "
                         "verification of the candidates")
    ap.add_argument("--tracking-iters", type=int, default=40)
    ap.add_argument("--k", type=int, default=5, help="candidates verified by ICP")
    ap.add_argument("--map-dataset", default=None)
    ap.add_argument("--map-basedir", default=None)
    ap.add_argument("--map-sequence", default=None)
    ap.add_argument("--map-config", default=None)
    ap.add_argument("--out", default=None, help="output directory (default: the record's)")
    a = ap.parse_args(argv)
    if not os.path.isfile(a.record):
        ap.error("--record %s: no such file" % a.record)
    if a.every < 1:
        ap.error("--every must be positive")
    if a.frames < 0:
        ap.error("--frames must be 0 (all) or positive")
    if a.tracking_iters < 1:
        ap.error("--tracking-iters must be positive")
    if not 1 <= a.k <= 8:
        ap.error("--k must be in [1, 8]")
    given = [v is not None for v in (a.map_dataset, a.map_basedir, a.map_sequence)]
    if any(given) and not all(given):
        ap.error("--map-dataset, --map-basedir and --map-sequence go together")
    if a.map_config is not None and not all(given):
        ap.error("--map-config needs --map-dataset, --map-basedir and --map-sequence")
    return a


def ate(gt_w2c, est_w2c):
    """(absolute ATE: RMSE of camera centres without alignment, Horn-aligned ATE as slam.ate_horn) in metres."""
    from splatam_b200 import slam
    c = lambda m: -(m[:3, :3].T @ m[:3, 3])
    d = np.stack([c(g) - c(e) for g, e in zip(gt_w2c, est_w2c)])
    horn = slam.ate_horn([torch.from_numpy(g) for g in gt_w2c], [torch.from_numpy(e) for e in est_w2c])
    return float(np.sqrt((d ** 2).sum(1).mean())), horn


def main(argv=None):
    a = parse_args(argv)
    from splatam_b200 import datasets, formats, mapping as M, reloc
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    rec = formats.read_record(a.record, formats.CHECKPOINT_KEYS + ("org_width", "org_height"))
    params = {k: torch.from_numpy(np.asarray(rec[k], np.float32)).to(dev).contiguous()
              for k in formats.CHECKPOINT_KEYS}
    T_map = params["cam_unnorm_rots"].shape[-1]
    cols = ([int(i) for i in np.asarray(rec["keyframe_time_indices"]).reshape(-1)] if "keyframe_time_indices" in rec
            else list(range(0, T_map, a.every)))
    if not cols or min(cols) < 0 or max(cols) >= T_map:
        raise SystemExit("%s: database columns %s outside the record's %d cameras" % (a.record, cols, T_map))
    height, width = int(rec["org_height"]), int(rec["org_width"])
    cfg = datasets.load_config(a.config) if a.config else None
    out_dir = a.out or os.path.dirname(os.path.abspath(a.record))
    t0 = time.perf_counter()
    with datasets.RGBDSequence(a.dataset, a.basedir, a.sequence, cfg, desired_height=height, desired_width=width,
                               device=dev, prefetch=2) as seq:
        n = len(seq) if a.frames == 0 else min(a.frames, len(seq))
        frames = [seq[t] for t in range(n)]
        K = seq.intrinsics.cpu().double().numpy()
        db = reloc.Database.from_record(params, cols, seq.cam, w2c0=frames[0]["w2c"])
        cfg = reloc.config(dict(k=a.k, photometric=a.photometric))
        res = reloc.localise_sequence(params, frames, K, db, cfg, pose_init=a.pose_init,
                                      tracking=dict(num_iters=a.tracking_iters))
        query_to_world = np.linalg.inv(seq.files.world_to_map)
        rel = [seq.files.poses[t].double().numpy() for t in range(n)]
    torch.cuda.synchronize(dev)
    wall = time.perf_counter() - t0
    os.makedirs(out_dir, exist_ok=True)
    path = os.path.join(out_dir, "localised.npz")
    np.savez(path, cam_unnorm_rots=res["rots"].cpu().numpy(), cam_trans=res["trans"].cpu().numpy(),
             lost=np.array(res["lost"]), relocalised=np.array(res["relocalised"]), health=res["health"])
    line = dict(record=a.record, out=path, frames=n, database=len(cols), lost=int(sum(res["lost"])),
                relocalised=int(sum(res["relocalised"])), wall_s=round(wall, 3))
    if a.map_dataset is not None:
        mcfg = datasets.load_config(a.map_config) if a.map_config else None
        files = datasets.SequenceFiles(a.map_dataset, a.map_basedir, a.map_sequence, mcfg)
        to_map = files.world_to_map @ query_to_world
        gt = [np.linalg.inv(to_map @ r) for r in rel]
        w2c0 = frames[0]["w2c"].double().cpu().numpy()
        est = [w2c0 @ M.camera_w2c(res["rots"][..., t], res["trans"][..., t])[0].double().cpu().numpy()
               for t in range(n)]
        line["ate_abs_m"], line["ate_horn_m"] = ate(gt, est)
    print("lost %d of %d frames, relocalised %d" % (line["lost"], n, line["relocalised"]))
    print(json.dumps(line))
    return line


if __name__ == "__main__":
    main()
