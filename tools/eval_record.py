#!/usr/bin/env python
"""Evaluates a finished SplaTAM run record without re-running SLAM, as the reference's scripts/eval_novel_view.py
does: opens a params.npz written by formats.save_run_record (tools/run_slam_dataset.py --out) or by the reference,
reads the sequence with splatam_b200.datasets and scores the map with the GPU evaluation.

  --split train  (default) the record's Gaussians and cameras through evaluate.evaluate, with the ATE of the record's
                 trajectory against the reader's ground truth; the record needs one camera column for every evaluated
                 frame; --exposure PATH (the run's exposure.npz) scores the renders through each frame's colour
                 correction
  --split test   the Gaussians through evaluate.evaluate_nvs on the held-out views, at their ground-truth poses
                 (scannetpp, replicav2)

Image size, eval_every and the mapping settings that choose the masks are the shipped ones of the dataset
(run_slam_dataset.HYPER).  The per-frame lists (psnr.txt, rmse.txt, l1.txt, ssim.txt, lpips.txt) and, unless
--no-frames, the rendered and ground-truth frames (rendered_rgb/, rendered_depth/, rgb/, depth/) are written to --out,
by default <record dir>/eval_train or <record dir>/eval_nvs.  --frames N evaluates the first N frames of the split.
--lpips-alexnet PATH --lpips-lin PATH add LPIPS, as for run_slam_dataset.py.  Prints one JSON line.  One GPU.

  python tools/eval_record.py --dataset replica --basedir data/Replica --sequence room0 --record runs/room0/params.npz
  python tools/eval_record.py --dataset replicav2 --basedir data/ReplicaV2 --sequence room_0 \\
      --record runs/room_0/params.npz --split test"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import torch  # noqa: E402
import run_slam_dataset as RSD  # noqa: E402


def parse_args(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--dataset", required=True, choices=sorted(RSD.HYPER))
    ap.add_argument("--basedir", required=True)
    ap.add_argument("--sequence", required=True)
    ap.add_argument("--record", required=True, help="params.npz of a finished run")
    ap.add_argument("--split", default="train", choices=("train", "test"))
    ap.add_argument("--out", default=None, help="default: <record dir>/eval_train or <record dir>/eval_nvs")
    ap.add_argument("--frames", type=int, default=0, help="evaluate only the first N frames of the split (0: all)")
    ap.add_argument("--no-frames", action="store_true", help="do not save the rendered and ground-truth frames")
    ap.add_argument("--lpips-alexnet", default=None, help="torchvision AlexNet weights (alexnet-owt-7be5be79.pth)")
    ap.add_argument("--lpips-lin", default=None, help="LPIPS v0.1 linear heads (alex.pth)")
    ap.add_argument("--exposure", default=None, metavar="PATH",
                    help="exposure.npz of the run (--split train): score each frame's render through its colour "
                         "correction")
    a = ap.parse_args(argv)
    if a.exposure is not None and a.split != "train":
        ap.error("--exposure applies to --split train only (held-out views have no exposure estimate)")
    if a.exposure is not None and not os.path.isfile(a.exposure):
        ap.error("--exposure %s: no such file" % a.exposure)
    if (a.lpips_alexnet is None) != (a.lpips_lin is None):
        ap.error("--lpips-alexnet and --lpips-lin go together")
    if a.frames < 0:
        ap.error("--frames must be 0 (all) or positive")
    if a.split == "test" and a.dataset not in ("scannetpp", "replicav2"):
        ap.error("--split test needs a dataset with a test split (scannetpp, replicav2)")
    if not os.path.isfile(a.record):
        ap.error("--record %s: no such file" % a.record)
    if a.out is None:
        a.out = os.path.join(os.path.dirname(os.path.abspath(a.record)), "eval_train" if a.split == "train" else "eval_nvs")
    return a


def main(argv=None):
    a = parse_args(argv)
    from splatam_b200 import datasets, evaluate, formats
    h = RSD.HYPER[a.dataset]
    files = datasets.SequenceFiles(a.dataset, a.basedir, a.sequence, desired_height=h["height"],
                                   desired_width=h["width"], split=a.split)
    T = min(a.frames, len(files)) if a.frames else len(files)
    # the train split renders every evaluated frame at the record's camera column for it
    rec = formats.read_record(a.record, formats.CHECKPOINT_KEYS if a.split == "train" else formats.GAUSSIAN_KEYS)
    if a.split == "train":
        formats.check_camera_columns(a.record, rec, evaluate.select_frames(T, h["eval_every"]))
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    net = None if a.lpips_alexnet is None else evaluate.LpipsAlex.load(a.lpips_alexnet, a.lpips_lin, dev)
    gauss = formats.record_tensors(rec, formats.GAUSSIAN_KEYS, dev)
    save = not a.no_frames
    with datasets.RGBDSequence(a.dataset, a.basedir, a.sequence, desired_height=h["height"], desired_width=h["width"],
                               device=dev, split=a.split) as seq:
        frames = RSD._Capped(seq, T)
        torch.cuda.synchronize(dev)
        t0 = time.perf_counter()
        if a.split == "train":
            cams = formats.record_tensors(rec, ("cam_unnorm_rots", "cam_trans"), dev)
            params = dict(gauss, **{k: v[..., :T] for k, v in cams.items()})
            if a.exposure is not None:
                expo = formats.load_exposure(a.exposure, num_frames=rec["cam_trans"].shape[-1], device=dev)
                params["cam_exposure"] = expo[..., :T].contiguous()
            gt_w2c = [torch.linalg.inv(seq.files.poses[t].to(dev)) for t in range(T)]
            res = evaluate.evaluate(params, frames, seq.cam, RSD.SIL_THRES, h["mapping_iters"], True,
                                    eval_every=h["eval_every"], gt_w2c=gt_w2c, out_dir=a.out, lpips=net,
                                    save_frames=save)
        else:
            res = evaluate.evaluate_nvs(gauss, frames, seq.cam, RSD.SIL_THRES, h["mapping_iters"], True,
                                        eval_every=h["eval_every"], out_dir=a.out, lpips=net, save_frames=save)
        eval_s = time.perf_counter() - t0
    line = dict(dataset=a.dataset, sequence=a.sequence, split=a.split, record=a.record, exposure=a.exposure, out=a.out,
                frames=T,
                width=int(h["width"]), height=int(h["height"]), gaussians=int(gauss["means3D"].shape[0]),
                evaluated_frames=len(res["frame_ids"]), frames_saved=save, psnr_db=res["psnr"], ms_ssim=res["ms_ssim"],
                depth_rmse_m=res["depth_rmse"], depth_l1_m=res["depth_l1"], eval_s=eval_s)
    if a.split == "train":
        line["ate_m"] = res["ate"]
    else:
        line["valid_frames"] = int(res["valid_nvs_frames"].sum())
    if net is not None:
        line["lpips"] = res["lpips"]
    print(json.dumps(line))
    return res


if __name__ == "__main__":
    main()
