#!/usr/bin/env python
"""Evaluates a finished SplaTAM run record without re-running SLAM, as the reference's scripts/eval_novel_view.py
does: opens a params.npz written by formats.save_run_record (tools/run_slam_dataset.py --out) or by the reference,
reads the sequence with splatam_b200.datasets and scores the map with the GPU evaluation.

  --split train  (default) the record's Gaussians and cameras through evaluate.evaluate, with the ATE of the record's
                 trajectory against the reader's ground truth; the record needs one camera column for every evaluated
                 frame
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
import importlib.util
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402
import torch  # noqa: E402


def _run_slam_dataset():
    spec = importlib.util.spec_from_file_location("run_slam_dataset", os.path.join(ROOT, "tools", "run_slam_dataset.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


RSD = _run_slam_dataset()


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
    a = ap.parse_args(argv)
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


def load_record(path, split, num_frames, eval_every):
    """The record's arrays (formats.load_params).  Checks that it has the five Gaussian tensors and, for the train
    split, a camera column for every frame evaluate.select_frames picks among `num_frames`: ValueError naming the first
    frame index without one."""
    from splatam_b200 import evaluate, formats
    rec = formats.load_params(path)
    need = formats.GAUSSIAN_KEYS + (("cam_unnorm_rots", "cam_trans") if split == "train" else ())
    missing = [k for k in need if k not in rec]
    if missing:
        raise ValueError("%s lacks %s" % (path, ", ".join(missing)))
    if split == "train":
        n_cam = min(rec["cam_unnorm_rots"].shape[-1], rec["cam_trans"].shape[-1])
        bad = [t for t in evaluate.select_frames(num_frames, eval_every) if t >= n_cam]
        if bad:
            raise ValueError("%s has %d camera columns; frame index %d has none" % (path, n_cam, bad[0]))
    return rec


def main(argv=None):
    a = parse_args(argv)
    from splatam_b200 import datasets, evaluate, formats
    h = RSD.HYPER[a.dataset]
    files = datasets.SequenceFiles(a.dataset, a.basedir, a.sequence, desired_height=h["height"],
                                   desired_width=h["width"], split=a.split)
    T = min(a.frames, len(files)) if a.frames else len(files)
    rec = load_record(a.record, a.split, T, h["eval_every"])
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    net = None if a.lpips_alexnet is None else evaluate.LpipsAlex.load(a.lpips_alexnet, a.lpips_lin, dev)
    t32 = lambda k: torch.from_numpy(np.ascontiguousarray(rec[k], dtype=np.float32)).to(dev)
    gauss = {k: t32(k) for k in formats.GAUSSIAN_KEYS}
    save = not a.no_frames
    with datasets.RGBDSequence(a.dataset, a.basedir, a.sequence, desired_height=h["height"], desired_width=h["width"],
                               device=dev, split=a.split) as seq:
        frames = RSD._Capped(seq, T)
        torch.cuda.synchronize(dev)
        t0 = time.perf_counter()
        if a.split == "train":
            params = dict(gauss, cam_unnorm_rots=t32("cam_unnorm_rots")[..., :T], cam_trans=t32("cam_trans")[..., :T])
            gt_w2c = [torch.linalg.inv(seq.files.poses[t].to(dev)) for t in range(T)]
            res = evaluate.evaluate(params, frames, seq.cam, RSD.SIL_THRES, h["mapping_iters"], True,
                                    eval_every=h["eval_every"], gt_w2c=gt_w2c, out_dir=a.out, lpips=net,
                                    save_frames=save)
        else:
            res = evaluate.evaluate_nvs(gauss, frames, seq.cam, RSD.SIL_THRES, h["mapping_iters"], True,
                                        eval_every=h["eval_every"], out_dir=a.out, lpips=net, save_frames=save)
        eval_s = time.perf_counter() - t0
    line = dict(dataset=a.dataset, sequence=a.sequence, split=a.split, record=a.record, out=a.out, frames=T,
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
