#!/usr/bin/env python
"""Offline map optimisation over all frames of a recorded sequence (splatam_b200.offline), as the reference's two
offline drivers run it, with the shipped hyper-parameters of R/configs/{replica,scannetpp}/{post_splatam_opt,
gaussian_splatting}.py.  One GPU.

  --mode post_splatam --record runs/room0/params.npz   refines a finished SplaTAM map (post_splatam_opt.py): the
                                                       record's Gaussians and `timestep`, each frame trained at the
                                                       record's camera column of its original index
  --mode gt_poses                                      3DGS with ground-truth poses (gaussian_splatting.py): frame 0
                                                       back-projected at the init size, every later frame grown at
                                                       its ground-truth pose, then the same loop

  python tools/run_offline_opt.py --mode post_splatam --record runs/room0/params.npz --dataset replica \\
      --basedir data/Replica --sequence room0 --out runs/room0_post
  python tools/run_offline_opt.py --mode gt_poses --dataset scannetpp --basedir data/ScanNet++/data \\
      --sequence 8b5caf3398 --nvs --out runs/8b5c_3dgs

--start / --end / --stride / --frames select the training frames (stride and frame count default to the config's);
--iters overrides the iteration count.  The map is evaluated after iteration 7000 and at the end with
evaluate.evaluate(at_gt_pose=True) over the eval reader (the config's eval_stride and eval_num_frames); --out writes
psnr.txt / rmse.txt / l1.txt / ssim.txt (and lpips.txt) under eval_7k/ and eval/ and the reference's post-opt
params.npz (formats.save_run_record without keyframe_time_indices).  --lpips-alexnet / --lpips-lin add LPIPS; --nvs
(scannetpp) also runs evaluate_nvs on the test split.  Prints one JSON line: the final evaluation, the training-frame
PSNR before and after the loop, initial and final Gaussian counts, wall time and iterations/s of the loop (the
iteration-7000 evaluation is timed apart, as eval_7k_s)."""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402
import torch  # noqa: E402

from splatam_b200 import offline  # noqa: E402

# (dataset, mode) -> reader sizes, strides, frame counts (-1: all) and iterations of the shipped config;
# learning rates, loss weights and the densify schedule are offline.LRS / LOSS_WEIGHTS / DENSIFY in all four.
# ScanNet++'s num_frames is -1 here: the shipped configs pick it per scene (scene_num_frames = [-1, 360], so one of the
# two scenes they list trains on its first 360 frames); give --frames 360 for that scene.
HYPER = {
    ("replica", "post_splatam"): dict(height=680, width=1200, stride=20, num_frames=100, eval_stride=5,
                                      eval_num_frames=400, iters=15000),
    ("scannetpp", "post_splatam"): dict(height=584, width=876, stride=1, num_frames=-1, eval_stride=1,
                                        eval_num_frames=-1, iters=30000),
    ("replica", "gt_poses"): dict(height=340, width=600, init_height=170, init_width=300, stride=1, num_frames=2000,
                                  eval_stride=10, eval_num_frames=200, iters=30000),
    ("scannetpp", "gt_poses"): dict(height=584, width=876, init_height=584, init_width=876, stride=1, num_frames=-1,
                                    eval_stride=1, eval_num_frames=-1, iters=7000),
}
MODES = ("post_splatam", "gt_poses")
SIL_THRES = 0.5
SEED = 0
EVAL_7K = 7000


def score(params, eval_frames, cam, iters, lpips=None, out_dir=None):
    """The offline drivers' `eval` (R/utils/gs_helpers.py:463-510) of the Gaussians `params`: evaluate.evaluate over the
    eval frames at their ground-truth poses, all frames, no presence mask (mapping_iters > 0)."""
    from splatam_b200 import evaluate
    return evaluate.evaluate(params, eval_frames, cam, SIL_THRES, iters, True, eval_every=1, at_gt_pose=True,
                             lpips=lpips, out_dir=out_dir)


def _frames(seq, n):
    n = len(seq) if n is None or n < 0 else min(n, len(seq))
    return [seq[t] for t in range(n)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--mode", required=True, choices=MODES)
    ap.add_argument("--record", default=None, help="post_splatam: the SplaTAM run's params.npz")
    ap.add_argument("--dataset", required=True, choices=sorted({d for d, _ in HYPER}))
    ap.add_argument("--basedir", required=True)
    ap.add_argument("--sequence", required=True)
    ap.add_argument("--config", default=None, help="data YAML (camera_params); default: the shipped camera")
    ap.add_argument("--start", type=int, default=0)
    ap.add_argument("--end", type=int, default=-1)
    ap.add_argument("--stride", type=int, default=0, help="training-frame stride (0: the config's)")
    ap.add_argument("--frames", type=int, default=0, help="use only the first N training frames (0: the config's)")
    ap.add_argument("--eval-frames", type=int, default=0, help="evaluate only the first N eval frames (0: the config's)")
    ap.add_argument("--iters", type=int, default=0)
    ap.add_argument("--prefetch", type=int, default=2)
    ap.add_argument("--out", default=None)
    ap.add_argument("--nvs", action="store_true", help="also evaluate novel views on the test split (scannetpp)")
    ap.add_argument("--lpips-alexnet", default=None, help="torchvision AlexNet weights (alexnet-owt-7be5be79.pth)")
    ap.add_argument("--lpips-lin", default=None, help="LPIPS v0.1 linear heads (alex.pth)")
    a = ap.parse_args()
    if (a.mode == "post_splatam") != (a.record is not None):
        ap.error("--record is required with --mode post_splatam and not accepted otherwise")
    if (a.lpips_alexnet is None) != (a.lpips_lin is None):
        ap.error("--lpips-alexnet and --lpips-lin go together")
    if a.nvs and a.dataset != "scannetpp":
        ap.error("--nvs needs a dataset with a test split (scannetpp)")
    from splatam_b200 import datasets, evaluate, formats
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    torch.manual_seed(SEED); np.random.seed(SEED)              # seed_everything: densify's split samples
    h = dict(HYPER[(a.dataset, a.mode)])
    stride = a.stride or h["stride"]
    n_train = a.frames or h["num_frames"]
    n_eval = a.eval_frames or h["eval_num_frames"]
    iters = a.iters or h["iters"]
    cfg = datasets.load_config(a.config) if a.config else None
    net = None if a.lpips_alexnet is None else evaluate.LpipsAlex.load(a.lpips_alexnet, a.lpips_lin, dev)
    reader = lambda s, hh, ww, **kw: datasets.RGBDSequence(a.dataset, a.basedir, a.sequence, cfg, start=a.start,
                                                            end=a.end, stride=s, desired_height=hh, desired_width=ww,
                                                            device=dev, prefetch=a.prefetch, **kw)
    seq = reader(stride, h["height"], h["width"])
    frames = _frames(seq, n_train)
    if a.mode == "post_splatam":
        index = seq.files.retained_inds[:len(frames)].tolist()      # original indices: start + stride * t
        mapper, train, radius, _ = offline.from_record(a.record, frames, index, dev)
    else:
        with reader(stride, h["init_height"], h["init_width"]) as init_seq:
            mapper, train, radius = offline.from_gt_poses(_frames(init_seq, len(frames)), frames, sil_thres=SIL_THRES)
    seq.close()
    initial = int(mapper.g.shapes["means3D"][0])
    psnr_before = offline.train_psnr(mapper, train)
    eval_seq = reader(h["eval_stride"], h["height"], h["width"])
    eval_frames = _frames(eval_seq, n_eval)
    eval_seq.close()

    sub = lambda name: None if a.out is None else os.path.join(a.out, name)
    evals, eval_s = {}, [0.0]

    def on_eval(it, m):           # timed apart: the loop's rate excludes the intermediate evaluation
        torch.cuda.synchronize(dev)
        t = time.perf_counter()
        evals[it] = score(m.g.params, eval_frames, seq.cam, iters, net, sub("eval_7k"))
        eval_s[0] += time.perf_counter() - t
    torch.cuda.synchronize(dev)
    t0 = time.perf_counter()
    counts = offline.optimize_map(mapper, train, iters, offline.MEANS3D_LR_FINAL, offline.DENSIFY, radius, seed=SEED,
                                  eval_at=(EVAL_7K,), on_eval=on_eval)
    torch.cuda.synchronize(dev)
    wall = time.perf_counter() - t0 - eval_s[0]
    res = score(mapper.g.params, eval_frames, seq.cam, iters, net, sub("eval"))
    psnr_after = offline.train_psnr(mapper, train)
    nvs = {}
    if a.nvs:
        with datasets.RGBDSequence(a.dataset, a.basedir, a.sequence, cfg, desired_height=h["height"],
                                   desired_width=h["width"], device=dev, prefetch=a.prefetch, split="test") as test:
            r = evaluate.evaluate_nvs(mapper.g.params, test, test.cam, SIL_THRES, iters, True, eval_every=1, lpips=net,
                                      out_dir=None if a.out is None else os.path.join(a.out, "eval_nvs"))
        nvs = dict(nvs_psnr_db=r["psnr"], nvs_ms_ssim=r["ms_ssim"], nvs_depth_rmse_m=r["depth_rmse"],
                   nvs_depth_l1_m=r["depth_l1"], nvs_valid_frames=int(r["valid_nvs_frames"].sum()),
                   **({} if net is None else dict(nvs_lpips=r["lpips"])))
    if a.out is not None:
        cam = mapper.cam
        formats.save_run_record(a.out, mapper.g.params, cam["cam_unnorm_rots"], cam["cam_trans"], mapper.timestep,
                                seq.intrinsics, seq.w2c, seq.width, seq.height, offline.record_poses(train), None)
    print(json.dumps(dict(
        mode=a.mode, dataset=a.dataset, sequence=a.sequence, width=seq.width, height=seq.height, stride=stride,
        frames=len(train), eval_frames=len(eval_frames), iters=iters, initial_gaussians=initial,
        gaussians=int(counts[-1]) if counts else initial, psnr_db=res["psnr"], ms_ssim=res["ms_ssim"],
        depth_l1_m=res["depth_l1"], **({} if net is None else dict(lpips=res["lpips"])),
        psnr_7k_db=evals[EVAL_7K]["psnr"] if EVAL_7K in evals else None,
        train_psnr_before_db=psnr_before, train_psnr_after_db=psnr_after, wall_s=wall,
        iters_per_s=iters / wall if wall > 0 else None, eval_7k_s=eval_s[0] if evals else None, **nvs,
        metric_note="psnr / ms_ssim / depth_l1 = evaluate at the eval frames' ground-truth poses after the last "
                    "iteration; train_psnr = mean PSNR of the training frames at their training poses; wall_s and "
                    "iters_per_s = the loop without the iteration-7000 evaluation (eval_7k_s)")))


if __name__ == "__main__":
    main()
