#!/usr/bin/env python
"""Times SplaTAM's final evaluation on one GPU: splatam_b200.evaluate over a 1200x680 view-filling map
(scenes.view_filling, Replica intrinsics) and 200 frames along slam.look_trajectory, against the reference's metric
path (R/utils/eval_helpers.py:463-507: PSNR and depth errors in PyTorch on the GPU, MS-SSIM by pytorch_msssim on the
CPU after .cpu(); the float32 restatement in oracle/metrics_torch.py stands in for pytorch_msssim, which is not
installed).  Prints the GPU name and power limit of the run and one JSON line:
  evaluate_frames_per_s      whole evaluate() (two renders + metrics per frame, one read-back at the end)
  metric_kernels_ms_per_frame  sb_frame_metrics + sb_ms_ssim on one frame, CUDA events over --reps calls
  reference_metrics_ms_per_frame  the reference-style metric path for one frame (GPU PyTorch + .cpu() + CPU MS-SSIM)
--nvs instead times evaluate.evaluate_nvs (renders at the ground-truth poses, the unmasked branch with its extra hole
count) over --frames held-out views of a view-filling map at ScanNet++'s 876x584 and ReplicaV2's 1200x680, and
prints nvs_frames_per_s per size.
--lpips instead times sb_lpips (csrc/lpips.cu) on one image pair at 1200x680 and 876x584 with seeded random weights (a
dense convolution's time does not depend on the weight values): the time per call from CUDA events over --reps calls,
each launch's time from a torch.profiler pass, GFLOP/s against the 67 TFLOP/s FP32 data-sheet rate, the same network
through torch.nn.functional on the GPU as the reference-style path, and evaluate() frames/s without and with LPIPS
over --frames frames at 1200x680.
Run:  python tools/time_eval.py [--frames 200] [--reps 100] [--ref-frames 5] [--nvs | --lpips]"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

import scenes  # noqa: E402


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, check=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:          # the name still comes from torch
        q = "%s, power limit unknown (%s)" % (torch.cuda.get_device_name(0), e)
    return q


def reference_metrics(im, depth_sil, gt_im, gt_depth, sil_thres, use_presence):
    """eval_helpers.py:465-507 as the reference runs it, with the float32 MS-SSIM restatement on the CPU."""
    from oracle import metrics_torch as O
    rastered_depth = depth_sil[0, :, :].unsqueeze(0)
    valid = gt_depth > 0
    rastered_depth = rastered_depth * valid
    presence = depth_sil[1, :, :] > sil_thres
    if use_presence:
        w_im, w_gt = im * presence * valid, gt_im * presence * valid
    else:
        w_im, w_gt = im * valid, gt_im * valid
    mse = ((w_im - w_gt) ** 2).view(3, -1).mean(1, keepdim=True)
    psnr = (20 * torch.log10(1.0 / torch.sqrt(mse))).mean()
    ssim = O.ms_ssim(w_im.unsqueeze(0).cpu(), w_gt.unsqueeze(0).cpu(), data_range=1.0, dtype=torch.float32)
    e = (rastered_depth - gt_depth) * presence if use_presence else rastered_depth - gt_depth
    rmse = (torch.sqrt(e ** 2) * valid).sum() / valid.sum()
    l1 = (torch.abs(e) * valid).sum() / valid.sum()
    return psnr.cpu(), ssim, rmse.cpu(), l1.cpu()


def time_nvs(frames_n, sil_thres):
    """{"WxH": evaluate_nvs frames/s} over a view-filling map seen from `frames_n` poses along slam.look_trajectory."""
    import splatam_b200 as S
    from splatam_b200 import evaluate as EV, slam
    from splatam_b200 import mapping as M
    dev = torch.device("cuda:0")
    out = {}
    for w, h in ((876, 584), (1200, 680)):
        cam_d = dict(w=w, h=h, fx=w / 2.0, fy=w / 2.0, cx=(w - 1) / 2.0, cy=(h - 1) / 2.0)
        sc = scenes.view_filling(margin=100, cam=cam_d)
        cam = sc.settings(S.GaussianRasterizationSettings, dev)
        gt = dict(means3D=sc.means3D, rgb_colors=sc.colors, unnorm_rotations=sc.rotations,
                  logit_opacities=torch.logit(sc.opacities.reshape(-1, 1)), log_scales=torch.log(sc.scales[:, :1]))
        gt = {k: v.to(dev).contiguous() for k, v in gt.items()}
        rots, trans = slam.look_trajectory(frames_n, dev, step=(0.002, -0.001, 0.001), rot_step=(0.0005, -0.0004, 0.0003))
        frames = [slam.render_frame(gt, rots, trans, t, cam) for t in range(frames_n)]
        for t, fr in enumerate(frames):
            fr["gt_w2c"] = M.camera_w2c(rots[..., t], trans[..., t])[0]
        EV.evaluate_nvs(gt, frames[:4], cam, sil_thres, 60, True)                 # warm-up
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        res = EV.evaluate_nvs(gt, frames, cam, sil_thres, 60, True)
        torch.cuda.synchronize()
        wall = time.perf_counter() - t0
        out["%dx%d" % (w, h)] = dict(nvs_frames_per_s=round(len(res["frame_ids"]) / wall, 2), gaussians=sc.P,
                                     evaluated=len(res["frame_ids"]), valid=int(res["valid_nvs_frames"].sum()),
                                     psnr=round(res["psnr"], 3))
    return out


# sb_lpips' launches in order, for the per-layer times of the profiled calls
_LPIPS_KERNELS = ("conv1", "pool1", "conv2", "pool2", "conv3", "conv4", "conv5", "head1", "head2", "head3", "head4",
                  "head5", "finalize")


def _lpips_gflop(N, H, W):
    """{conv1..conv5: GFLOP (2 x MAC)} of one sb_lpips call on N pairs (2N images)."""
    from oracle import lpips_torch as OL
    x = torch.empty(2 * N, 3, H, W, device="meta")
    alex, _ = OL.random_state_dicts(0)
    fs = OL.features(x, alex, dtype=torch.float32)
    return {"conv%d" % (l + 1): 2.0 * f.numel() * cin * k * k / 1e9
            for l, (f, (_, cin, _, k, _, _)) in enumerate(zip(fs, OL.ALEX_CONVS))}


def time_lpips(frames_n, reps, sil_thres):
    """sb_lpips at 1200x680 and 876x584 (one pair, seeded random weights): time per call from CUDA events over `reps`
    calls, the time of each launch from a torch.profiler pass, GFLOP/s against the 67 TFLOP/s FP32 data-sheet rate,
    the same network through torch.nn.functional on the GPU (cuDNN with PyTorch's default TF32 setting), and
    evaluate() frames/s without and with LPIPS over `frames_n` frames of a view-filling map."""
    import tempfile
    import splatam_b200 as S
    from oracle import lpips_torch as OL
    from splatam_b200 import _lib, evaluate as EV, slam
    dev = torch.device("cuda:0")
    alex, lin = OL.random_state_dicts(seed=0)
    net = EV.LpipsAlex.from_state_dicts(alex, lin, dev)
    wdev = {k: v.to(dev) for k, v in dict(alex, **lin).items()}
    out = {}
    for w, h in ((1200, 680), (876, 584)):
        g = torch.Generator().manual_seed(w)
        x = torch.rand(1, 3, h, w, generator=g).to(dev)
        y = (x + 0.1 * torch.randn(x.shape, generator=g).to(dev)).clamp(0, 1)
        mean = torch.empty((), dtype=torch.float64, device=dev)
        ws = torch.empty(_lib.nbytes("sb_lpips_workspace_bytes", 1, h, w), dtype=torch.uint8, device=dev)
        call = lambda: EV._lpips_into(x, y, net, None, mean, ws)
        for _ in range(10):
            call()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            call()
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / reps
        # per-launch times: one profiled pass, kernels matched to _LPIPS_KERNELS by launch order
        prof_calls = 20
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            for _ in range(prof_calls):
                call()
            torch.cuda.synchronize()
        with tempfile.TemporaryDirectory() as tmp:
            path = os.path.join(tmp, "trace.json")
            prof.export_chrome_trace(path)
            events = json.load(open(path))["traceEvents"]
        kernels = sorted((e for e in events if e.get("cat") == "kernel"), key=lambda e: e["ts"])
        assert len(kernels) == prof_calls * len(_LPIPS_KERNELS), len(kernels)
        per = {k: 0.0 for k in _LPIPS_KERNELS}
        for i, e in enumerate(kernels):
            per[_LPIPS_KERNELS[i % len(_LPIPS_KERNELS)]] += e["dur"] / 1e3 / prof_calls
        gflop = _lpips_gflop(1, h, w)
        total_gflop = sum(gflop.values())
        # the reference-style path: the same network through torch.nn.functional on the GPU
        ref = lambda: OL.lpips(x, y, wdev, dtype=torch.float32)
        for _ in range(5):
            ref()
        e0.record()
        for _ in range(20):
            r = ref()
        e1.record()
        torch.cuda.synchronize()
        ref_ms = e0.elapsed_time(e1) / 20
        out["%dx%d" % (w, h)] = dict(
            lpips_ms_per_call=round(ms, 4), layer_ms={k: round(v, 4) for k, v in per.items()},
            gflop_per_call=round(total_gflop, 2), gflop_per_s=round(total_gflop / ms * 1e3, 1),
            share_of_67_tflops=round(total_gflop / ms * 1e3 / 67e3, 3),
            conv_gflop_per_s={k: round(gflop[k] / per[k] * 1e3, 1) for k in gflop},
            functional_ms_per_call=round(ref_ms, 3), functional_cudnn_tf32=torch.backends.cudnn.allow_tf32,
            lpips=[mean.item(), float(r[0])])
    # evaluate() with and without LPIPS on a 1200x680 view-filling map, run alternately
    sc = scenes.view_filling(margin=100)
    cam = sc.settings(S.GaussianRasterizationSettings, dev)
    gt = dict(means3D=sc.means3D, rgb_colors=sc.colors, unnorm_rotations=sc.rotations,
              logit_opacities=torch.logit(sc.opacities.reshape(-1, 1)), log_scales=torch.log(sc.scales[:, :1]))
    gt = {k: v.to(dev).contiguous() for k, v in gt.items()}
    rots, trans = slam.look_trajectory(frames_n, dev, step=(0.002, -0.001, 0.001), rot_step=(0.0005, -0.0004, 0.0003))
    frames = [slam.render_frame(gt, rots, trans, t, cam) for t in range(frames_n)]
    params = dict(gt, cam_unnorm_rots=rots, cam_trans=trans)
    g = torch.Generator().manual_seed(1)
    params["rgb_colors"] = (gt["rgb_colors"] + 0.05 * torch.randn(gt["rgb_colors"].shape, generator=g).to(dev)).clamp(0, 1)
    fps = {"without": [], "with": []}
    for lp in (None, net):
        EV.evaluate(params, frames[:4], cam, sil_thres, 0, False, lpips=lp)           # warm-up
    for _ in range(2):
        for key, lp in (("without", None), ("with", net)):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            res = EV.evaluate(params, frames, cam, sil_thres, 0, False, lpips=lp)
            torch.cuda.synchronize()
            fps[key].append(round(frames_n / (time.perf_counter() - t0), 2))
    out["evaluate_1200x680"] = dict(frames=frames_n, frames_per_s_without_lpips=fps["without"],
                                    frames_per_s_with_lpips=fps["with"], lpips=round(res["lpips"], 6))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=200)
    ap.add_argument("--reps", type=int, default=100)
    ap.add_argument("--ref-frames", type=int, default=5)
    ap.add_argument("--sil-thres", type=float, default=0.5)
    ap.add_argument("--nvs", action="store_true", help="time evaluate_nvs at 876x584 and 1200x680 instead")
    ap.add_argument("--lpips", action="store_true", help="time sb_lpips and evaluate() with LPIPS instead")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "time_eval.py measures on a CUDA device"
    if args.lpips:
        print(json.dumps(dict(gpu=gpu_info(), **time_lpips(args.frames, args.reps, args.sil_thres))))
        return
    if args.nvs:
        print(json.dumps(dict(gpu=gpu_info(), frames=args.frames, **time_nvs(args.frames, args.sil_thres))))
        return
    import splatam_b200 as S
    from splatam_b200 import _lib, evaluate as EV, slam
    from splatam_b200 import mapping as M
    dev = torch.device("cuda:0")
    print("GPU:", gpu_info(), flush=True)
    sc = scenes.view_filling(margin=100)          # surface beyond the borders: the moving camera sees a covered view
    cam = sc.settings(S.GaussianRasterizationSettings, dev)
    gt = dict(means3D=sc.means3D, rgb_colors=sc.colors, unnorm_rotations=sc.rotations,
              logit_opacities=torch.logit(sc.opacities.reshape(-1, 1)), log_scales=torch.log(sc.scales[:, :1]))
    gt = {k: v.to(dev).contiguous() for k, v in gt.items()}
    T = args.frames
    rots, trans = slam.look_trajectory(T, dev, step=(0.002, -0.001, 0.001), rot_step=(0.0005, -0.0004, 0.0003))
    frames = [slam.render_frame(gt, rots, trans, t, cam) for t in range(T)]
    g = torch.Generator().manual_seed(1)
    # the evaluated map: colours, sizes and poses a little off the generating scene, as after a SLAM run
    noise = lambda t, s: t + s * torch.randn(t.shape, generator=g).to(dev)
    params = dict(gt, cam_unnorm_rots=noise(rots, 0.0005), cam_trans=noise(trans, 0.001))
    params["cam_unnorm_rots"][..., 0], params["cam_trans"][..., 0] = rots[..., 0], trans[..., 0]
    params["rgb_colors"] = noise(gt["rgb_colors"], 0.05).clamp(0, 1)
    params["log_scales"] = noise(gt["log_scales"], 0.05)
    gt_w2c = slam.w2c_list(rots, trans)

    # evaluate(): warm up on a few frames, then the whole sequence
    EV.evaluate(params, frames[:4], cam, args.sil_thres, 0, False)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = EV.evaluate(params, frames, cam, args.sil_thres, 0, False, gt_w2c=gt_w2c)
    torch.cuda.synchronize()
    wall = time.perf_counter() - t0

    # the metric kernels alone on frame 1's renders, CUDA events over --reps calls
    H, W = sc.h, sc.w
    with torch.no_grad():
        im, ds, _, _ = M._render_pair(params, dict(frames[1], cam=cam), M.default_render, True, camera_grad=False)
    im, ds = im.contiguous(), ds.contiguous()
    gt_im, gt_d = frames[1]["im"].contiguous(), frames[1]["depth"].contiguous()
    w_im, w_gt = torch.empty_like(im), torch.empty_like(im)
    metrics = torch.zeros(6, dtype=torch.float64, device=dev)
    ws_f = torch.empty(_lib.nbytes("sb_frame_metrics_workspace_bytes", H, W), dtype=torch.uint8, device=dev)
    ws_s = torch.empty(_lib.nbytes("sb_ms_ssim_workspace_bytes", 1, 3, H, W), dtype=torch.uint8, device=dev)

    def kernels():
        _lib.call("sb_frame_metrics", im, ds, gt_im, gt_d, H, W, args.sil_thres, 1, w_im, w_gt, ws_f, ws_f.numel(),
                  metrics, device=dev)
        EV._ms_ssim_into(w_im[None], w_gt[None], 1.0, None, metrics[5], ws_s)
    for _ in range(10):
        kernels()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(args.reps):
        kernels()
    e1.record()
    torch.cuda.synchronize()
    kernel_ms = e0.elapsed_time(e1) / args.reps

    # the reference-style metric path on the same renders
    reference_metrics(im, ds, gt_im, gt_d, args.sil_thres, True)          # warm-up
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(args.ref_frames):
        ref = reference_metrics(im, ds, gt_im, gt_d, args.sil_thres, True)
    torch.cuda.synchronize()
    ref_ms = (time.perf_counter() - t0) * 1e3 / args.ref_frames
    print(json.dumps(dict(
        gpu=gpu_info(), width=W, height=H, gaussians=sc.P, frames=T,
        evaluate_frames_per_s=round(T / wall, 2), evaluate_wall_s=round(wall, 3),
        metric_kernels_ms_per_frame=round(kernel_ms, 4), reference_metrics_ms_per_frame=round(ref_ms, 2),
        cpu_threads=torch.get_num_threads(), psnr=round(out["psnr"], 4), ms_ssim=round(out["ms_ssim"], 6),
        depth_rmse=round(out["depth_rmse"], 6), ate=out["ate"],
        frame1_kernel_vs_reference_style=dict(psnr=[metrics[0].item(), float(ref[0])],
                                              ms_ssim=[metrics[5].item(), float(ref[1])]))))


if __name__ == "__main__":
    main()
