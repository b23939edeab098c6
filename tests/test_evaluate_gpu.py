"""GPU: the metric kernels of csrc/eval_metrics.cu and splatam_b200.evaluate against the float64 oracle
(oracle/metrics_torch.py), against the reference's own final `eval` (tests/golden/eval/ref_eval.npz), and end to end
on the SLAM test sequence over the fused and the plain render paths.

MS-SSIM bound per (image, channel): max(1e-5, 2 x the error of the float32 restatement of the same definition against
float64 on the same input, both on the CPU) -- the kernel has to be at least as close to the definition as a float32
PyTorch implementation of it."""
import os

import numpy as np
import pytest
import torch

import scenes
from util import GOLDEN, load

pytestmark = pytest.mark.gpu


def ms_ssim_bound(x, y):
    """[N,C] float64 tolerance of the kernel on CPU images x, y (see the module docstring), and the float64 values."""
    from oracle import metrics_torch as O
    ref = O.ms_ssim(x, y, size_average=False)
    f32 = O.ms_ssim(x.float(), y.float(), size_average=False, dtype=torch.float32).double()
    return torch.clamp(2 * (f32 - ref).abs(), min=1e-5), ref


def _pair(kind, N, C, H, W, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.rand(N, C, H, W, generator=g)
    if kind == "random":
        y = torch.rand(N, C, H, W, generator=g)
    elif kind == "correlated":
        y = (x + 0.1 * torch.randn(N, C, H, W, generator=g)).clamp(0, 1.2)
    elif kind == "inverted":              # y = 1 - x: negative cs on the fine levels, relu drives them to 0
        y = 1 - x
    elif kind == "constant":
        x, y = torch.full((N, C, H, W), 0.3), torch.full((N, C, H, W), 0.7)
    elif kind == "smooth":               # correlated low-frequency content, the regime of rendered frames
        yy, xx = torch.meshgrid(torch.arange(H, dtype=torch.float32), torch.arange(W, dtype=torch.float32), indexing="ij")
        x = 0.5 + 0.3 * torch.sin(xx / 17.0 + yy / 23.0).expand(N, C, H, W) + 0.02 * x
        y = x + 0.03 * torch.randn(N, C, H, W, generator=g)
    return x, y


CASES = [("random", 1, 3, 171, 199), ("correlated", 1, 3, 171, 199), ("inverted", 1, 3, 171, 199),
         ("constant", 1, 3, 171, 199), ("correlated", 2, 3, 161, 161), ("random", 2, 1, 192, 320),
         ("correlated", 1, 1, 192, 320), ("smooth", 1, 3, 680, 1200), ("correlated", 1, 3, 680, 1200)]


@pytest.mark.parametrize("kind,N,C,H,W", CASES)
def test_ms_ssim_matches_float64_definition(cuda_device, kind, N, C, H, W):
    from splatam_b200.evaluate import ms_ssim
    x, y = _pair(kind, N, C, H, W, seed=H + W + N + C)
    bound, ref = ms_ssim_bound(x, y)
    got = ms_ssim(x.to(cuda_device), y.to(cuda_device), size_average=False).cpu()
    assert got.shape == (N, C) and got.dtype == torch.float64
    err = (got - ref).abs()
    assert (err <= bound).all(), (err.max().item(), bound.min().item())
    mean = ms_ssim(x.to(cuda_device), y.to(cuda_device)).item()
    assert abs(mean - ref.mean().item()) <= bound.max().item()
    if kind == "inverted":
        assert (ref < 0.2).all()           # cs of the finest levels clamps to 0 and dominates the product


def test_ms_ssim_non_contiguous_inputs(cuda_device):
    from splatam_b200.evaluate import ms_ssim
    x, y = _pair("correlated", 1, 3, 199, 171, seed=3)
    xt, yt = x.transpose(-1, -2), y.transpose(-1, -2)             # [1,3,171,199] views, not contiguous
    bound, ref = ms_ssim_bound(xt.contiguous(), yt.contiguous())
    xg, yg = x.to(cuda_device).transpose(-1, -2), y.to(cuda_device).transpose(-1, -2)
    assert not xg.is_contiguous()
    got = ms_ssim(xg, yg, size_average=False).cpu()
    assert ((got - ref).abs() <= bound).all()
    sliced = torch.rand(1, 6, 171, 199, device=cuda_device)[:, ::2]               # channel stride 2
    assert ms_ssim(sliced, sliced).item() == 1.0


def test_identical_images_and_determinism(cuda_device):
    from splatam_b200.evaluate import ms_ssim
    x, y = _pair("correlated", 2, 3, 680, 1200, seed=9)
    x, y = x.to(cuda_device), y.to(cuda_device)
    assert ms_ssim(x, x.clone()).item() == 1.0
    assert torch.equal(ms_ssim(x, x.clone(), size_average=False), torch.ones(2, 3, dtype=torch.float64, device=cuda_device))
    a, b = ms_ssim(x, y, size_average=False), ms_ssim(x, y, size_average=False)
    assert torch.equal(a, b)
    with pytest.raises(Exception, match="smaller image side"):
        ms_ssim(x[..., :160, :], y[..., :160, :])


def _frames_from_case(case, dev):
    frames = []
    w2c0 = torch.linalg.inv(case["dataset"][0][3])
    for t, (color, depth, _, _) in enumerate(case["dataset"]):
        frames.append(dict(id=t, im=(color.permute(2, 0, 1) / 255).to(dev), depth=depth.permute(2, 0, 1).to(dev),
                           w2c=w2c0.to(dev)))
    return frames


@pytest.mark.parametrize("name", ["masked", "unmasked_every3"])
def test_evaluate_matches_reference_eval(cuda_device, tmp_path, name):
    """evaluate over the fixture's preset renders == the reference's eval over the same renders."""
    from splatam_b200.evaluate import evaluate
    gen = load("tests/golden/eval/make_golden_eval.py")
    fx = np.load(os.path.join(GOLDEN, "eval", "ref_eval.npz"))
    dev = cuda_device
    case = gen.eval_case(name)
    params = {k: v.to(dev) for k, v in case["params"].items()}
    renders = {t: (im.to(dev), ds.to(dev)) for t, (im, ds) in case["renders"].items()}
    calls = []

    def render(settings, means3D, colors_precomp, **rv):
        t = gen.frame_from_render_call(params, means3D)
        depth_call = bool((colors_precomp[:, 1] == 1).all())
        calls.append((t, depth_call))
        return renders[t][1 if depth_call else 0].clone(), torch.zeros(means3D.shape[0], dtype=torch.int32), None
    gt_w2c = [torch.linalg.inv(pose) for _, _, _, pose in case["dataset"]]
    out = evaluate(params, _frames_from_case(case, dev), None, case["sil_thres"], case["mapping_iters"],
                   case["add_new_gaussians"], eval_every=case["eval_every"], gt_w2c=gt_w2c, fused=False, render=render,
                   out_dir=str(tmp_path))
    ids = fx[name + "_ids"].tolist()
    assert out["frame_ids"] == ids and sorted(set(t for t, _ in calls)) == ids
    assert np.abs(out["psnr_per_frame"] - fx[name + "_psnr"]).max() < 1e-4
    for key, ref in (("depth_rmse_per_frame", "rmse"), ("depth_l1_per_frame", "l1")):
        assert np.abs(out[key] / fx[name + "_" + ref] - 1).max() < 1e-5, key
    assert (out["valid_pixels"] == fx[name + "_n_valid"]).all() and (out["mask_pixels"] == fx[name + "_n_mask"]).all()
    assert abs(out["ate"] - float(fx[name + "_ate"])) < 1e-6 * float(fx[name + "_ate"])
    assert out["lpips"] is None
    from oracle import metrics_torch as O
    for k, t in enumerate(ids):
        im, depth_sil = case["renders"][t]
        color, depth = case["dataset"][t][:2]
        m = O.frame_metrics(im, depth_sil, color.permute(2, 0, 1) / 255, depth.permute(2, 0, 1), case["sil_thres"],
                            case["mapping_iters"] == 0 and not case["add_new_gaussians"])
        bound, _ = ms_ssim_bound(m["weighted_im"][None], m["weighted_gt"][None])
        assert abs(out["ms_ssim_per_frame"][k] - fx[name + "_ssim"][k]) <= bound.max().item(), t
    for fname, key in (("psnr", "psnr_per_frame"), ("ssim", "ms_ssim_per_frame")):
        assert np.array_equal(np.atleast_1d(np.loadtxt(tmp_path / (fname + ".txt"))), out[key])
    assert abs(out["psnr"] - fx[name + "_psnr"].mean()) < 1e-4


def _slam_sequence(dev, T=9):
    """test_slam_gpu.py's 320x192 sequence: ground-truth frames of a room scene along slam.look_trajectory, a map
    with perturbed colours and scales, and a trajectory estimate with small pose errors."""
    import splatam_b200 as S
    from splatam_b200 import slam
    sc = scenes.room(seed=31, P=30_000, cam=dict(w=320, h=192, fx=160.0, fy=160.0, cx=159.5, cy=95.5))
    cam = sc.settings(S.GaussianRasterizationSettings, dev)
    gt = sc.splatam_params()
    gt = {k: v.to(dev) for k, v in gt.items()}
    rots, trans = slam.look_trajectory(T, dev)
    frames = [slam.render_frame(gt, rots, trans, t, cam) for t in range(T)]
    g = torch.Generator().manual_seed(5)
    est = dict(gt)
    est["rgb_colors"] = (gt["rgb_colors"] + 0.08 * torch.randn(gt["rgb_colors"].shape, generator=g).to(dev)).clamp(0, 1)
    est["log_scales"] = gt["log_scales"] + 0.05 * torch.randn(gt["log_scales"].shape, generator=g).to(dev)
    est["cam_unnorm_rots"] = rots + 0.002 * torch.randn(rots.shape, generator=g).to(dev)
    est["cam_trans"] = trans + 0.005 * torch.randn(trans.shape, generator=g).to(dev)
    est["cam_unnorm_rots"][..., 0], est["cam_trans"][..., 0] = rots[..., 0], trans[..., 0]
    return cam, frames, est, slam.w2c_list(rots, trans)


def test_evaluate_end_to_end_fused_and_plain(cuda_device):
    from oracle import metrics_torch as O
    from splatam_b200 import mapping as M
    from splatam_b200.evaluate import evaluate
    dev = cuda_device
    cam, frames, params, gt_w2c = _slam_sequence(dev)
    before = {k: v.clone() for k, v in params.items()}
    for mapping_iters, add_new in ((0, False), (40, True)):
        res = {}
        for fused in (True, False):
            out = evaluate(params, frames, cam, 0.5, mapping_iters, add_new, eval_every=2, gt_w2c=gt_w2c, fused=fused)
            assert out["frame_ids"] == [0, 1, 3, 5, 7]
            for k, t in enumerate(out["frame_ids"]):
                with torch.no_grad():
                    im, ds, _, _ = M._render_pair(params, dict(frames[t], cam=cam), M.default_render, fused, False)
                m = O.frame_metrics(im.cpu(), ds.cpu(), frames[t]["im"].cpu(), frames[t]["depth"].cpu(), 0.5,
                                    mapping_iters == 0 and not add_new)
                assert abs(out["psnr_per_frame"][k] - float(m["psnr"])) < 1e-4, (fused, t)
                assert abs(out["depth_rmse_per_frame"][k] / float(m["depth_rmse"]) - 1) < 1e-5
                assert abs(out["depth_l1_per_frame"][k] / float(m["depth_l1"]) - 1) < 1e-5
                assert out["mask_pixels"][k] == int(m["n_mask"])
                bound, ref = ms_ssim_bound(m["weighted_im"][None], m["weighted_gt"][None])
                assert abs(out["ms_ssim_per_frame"][k] - ref.mean().item()) <= bound.max().item(), (fused, t)
            res[fused] = out
        print("evaluate (mapping_iters=%d): PSNR %.3f dB, MS-SSIM %.5f, depth RMSE %.5f m, ATE %.5f m"
              % (mapping_iters, res[True]["psnr"], res[True]["ms_ssim"], res[True]["depth_rmse"], res[True]["ate"]))
        assert np.abs(res[True]["psnr_per_frame"] - res[False]["psnr_per_frame"]).max() < 1e-4
        assert np.abs(res[True]["ms_ssim_per_frame"] - res[False]["ms_ssim_per_frame"]).max() < 1e-5
        assert res[True]["ate"] == res[False]["ate"] and res[True]["ate"] > 0
        assert 15.0 < res[True]["psnr"] < 60.0 and 0.5 < res[True]["ms_ssim"] < 1.0
    for k, v in params.items():
        assert torch.equal(v, before[k]), k
