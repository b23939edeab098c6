"""GPU: splatam_b200.evaluate.evaluate_nvs against the reference's own `eval_nvs` (tests/golden/eval/ref_eval_nvs.npz)
with the tolerances of test_evaluate_gpu.py, fused against plain rendering at ground-truth poses on an anisotropic map,
and end to end: SplaTAM on the train split of a rendered ReplicaV2-layout sequence on disk, then evaluate_nvs on its
test split."""
import os

import numpy as np
import pytest
import torch

import scenes
from util import GOLDEN, load
from test_evaluate_gpu import ms_ssim_bound

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("name", ["unmasked_every1", "masked_every2", "none_valid"])
def test_evaluate_nvs_matches_reference_eval_nvs(cuda_device, tmp_path, name):
    """evaluate_nvs over the fixture's preset renders == the reference's eval_nvs over the same renders."""
    from oracle import metrics_torch as O
    from splatam_b200.evaluate import evaluate_nvs
    gen = load("tests/golden/eval/make_golden_eval_nvs.py")
    fx = np.load(os.path.join(GOLDEN, "eval", "ref_eval_nvs.npz"))
    dev = cuda_device
    case = gen.nvs_case(name)
    params = {k: v.to(dev) for k, v in case["params"].items()}
    renders = {t: (im.to(dev), ds.to(dev)) for t, (im, ds) in case["renders"].items()}
    gt_w2c = case["gt_w2c"].to(dev)
    w2c0 = torch.linalg.inv(case["dataset"][0][3]).to(dev)
    frames = [dict(id=t, im=(c.permute(2, 0, 1) / 255).to(dev), depth=d.permute(2, 0, 1).to(dev), w2c=w2c0,
                   gt_w2c=gt_w2c[t]) for t, (c, d, _, _) in enumerate(case["dataset"])]
    calls = []

    def render(settings, means3D, colors_precomp, **rv):
        t = gen.frame_from_render_call(gt_w2c, means3D)
        depth_call = bool((colors_precomp[:, 1] == 1).all())
        calls.append(t)
        return renders[t][1 if depth_call else 0].clone(), torch.zeros(means3D.shape[0], dtype=torch.int32), None
    out = evaluate_nvs(params, frames, None, case["sil_thres"], case["mapping_iters"], case["add_new_gaussians"],
                       eval_every=case["eval_every"], fused=False, render=render, out_dir=str(tmp_path))
    ids = fx[name + "_ids"].tolist()
    assert out["frame_ids"] == ids and sorted(set(calls)) == ids
    assert np.abs(out["psnr_per_frame"] - fx[name + "_psnr"]).max() < 1e-4
    for key, ref in (("depth_rmse_per_frame", "rmse"), ("depth_l1_per_frame", "l1")):
        assert np.abs(out[key] / fx[name + "_" + ref] - 1).max() < 1e-5, key
    assert (out["valid_pixels"] == fx[name + "_n_valid"]).all() and (out["mask_pixels"] == fx[name + "_n_mask"]).all()
    assert (out["hole_pixels"] == fx[name + "_holes"]).all()
    assert out["valid_nvs_frames"].dtype == bool and (out["valid_nvs_frames"] == fx[name + "_valid"]).all()
    assert out["lpips"] is None
    use_presence = case["mapping_iters"] == 0 and not case["add_new_gaussians"]
    for k, t in enumerate(ids):
        im, depth_sil = case["renders"][t]
        color, depth = case["dataset"][t][:2]
        m = O.frame_metrics(im, depth_sil, color.permute(2, 0, 1) / 255, depth.permute(2, 0, 1), case["sil_thres"],
                            use_presence)
        bound, _ = ms_ssim_bound(m["weighted_im"][None], m["weighted_gt"][None])
        assert abs(out["ms_ssim_per_frame"][k] - fx[name + "_ssim"][k]) <= bound.max().item(), t
    valid = fx[name + "_valid"]
    if valid.any():
        assert abs(out["psnr"] - fx[name + "_psnr"][valid].mean()) < 1e-4
        assert abs(out["depth_l1"] / fx[name + "_l1"][valid].mean() - 1) < 1e-5
    else:
        assert all(np.isnan(out[k]) for k in ("psnr", "ms_ssim", "depth_rmse", "depth_l1"))
    for fname, key in (("psnr", "psnr_per_frame"), ("ssim", "ms_ssim_per_frame"), ("l1", "depth_l1_per_frame")):
        assert np.array_equal(np.atleast_1d(np.loadtxt(tmp_path / (fname + ".txt"))), out[key])
    assert np.array_equal(np.load(tmp_path / "valid_nvs_frames.npy"), out["valid_nvs_frames"])


def test_fused_and_plain_render_at_the_ground_truth_pose(cuda_device):
    """An anisotropic map seen from held-out poses: both render paths give the same metrics, and equal those of
    `evaluate` with the camera estimate set to the same poses (so the means and rotations follow gt_w2c)."""
    import splatam_b200 as S
    from splatam_b200 import mapping as M, slam
    from splatam_b200.evaluate import evaluate, evaluate_nvs
    dev = cuda_device
    sc = scenes.room(seed=41, P=30_000, cam=dict(w=320, h=192, fx=160.0, fy=160.0, cx=159.5, cy=95.5))
    cam = sc.settings(S.GaussianRasterizationSettings, dev)
    g = torch.Generator().manual_seed(6)
    params = sc.splatam_params(isotropic=False)
    params["log_scales"] = params["log_scales"] + 0.3 * torch.randn(sc.scales.shape, generator=g)
    params = {k: v.to(dev) for k, v in params.items()}
    assert params["log_scales"].shape[1] == 3
    T = 6
    rots, trans = slam.look_trajectory(T, dev, rot_step=(0.02, -0.015, 0.01))
    frames = [slam.render_frame(params, rots, trans, t, cam) for t in range(T)]
    for t, fr in enumerate(frames):
        fr["gt_w2c"] = M.camera_w2c(rots[..., t], trans[..., t])[0]
        fr["im"] = (fr["im"] + 0.03 * torch.randn(fr["im"].shape, generator=g).to(dev)).clamp(0, 1)
    res = {}
    for fused in (True, False):
        res[fused] = evaluate_nvs(params, frames, cam, 0.5, 30, True, fused=fused)
        assert res[fused]["frame_ids"] == [1, 2, 3, 4, 5]
    est = dict(params, cam_unnorm_rots=rots, cam_trans=trans)
    ref = evaluate(est, frames, cam, 0.5, 30, True, fused=False)
    for k in ("psnr_per_frame", "ms_ssim_per_frame", "depth_l1_per_frame"):
        assert np.abs(res[True][k] - res[False][k]).max() < 1e-4, k
        assert np.abs(res[False][k] - ref[k][1:]).max() < 1e-3, k
    assert (res[True]["hole_pixels"] == res[False]["hole_pixels"]).all()
    assert (res[True]["valid_nvs_frames"] == (res[True]["hole_pixels"] * 1000 <= 320 * 192)).all()
    assert 20.0 < res[True]["psnr_per_frame"].min() and res[True]["psnr_per_frame"].max() < 60.0


def _write_replicav2(dst, T, device):
    """A rendered ReplicaV2-layout sequence: scenes.write_replica_sequence's frames, the even ones as the train split
    imap/00 and the odd ones as the held-out test split imap/01 (PNG colour, millimetre depth, traj_w_c.txt)."""
    import shutil
    from PIL import Image
    raw = os.path.join(dst, "raw")
    w2c = scenes.write_replica_sequence(raw, T, device, png_depth_scale=1000.0)
    lines = open(os.path.join(raw, "traj.txt")).read().splitlines()
    for split, ts in (("00", range(0, T, 2)), ("01", range(1, T, 2))):
        base = os.path.join(dst, "room_0", "imap", split)
        os.makedirs(os.path.join(base, "rgb")); os.makedirs(os.path.join(base, "depth"))
        for i, t in enumerate(ts):
            with Image.open(os.path.join(raw, "results", "frame%06d.jpg" % t)) as im:
                im.save(os.path.join(base, "rgb", "rgb_%d.png" % i))
            shutil.copy(os.path.join(raw, "results", "depth%06d.png" % t), os.path.join(base, "depth", "depth_%d.png" % i))
        with open(os.path.join(base, "traj_w_c.txt"), "w") as f:
            f.write("\n".join(lines[t] for t in ts) + "\n")
    return w2c


def test_run_slam_on_train_split_then_evaluate_nvs_on_test_split(tmp_path, cuda_device):
    from splatam_b200 import datasets as D, evaluate, slam
    T = 11                                               # train 0, 2, .., 10; the test views lie between them
    w2c = _write_replicav2(str(tmp_path), T, cuda_device)
    with D.RGBDSequence("replicav2", str(tmp_path), "room_0", device=cuda_device, prefetch=2) as seq:
        assert (seq.height, seq.width) == (680, 1200) and len(seq) == 6
        K = seq.intrinsics.cpu()
        init, radius = slam.initialize_map(seq[0], K)
        prune = dict(start_after=0, remove_big_after=0, stop_after=20, prune_every=20, removal_opacity_threshold=0.005,
                     final_removal_opacity_threshold=0.005, reset_opacities=False, reset_opacities_every=500)
        timing = {}
        out = slam.run_slam(init, seq, seq.cam, seed=3, tracking_iters=20, mapping_iters=10, keyframe_every=5,
                            map_every=1, window=24, sil_thres=0.5, intrinsics=K, add_new_gaussians=True,
                            prune_dict=prune, scene_radius=radius, select_keyframes=True, first_frame_iters=10,
                            tracking_lrs=(0.001, 0.004), depth_loss_thres=0.0, timing=timing)
        assert timing["tracking_iters"] == 2 * 20 * (len(seq) - 1)        # a threshold of 0 is never met
        gauss = out["gauss"]
    with D.RGBDSequence("replicav2", str(tmp_path), "room_0", device=cuda_device, prefetch=2, split="test") as test:
        assert len(test) == 1 + T // 2
        gt = torch.stack([g.cpu().double() for g in test.gt_w2c])
        assert torch.allclose(gt, w2c[[0] + list(range(1, T, 2))], atol=1e-5)
        res = evaluate.evaluate_nvs(gauss, test, test.cam, 0.5, 10, True)
    print("evaluate_nvs: PSNR %.3f dB, MS-SSIM %.5f, depth L1 %.5f m, holes %s"
          % (res["psnr"], res["ms_ssim"], res["depth_l1"], res["hole_pixels"].tolist()))
    assert res["frame_ids"] == [1, 2, 3, 4, 5]
    for k in ("psnr", "ms_ssim", "depth_rmse", "depth_l1"):
        assert np.isfinite(res[k]), (k, res[k])
    assert res["valid_nvs_frames"].all(), res["hole_pixels"]
    assert res["psnr"] > 15.0
