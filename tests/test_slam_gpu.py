"""BASELINE configs 4/5 stand-in (the datasets are not available offline): a slim SplaTAM-style SLAM run --
tracking every frame, keyframe mapping -- over a synthetic RGB-D sequence, with this repo's fused path, its plain
operator path, and the unmodified reference extension (its run is stored in tests/golden/reference/loops.npz).
End metrics (ATE-RMSE, PSNR) must agree."""
import os

import numpy as np
import pytest
import torch

import scenes
from util import GOLDEN

pytestmark = pytest.mark.gpu


def _sequence(dev, Settings, T=9):
    from splatam_b200 import slam
    sc = scenes.room(seed=31, P=30_000, cam=dict(w=320, h=192, fx=160.0, fy=160.0, cx=159.5, cy=95.5))
    cam = sc.settings(Settings, dev)
    gt = sc.splatam_params()
    gt = {k: v.to(dev) for k, v in gt.items()}
    rots, trans = slam.look_trajectory(T, dev)
    g = torch.Generator().manual_seed(5)
    init = dict(gt)
    init["rgb_colors"] = (gt["rgb_colors"] + 0.08 * torch.randn(gt["rgb_colors"].shape, generator=g).to(dev)).clamp(0, 1)
    init["log_scales"] = gt["log_scales"] + 0.05 * torch.randn(gt["log_scales"].shape, generator=g).to(dev)
    return sc, cam, gt, init, rots, trans


def _frames(dev, Settings):
    import splatam_b200 as S
    from splatam_b200 import slam
    sc, cam, gt, init, rots_gt, trans_gt = _sequence(dev, S.GaussianRasterizationSettings)
    frames = [slam.render_frame(gt, rots_gt, trans_gt, t, cam) for t in range(rots_gt.shape[-1])]
    cam = sc.settings(Settings, dev)
    return cam, [dict(f, cam=cam) for f in frames], init, rots_gt, trans_gt


def reference_run(ref, dev):
    """The slim SLAM run over the reference extension `ref` (stored by tests/golden/make_golden_reference.py)."""
    from splatam_b200 import slam
    cam, frames, init, rots_gt, trans_gt = _frames(dev, ref.GaussianRasterizationSettings)
    render = lambda settings, **rv: ref.GaussianRasterizer(raster_settings=settings)(**rv)
    out = slam.run_slam(init, frames, cam, render=render, fused=False)
    return dict(ate=slam.ate_rmse(out["rots"], out["trans"], rots_gt, trans_gt), psnr=out["psnr"])


def test_slim_slam_ate_and_psnr_match_reference(cuda_device):
    import splatam_b200 as S
    from splatam_b200 import slam
    dev = cuda_device
    cam, frames, init, rots_gt, trans_gt = _frames(dev, S.GaussianRasterizationSettings)
    out = {}
    out["fused"] = slam.run_slam(init, frames, cam, fused=True)
    out["plain"] = slam.run_slam(init, frames, cam, fused=False)
    ate = {k: slam.ate_rmse(v["rots"], v["trans"], rots_gt, trans_gt) for k, v in out.items()}
    ps = {k: v["psnr"] for k, v in out.items()}
    z = np.load(os.path.join(GOLDEN, "reference", "loops.npz"))
    ate["reference"], ps["reference"] = float(z["slam_ate"]), float(z["slam_psnr"])
    print("ATE-RMSE [m]", ate, "PSNR [dB]", ps)
    travelled = float(trans_gt[0, :, -1].norm())
    for k in ate:
        assert ate[k] < 0.03 * travelled, (k, ate[k], travelled)       # tracks within 3 % of the path length
        assert ps[k] > 28.0, (k, ps[k])
    # run-to-run spread of ONE implementation is already ~1.3 dB (the reference arm alone gave 32.8 and 34.1 dB on
    # two runs: float-atomic ordering feeds a 160-step optimisation), so the arms are compared at 2 dB
    base = "reference"
    for k in ate:
        assert abs(ps[k] - ps[base]) < 2.0, (k, ps)
        assert abs(ate[k] - ate[base]) < 0.01 * travelled, (k, ate)


def _opaque_sequence(dev, Settings, T=9):
    """Dense, opaque corridor so that the rendered depth behaves like a depth sensor: scenes.room's wall points
    with x and y shrunk 4x (far wall plus all four side walls in view -> geometry that constrains every pose
    axis, and a 4x finer texture), ~10 layers of opacity-0.9 splats behind every pixel; the floating clutter is
    dropped (its soft edges blend depths -- "flying pixels" -- and bias tracking).  depth = alpha-weighted depth /
    silhouette, 0 where nothing is seen."""
    from splatam_b200 import slam
    sc = scenes.room(seed=32, P=200_000, cam=dict(w=320, h=192, fx=160.0, fy=160.0, cx=159.5, cy=95.5))
    cam = sc.settings(Settings, dev)
    walls = int(0.85 * sc.P)             # scenes.room lists the wall points first
    means = sc.means3D.clone()
    means[:, :2] *= 0.25
    colors = 0.5 + 0.5 * torch.sin(means * 40.0 + torch.tensor([0.0, 2.0, 4.0]))   # ~17 px wavelength at the far wall
    gt = dict(means3D=means, rgb_colors=colors, unnorm_rotations=sc.rotations,
              logit_opacities=torch.logit(sc.opacities.clamp(0.02, 0.98)), log_scales=torch.log(1.5 * sc.scales[:, :1]))
    gt = {k: v[:walls].to(dev).contiguous() for k, v in gt.items()}
    rots, trans = slam.look_trajectory(T, dev)
    frames = [slam.render_frame(gt, rots, trans, t, cam) for t in range(T)]
    for f in frames:
        f["depth"] = torch.where(f["sil"] > 0.9, f["depth"] / f["sil"].clamp(min=1e-6), torch.zeros_like(f["depth"]))
    return cam, frames, rots, trans


def test_full_loop_from_rgbd_only(cuda_device, tmp_path):
    """SplaTAM's whole loop from RGB-D frames alone: map initialised by back-projecting frame 0 and mapped, every
    frame tracked, every second frame grows the map from its silhouette holes (add_new_gaussians), selects its
    mapping window by re-projection overlap, maps with pruning, and checkpoints params<t>.npz; the final params.npz
    exports to PLY."""
    import splatam_b200 as S
    from splatam_b200 import formats, slam
    dev = cuda_device
    cam, frames, rots_gt, trans_gt = _opaque_sequence(dev, S.GaussianRasterizationSettings)
    K = torch.tensor([[160.0, 0, 159.5], [0, 160.0, 95.5], [0, 0, 1]])
    assert float((frames[0]["depth"] > 0).float().mean()) > 0.95
    init, radius = slam.initialize_map(frames[0], K)
    P0 = init["means3D"].shape[0]
    assert 0.95 * 320 * 192 < P0 <= 320 * 192
    prune = dict(start_after=0, remove_big_after=0, stop_after=20, prune_every=4, removal_opacity_threshold=0.005,
                 final_removal_opacity_threshold=0.005, reset_opacities=False, reset_opacities_every=500)
    torch.manual_seed(3); np.random.seed(3)
    out = slam.run_slam(init, frames, cam, fused=True, intrinsics=K, add_new_gaussians=True, sil_thres=0.5,
                        prune_dict=prune, scene_radius=radius, select_keyframes=True, window=4, mapping_iters=12,
                        first_frame_iters=60, tracking_iters=40, checkpoint_dir=str(tmp_path))
    ate = slam.ate_rmse(out["rots"], out["trans"], rots_gt, trans_gt)
    travelled = float(trans_gt[0, :, -1].norm())
    print("full loop: ATE-RMSE [m]", ate, "PSNR [dB]", out["psnr"], "Gaussians per mapped frame", out["counts"])
    assert ate < 0.05 * travelled, (ate, travelled)
    assert out["psnr"] > 19.0, out["psnr"]        # 12 mapping iterations per keyframe on a ~17-px-wavelength texture
    assert out["counts"][-1] != P0                      # the map was edited (grown by new views and/or pruned)
    ck = formats.load_params(str(tmp_path / "params.npz"))
    assert ck["means3D"].shape == (out["counts"][-1], 3) and ck["cam_trans"].shape == (1, 3, 9)
    assert (tmp_path / "params8.npz").exists()
    ply = formats.export_ply(str(tmp_path / "params.npz"))
    assert formats.load_ply(ply)["means3D"].shape == ck["means3D"].shape
