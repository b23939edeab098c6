"""Host logic of the SLAM harness (splatam_b200/slam.py) on CPU: tracking every frame, overlap keyframe selection,
mapping with pruning, checkpoints -- with the float32 brute-force composite from oracle/ standing in for the
rasterizer (the product operator has no CPU fallback; the GPU runs are tests/test_slam_gpu.py)."""
import numpy as np
import torch

import scenes
from util import cpu_render
from splatam_b200 import formats, slam


def test_slam_loop_host_logic(tmp_path):
    import splatam_b200 as S
    torch.set_num_threads(4)
    sc = scenes.config1(seed=8, P=160, w=48, h=32)
    cam = sc.settings(S.GaussianRasterizationSettings, "cpu")
    gt = sc.splatam_params(opacity_clamp=(0.05, 0.95))
    T = 4
    rots, trans = slam.look_trajectory(T, "cpu", step=(0.004, -0.002, 0.003), rot_step=(0.001, -0.001, 0.0005))
    frames = [slam.render_frame(gt, rots, trans, t, cam, render=cpu_render) for t in range(T)]
    assert frames[0]["im"].shape == (3, 32, 48) and frames[0]["depth"].shape == (1, 32, 48) and "sil" in frames[0]
    K = torch.tensor([[sc.fx, 0, sc.cx], [0, sc.fy, sc.cy], [0, 0, 1]])
    prune = dict(start_after=0, remove_big_after=0, stop_after=20, prune_every=1, removal_opacity_threshold=0.06,
                 final_removal_opacity_threshold=0.06, reset_opacities=False, reset_opacities_every=500)
    torch.manual_seed(1); np.random.seed(1)
    out = slam.run_slam(gt, frames, cam, render=cpu_render, fused=False, tracking_iters=3, mapping_iters=2,
                        keyframe_every=2, window=3, intrinsics=K, prune_dict=prune, scene_radius=10.0,
                        select_keyframes=True, checkpoint_dir=str(tmp_path))
    assert out["rots"].shape == (1, 4, T) and out["trans"].shape == (1, 3, T)
    assert torch.isfinite(out["rots"]).all() and torch.isfinite(out["trans"]).all() and np.isfinite(out["psnr"])
    assert out["counts"][0] == 160 and out["counts"][-1] <= 160          # pruning can only shrink this map
    ate = slam.ate_rmse(out["rots"], out["trans"], rots, trans)
    assert ate < float(trans[0, :, -1].norm()) * 1.5                       # 3 tracking iterations: sane, not converged
    ck = formats.load_params(str(tmp_path / "params.npz"))
    assert ck["means3D"].shape[0] == out["counts"][-1] and ck["cam_unnorm_rots"].shape == (1, 4, T)
    assert (tmp_path / "params2.npz").exists()
    assert slam.ate_rmse(rots, trans, rots, trans) == 0.0 and slam.psnr(frames[0]["im"], frames[0]["im"] * 0 + 0.5) > 0


def test_slam_loop_with_gradient_densification(tmp_path):
    """The reference's optional densification branch inside the mapping iterations (splatam.py:863-864): the map is
    cloned / split by the 2D-mean gradient statistic and pruned, the loop carries on with the resized map."""
    import splatam_b200 as S
    torch.set_num_threads(4)
    sc = scenes.config1(seed=8, P=120, w=48, h=32)
    cam = sc.settings(S.GaussianRasterizationSettings, "cpu")
    gt = sc.splatam_params(opacity_clamp=(0.05, 0.95))
    T = 3
    rots, trans = slam.look_trajectory(T, "cpu", step=(0.004, -0.002, 0.003), rot_step=(0.001, -0.001, 0.0005))
    frames = [slam.render_frame(gt, rots, trans, t, cam, render=cpu_render) for t in range(T)]
    init = dict(gt)
    init["rgb_colors"] = (gt["rgb_colors"] + 0.2).clamp(0, 1)          # a wrong map: non-zero gradients everywhere
    dd = dict(start_after=0, remove_big_after=0, stop_after=10, densify_every=1, grad_thresh=1e-7, num_to_split_into=2,
              removal_opacity_threshold=0.02, final_removal_opacity_threshold=0.02, reset_opacities=False,
              reset_opacities_every=100)
    torch.manual_seed(2); np.random.seed(2)
    out = slam.run_slam(init, frames, cam, render=cpu_render, fused=False, tracking_iters=2, mapping_iters=2,
                        keyframe_every=1, window=2, scene_radius=0.5, densify_dict=dd)
    assert out["counts"][-1] != 120 and torch.isfinite(out["gauss"]["means3D"]).all() and np.isfinite(out["psnr"])
    assert out["gauss"]["means3D"].shape[0] == out["counts"][-1] == out["gauss"]["logit_opacities"].shape[0]


def test_scene_splatam_params_equals_the_inline_map():
    """Scene.splatam_params against the statement the tests and tools wrote out before it: both opacity clamps they
    use and none, isotropic and anisotropic scales.  config1's opacities reach past both clamps, and half of its
    Gaussians are anisotropic."""
    sc = scenes.config1(seed=8, P=160, w=48, h=32)
    for clamp in ((0.02, 0.98), (0.05, 0.95), None):
        op = sc.opacities if clamp is None else sc.opacities.clamp(*clamp)
        assert clamp is None or not torch.equal(op, sc.opacities), clamp     # the clamp changes some opacity
        for iso in (True, False):
            ref = dict(means3D=sc.means3D, rgb_colors=sc.colors, unnorm_rotations=sc.rotations,
                       logit_opacities=torch.logit(op), log_scales=torch.log(sc.scales[:, :1] if iso else sc.scales))
            got = sc.splatam_params(opacity_clamp=clamp, isotropic=iso)
            assert list(got) == list(ref) and all(torch.equal(got[k], ref[k]) for k in ref), (clamp, iso)
    assert not torch.equal(sc.scales[:, :1].expand(-1, 3), sc.scales)       # the anisotropic case is one
