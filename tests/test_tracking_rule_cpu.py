"""CPU: the depth-loss rule of mapping.track_frame's eager loop (the reference's use_depth_loss_thres,
R/scripts/splatam.py:727-738), bit for bit, with the float32 brute-force composite from oracle/ standing in for the
rasterizer (deterministic, unlike the GPU backward's float atomics): a threshold that is always met gives the run of
num_iters iterations, a threshold of 0 the run of 2 * num_iters, and a NaN threshold, which no depth sum is below,
continues as the reference's `losses['depth'] < thres` test does."""
import torch

import scenes
from util import cpu_render
from splatam_b200 import mapping as M, slam

N = 4


def _problem():
    import splatam_b200 as S
    torch.set_num_threads(4)
    sc = scenes.config1(seed=8, P=160, w=48, h=32)
    cam = sc.settings(S.GaussianRasterizationSettings, "cpu")
    gauss = sc.splatam_params(opacity_clamp=(0.05, 0.95))
    rots, trans = slam.look_trajectory(2, "cpu", step=(0.02, -0.01, 0.015), rot_step=(0.01, -0.01, 0.005))
    return gauss, slam.render_frame(gauss, rots, trans, 1, cam, render=cpu_render)


def _track(gauss, frame, num_iters, **kw):
    rots = torch.zeros(1, 4, 2); rots[:, 0] = 1.0
    p = dict(gauss, cam_unnorm_rots=rots, cam_trans=torch.zeros(1, 3, 2))
    losses = M.track_frame(p, frame, render=cpu_render, num_iters=num_iters, fused=False, **kw)
    return losses, p["cam_unnorm_rots"][..., 1].detach().clone(), p["cam_trans"][..., 1].detach().clone()


def _equal(a, b):
    return a[0] == b[0] and torch.equal(a[1], b[1]) and torch.equal(a[2], b[2])


def test_rule_is_bit_equal_to_fixed_iteration_runs():
    gauss, frame = _problem()
    base_n, base_2n = _track(gauss, frame, N), _track(gauss, frame, 2 * N)
    assert not _equal(base_n, base_2n)
    assert _equal(_track(gauss, frame, N, depth_loss_thres=float("inf")), base_n)
    assert _equal(_track(gauss, frame, N, depth_loss_thres=0.0), base_2n)
    # the rule looks at the unweighted depth sum of iteration N, evaluated before its Adam step
    keep = {}
    p = dict(gauss, cam_unnorm_rots=torch.zeros(1, 4, 2), cam_trans=torch.zeros(1, 3, 2))
    p["cam_unnorm_rots"][:, 0] = 1.0
    with torch.no_grad():
        M.tracking_loss(p, frame, cpu_render, keep=keep)
    assert keep["depth"] > 0
    run = _track(gauss, frame, N, depth_loss_thres=float("nan"))          # never below: the reference continues
    assert _equal(run, base_2n)
