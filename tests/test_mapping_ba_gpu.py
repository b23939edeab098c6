"""GPU tests of keyframe-pose refinement in the mapper's fused path: FusedAdam over the cameras, the single backward of
csrc/prepare.cu giving Gaussian and pose gradients, the captured step with its static pose leaves and scatter into the
pose-gradient table -- against the reference's own do_ba=True loop (tests/golden/ba/ref_ba.npz), eager against graph,
without host synchronisation, and the poses converging back to the ones the frames were rendered at."""
import math
import os

import numpy as np
import pytest
import torch

import scenes
from util import GOLDEN, load

pytestmark = pytest.mark.gpu

CAM_LRS = dict(cam_unnorm_rots=0.0004, cam_trans=0.002)       # Replica's tracking rates
FROZEN = dict(means3D=0.0, rgb_colors=0.0, unnorm_rotations=0.0, logit_opacities=0.0, log_scales=0.0)


@pytest.fixture(scope="module")
def gen():
    return load("tests/golden/ba/make_golden_ba.py")


def _rel(a, b):
    return float((a - b).norm() / b.norm().clamp_min(1e-20))


@pytest.mark.parametrize("aniso", [False, True])
def test_fused_mapper_matches_reference_do_ba(gen, aniso, cuda_device):
    """The fused path (prepare kernel with both gradients, fused loss kernels, FusedAdam over map and cameras) with the
    fixture's brute-force rasterizer, against the reference's loop."""
    from splatam_b200 import mapping as M
    from splatam_b200.formats import GAUSSIAN_KEYS
    import splatam_b200 as S
    dev = cuda_device
    fx = np.load(os.path.join(GOLDEN, "ba", "ref_ba.npz"))
    tag = "aniso_" if aniso else "iso_"
    t = lambda a: torch.from_numpy(np.array(a)).to(dev)
    cam = scenes.config1(seed=8, P=160, w=48, h=32).settings(S.GaussianRasterizationSettings, dev)
    frames = [dict(id=k, cam=cam, w2c=torch.eye(4, device=dev), im=t(fx[tag + "im%d" % k]),
                   depth=t(fx[tag + "depth%d" % k])) for k in range(gen.T)]
    mapper = M.ShardedMapper({k: t(fx[tag + "in_" + k]) for k in GAUSSIAN_KEYS}, t(fx[tag + "in_cam_unnorm_rots"]),
                             t(fx[tag + "in_cam_trans"]), lrs=gen.lrs(aniso), render=gen.render, fused=True)
    mapper.schedule = lambda n: [0]
    for it, k in enumerate(fx["iter_ids"]):
        if it == int(fx["prune_iter"]):
            mapper.g.zero_grad()
            loss, _ = mapper.accumulate(frames[int(k)])
            grads = [mapper.cam[n].grad.clone() for n in M.CAM_KEYS]
            mapper.prune_gaussians(it, gen.PRUNE, float(fx[tag + "scene_radius"]))
            mapper._cam_step()
        else:
            loss, _, _ = mapper.step([frames[int(k)]])
            grads = [mapper.cam[n].grad for n in M.CAM_KEYS]
        ref = float(fx[tag + "loss"][it])
        assert abs(float(loss) - ref) < 3e-6 * max(1.0, abs(ref)), (it, float(loss), ref)
        for n, g in zip(M.CAM_KEYS, grads):
            assert _rel(g, t(fx[tag + "grad_%s_%d" % (n, it)])) < 2e-4, (it, n)
        p = mapper.params()
        for key in gen.KEYS:
            a, b = p[key].detach(), t(fx[tag + "out_%s_%d" % (key, it)])
            assert a.shape == b.shape and torch.allclose(a, b, rtol=1e-5, atol=2e-6), \
                (it, key, float((a - b).abs().max()))


def _scene(dev, T=3, seed=3):
    """A view-filling map, T frames rendered from it at known poses, and the same poses perturbed by 1 cm / 0.3 deg."""
    import splatam_b200 as S
    from splatam_b200 import mapping as M, slam
    sc = scenes.view_filling(seed=31, cam=dict(w=320, h=192, fx=160.0, fy=160.0, cx=159.5, cy=95.5), stride=1,
                             margin=16)
    cam = sc.settings(S.GaussianRasterizationSettings, dev)
    gauss = sc.splatam_params()
    gauss = {k: v.clone().to(dev) for k, v in gauss.items()}
    rots, trans = slam.look_trajectory(T, dev, step=(0.01, -0.005, 0.008), rot_step=(0.002, -0.002, 0.001))
    frames = [slam.render_frame(gauss, rots, trans, t, cam) for t in range(T)]
    g = torch.Generator().manual_seed(seed)
    d = torch.randn(1, 3, T, generator=g)
    ax = torch.randn(1, 3, T, generator=g)
    pr, pt = rots.clone(), trans.clone()
    pr[:, 1:] += (ax / ax.norm(dim=1, keepdim=True) * math.radians(0.3) / 2).to(dev)
    pt += (0.01 * d / d.norm(dim=1, keepdim=True)).to(dev)
    return gauss, frames, (rots, trans), (pr, pt), M


def _trans_err(mapper, truth):
    return float((mapper.cam["cam_trans"].detach() - truth[1]).norm(dim=1).mean())


def _rot_err(mapper, truth):
    """Mean rotation angle (rad) between the mapper's and the true camera rotations, from the relative quaternion in
    float64 (atan2 keeps sub-degree angles accurate where acos of a dot product near 1 would not)."""
    a = torch.nn.functional.normalize(mapper.cam["cam_unnorm_rots"].detach().double(), dim=1)[0].T      # [T,4]
    b = torch.nn.functional.normalize(truth[0].double(), dim=1)[0].T
    w = (a * b).sum(1)                                                   # real part of conj(b) * a
    v = b[:, :1] * a[:, 1:] - a[:, :1] * b[:, 1:] - torch.linalg.cross(b[:, 1:], a[:, 1:], dim=1)
    return float((2 * torch.atan2(v.norm(dim=1), w.abs())).mean())


@pytest.mark.parametrize("graph", [False, True])
def test_poses_converge_back_to_the_rendered_ones(graph, cuda_device):
    """60 mapping steps over three keyframes with the Gaussians frozen and the cameras at Replica's tracking rates: the
    mean translation error and the mean rotation error each fall at least by half."""
    gauss, frames, truth, (pr, pt), M = _scene(cuda_device)
    mapper = M.ShardedMapper(gauss, pr, pt, lrs=dict(FROZEN, **CAM_LRS), seed=1)
    if graph:
        mapper.enable_graph(frames)
    e0, r0 = _trans_err(mapper, truth), _rot_err(mapper, truth)
    assert 0.005 < e0 and math.radians(0.1) < r0
    for _ in range(60):
        mapper.step(frames)
    mapper.poll_overflow(frames, block=True)
    assert mapper.effective_steps()[1] == 0
    e1, r1 = _trans_err(mapper, truth), _rot_err(mapper, truth)
    assert e1 < 0.5 * e0, (e0, e1)
    assert r1 < 0.5 * r0, (r0, r1)


def test_graph_matches_eager_and_an_overflowed_step_moves_no_pose(cuda_device):
    """20 steps eager and 20 replayed from the captured step (same schedule) end at the same poses and map to float
    tolerance; a capture with a far too small capacity overflows its first step, which moves neither the map nor the
    poses, and the re-captured graph then continues."""
    gauss, frames, truth, (pr, pt), M = _scene(cuda_device)
    lrs = dict(M.ShardedMapper.DEFAULT_LRS, **CAM_LRS)
    eager = M.ShardedMapper(gauss, pr, pt, lrs=lrs, seed=2)
    graphed = M.ShardedMapper(gauss, pr, pt, lrs=lrs, seed=2)
    graphed.enable_graph(frames)
    for _ in range(20):
        eager.step(frames)
        graphed.step(frames)
    graphed.poll_overflow(frames, block=True)
    assert graphed.effective_steps() == (20, 0)
    for k in M.CAM_KEYS:
        a, b = eager.cam[k].detach(), graphed.cam[k].detach()
        assert torch.allclose(a, b, rtol=0, atol=2e-5), (k, float((a - b).abs().max()))
    assert not torch.equal(eager.cam["cam_trans"].detach(), pt)
    assert _rel(graphed.g.flat.detach(), eager.g.flat.detach()) < 1e-4

    tiny = M.ShardedMapper(gauss, pr, pt, lrs=lrs, seed=2)
    tiny.enable_graph(frames, capacity=1024)
    cams0 = {k: v.detach().clone() for k, v in tiny.cam.items()}
    flat0 = tiny.g.flat.detach().clone()
    tiny.step(frames)
    torch.cuda.synchronize(cuda_device)
    for k in M.CAM_KEYS:
        assert torch.equal(tiny.cam[k].detach(), cams0[k]), k
    assert torch.equal(tiny.g.flat.detach(), flat0)
    assert tiny.poll_overflow(frames, block=True) and tiny.overflow_events == 1
    tiny.step(frames)
    tiny.poll_overflow(frames, block=True)
    assert tiny.effective_steps() == (1, 1)
    assert not torch.equal(tiny.cam["cam_trans"].detach(), cams0["cam_trans"])


def test_captured_step_with_refinement_is_sync_free(cuda_device):
    gauss, frames, truth, (pr, pt), M = _scene(cuda_device)
    mapper = M.ShardedMapper(gauss, pr, pt, lrs=dict(M.ShardedMapper.DEFAULT_LRS, **CAM_LRS), seed=4)
    mapper.enable_graph(frames)
    mapper.step(frames)                     # first step: creates the optimizers' device clocks
    torch.cuda.synchronize(cuda_device)
    torch.cuda.set_sync_debug_mode("error")
    try:
        for _ in range(5):
            mapper.step(frames)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    mapper.poll_overflow(frames, block=True)
    assert mapper.effective_steps() == (6, 0)


def test_fused_pose_update_invalidates_the_pose_cache(cuda_device):
    """FusedAdam writes the camera buffer through a raw pointer; the pose cache must still never serve the pose from
    before the update (render_frame / evaluation / the captured step's static pose read it)."""
    gauss, frames, truth, (pr, pt), M = _scene(cuda_device)
    mapper = M.ShardedMapper(gauss, pr, pt, lrs=dict(M.ShardedMapper.DEFAULT_LRS, **CAM_LRS), seed=4)
    mapper.schedule = lambda n: [1]
    stale = [v.clone() for v in M.fused_pose_cached(mapper.params(), 1)]
    mapper.step(frames)
    now = M.fused_pose_cached(mapper.params(), 1)
    fresh = M.pose_matrices({k: v.detach() for k, v in mapper.cam.items()}, 1)
    assert not torch.equal(now[0], stale[0])
    for x, y in zip(now, fresh):
        assert torch.equal(x, y)


def test_run_slam_with_refinement_graph_and_eager(cuda_device, tmp_path):
    """run_slam's mapping_cam_lrs on the fused path, eager and graph: the run completes, the poses differ from a run
    without refinement, and each keyframe stores its pose once, after its own mapping phase (checkpoint k holds column k
    as it was then), and keeps it while later phases move the column."""
    from splatam_b200 import formats, slam
    gauss, frames, truth, _, M = _scene(cuda_device, T=4)
    cam = frames[0]["cam"]
    kw = dict(tracking_iters=4, mapping_iters=6, keyframe_every=1, window=3)
    off = slam.run_slam(gauss, frames, cam, **kw)
    for graph in (False, True):
        d = str(tmp_path / ("g" if graph else "e"))
        on = slam.run_slam(gauss, frames, cam, graph=graph, mapping_cam_lrs=(0.0004, 0.002), checkpoint_dir=d,
                           checkpoint_every=1, **kw)
        assert torch.isfinite(on["trans"]).all() and not torch.equal(on["trans"], off["trans"])
        assert on["psnr"] > 20.0
        est = on["keyframe_est_w2c"]
        for k in range(1, len(frames)):
            ck = formats.load_checkpoint(d, k, cuda_device)
            assert torch.equal(est[k], slam._curr_w2c(ck["cam_unnorm_rots"], ck["cam_trans"], k)), (graph, k)
        final = [slam._curr_w2c(on["rots"], on["trans"], k) for k in range(len(frames))]
        assert any(not torch.equal(est[k], final[k]) for k in range(1, len(frames) - 1))
