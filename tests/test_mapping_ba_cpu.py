"""CPU: keyframe-pose refinement in the mapper's torch path (ShardedMapper with non-zero camera rates) against the
reference's own get_loss(mapping=True, do_ba=True) + initialize_optimizer + prune_gaussians loop
(tests/golden/ba/ref_ba.npz, written by tests/golden/ba/make_golden_ba.py), and the rules around it: momentum, map
edits, zero rates, the pose cache and exact resume."""
import os

import numpy as np
import pytest
import torch

from util import GOLDEN, load

FIX = os.path.join(GOLDEN, "ba", "ref_ba.npz")


@pytest.fixture(scope="module")
def gen():
    return load("tests/golden/ba/make_golden_ba.py")


@pytest.fixture(scope="module")
def fx():
    return np.load(FIX)


def _t(a):
    return torch.from_numpy(np.array(a))


def _inputs(fx, tag):
    from splatam_b200.formats import GAUSSIAN_KEYS
    gauss = {k: _t(fx[tag + "in_" + k]) for k in GAUSSIAN_KEYS}
    cams = {k: _t(fx[tag + "in_" + k]) for k in ("cam_unnorm_rots", "cam_trans")}
    return gauss, cams


def _frames(gen, fx, tag):
    import scenes
    cam = gen.camera(scenes.config1(seed=8, P=160, w=48, h=32))
    return [dict(id=t, cam=cam, w2c=torch.eye(4), im=_t(fx[tag + "im%d" % t]), depth=_t(fx[tag + "depth%d" % t]))
            for t in range(gen.T)]


def _mapper(gen, fx, tag, aniso, **kw):
    from splatam_b200 import mapping as M
    gauss, cams = _inputs(fx, tag)
    lrs = kw.pop("lrs", gen.lrs(aniso))
    return M.ShardedMapper(gauss, cams["cam_unnorm_rots"], cams["cam_trans"], lrs=lrs, render=gen.render, fused=False,
                           **kw)


def _one(mapper, frame):
    """One mapping step of exactly this keyframe."""
    mapper.schedule = lambda n: [0]
    return mapper.step([frame])


@pytest.mark.parametrize("aniso", [False, True])
def test_torch_mapper_matches_reference_do_ba(gen, fx, aniso):
    """Loss, full camera gradients and all seven tensors after every step equal the reference's; on the prune iteration
    (prune between backward and step, as the reference's loop) the Gaussians take no step and the cameras do."""
    tag = "aniso_" if aniso else "iso_"
    frames = _frames(gen, fx, tag)
    mapper = _mapper(gen, fx, tag, aniso)
    assert mapper.refine_poses
    radius = float(fx[tag + "scene_radius"])
    for it, k in enumerate(fx["iter_ids"]):
        if it == int(fx["prune_iter"]):
            mapper.g.zero_grad()
            loss, _ = mapper.accumulate(frames[int(k)])
            g_rot = mapper.cam["cam_unnorm_rots"].grad.clone()
            g_tr = mapper.cam["cam_trans"].grad.clone()
            mapper.prune_gaussians(it, gen.PRUNE, radius)
            # the pose gradient survives the map edit
            assert torch.equal(mapper.cam["cam_unnorm_rots"].grad, g_rot)
            mapper._cam_step()
            loss = float(loss)
        else:
            loss, _, _ = _one(mapper, frames[int(k)])
            g_rot, g_tr = mapper.cam["cam_unnorm_rots"].grad, mapper.cam["cam_trans"].grad
        ref = float(fx[tag + "loss"][it])
        assert abs(loss - ref) < 2e-6 * max(1.0, abs(ref)), it
        for name, g in (("cam_unnorm_rots", g_rot), ("cam_trans", g_tr)):
            b = _t(fx[tag + "grad_%s_%d" % (name, it)])
            assert float((g - b).norm() / b.norm()) < 1e-5, (it, name)
            # dense with zeros outside the drawn column
            others = [c for c in range(gen.T) if c != int(k)]
            assert torch.count_nonzero(g[..., others]) == 0 and torch.count_nonzero(b[..., others]) == 0
        p = mapper.params()
        for key in gen.KEYS:
            a, b = p[key].detach(), _t(fx[tag + "out_%s_%d" % (key, it)])
            assert a.shape == b.shape, (it, key)
            assert torch.allclose(a, b, rtol=1e-6, atol=1e-6), (it, key, float((a - b).abs().max()))


def test_momentum_moves_a_column_whose_gradient_is_zero(gen, fx):
    """A column refined earlier keeps moving on its Adam momentum while another keyframe is drawn; a column never
    drawn does not move."""
    tag = "iso_"
    frames = _frames(gen, fx, tag)
    mapper = _mapper(gen, fx, tag, False)
    _one(mapper, frames[1])
    before = {k: v.detach().clone() for k, v in mapper.cam.items()}
    _one(mapper, frames[2])
    assert torch.count_nonzero(mapper.cam["cam_trans"].grad[..., 1]) == 0
    for k in mapper.cam:
        assert not torch.equal(mapper.cam[k][..., 1], before[k][..., 1]), k      # momentum of the earlier step
        assert not torch.equal(mapper.cam[k][..., 2], before[k][..., 2]), k      # this step's keyframe
        assert torch.equal(mapper.cam[k][..., 0], before[k][..., 0]), k          # never drawn


def test_prune_and_grow_keep_the_pose_moments(gen, fx):
    tag = "aniso_"
    frames = _frames(gen, fx, tag)
    mapper = _mapper(gen, fx, tag, True)
    _one(mapper, frames[1])
    state = {id(p): {k: v.clone() for k, v in mapper.cam_opt.state[p].items()} for p in mapper.cam.values()}
    opt = mapper.cam_opt
    P = mapper.g.shapes["means3D"][0]
    assert mapper.prune_gaussians(0, dict(gen.PRUNE, start_after=0), float(fx[tag + "scene_radius"])) < P
    mapper.add_gaussians({k: v.detach()[:5].clone() for k, v in mapper.g.params.items()})
    assert mapper.cam_opt is opt
    for p in mapper.cam.values():
        for k, v in state[id(p)].items():
            assert torch.equal(mapper.cam_opt.state[p][k], v), k
        assert p.grad.untyped_storage().data_ptr() == mapper.g.bucket.untyped_storage().data_ptr()   # the new bucket
    mapper.reset_optimizer()
    assert mapper.cam_opt is not opt and not mapper.cam_opt.state


def test_zero_camera_rates_change_nothing(gen, fx):
    """At zero camera rates the cameras stay bit-identical and the Gaussians equal those of a mapper built without the
    camera keys, with no pose table in the bucket."""
    tag = "aniso_"
    frames = _frames(gen, fx, tag)
    base = {k: v for k, v in gen.lrs(True).items() if not k.startswith("cam_")}
    a = _mapper(gen, fx, tag, True, lrs=dict(base, cam_unnorm_rots=0.0, cam_trans=0.0))
    b = _mapper(gen, fx, tag, True, lrs=base)
    assert not a.refine_poses and a.g.bucket.numel() == b.g.bucket.numel() and a.g.pose_grad.numel() == 0
    cams0 = {k: v.clone() for k, v in a.cam.items()}
    for k in (1, 0, 2):
        _one(a, frames[k]); _one(b, frames[k])
    for k in cams0:
        assert torch.equal(a.cam[k], cams0[k])
    for k in a.g.params:
        assert torch.equal(a.g.params[k], b.g.params[k]), k
    a.set_lr("cam_trans", 0.0)
    with pytest.raises(ValueError):
        a.set_lr("cam_trans", 0.001)


def test_pose_cache_never_serves_a_pose_from_before_an_update(gen, fx):
    """fused_pose_cached keys on the camera tensors' version: after a refinement step it returns the new pose."""
    from splatam_b200 import mapping as M
    tag = "iso_"
    frames = _frames(gen, fx, tag)
    mapper = _mapper(gen, fx, tag, False)
    _one(mapper, frames[1])
    stale = [v.clone() for v in M.fused_pose_cached(mapper.params(), 1)]
    _one(mapper, frames[1])
    now = M.fused_pose_cached(mapper.params(), 1)
    fresh = M.pose_matrices({k: v.detach() for k, v in mapper.cam.items()}, 1)
    assert not torch.equal(now[0], stale[0])
    for x, y in zip(now, fresh):
        assert torch.equal(x, y)


def test_set_lr_reaches_the_camera_groups(gen, fx):
    tag = "iso_"
    mapper = _mapper(gen, fx, tag, False)
    mapper.set_lr("cam_trans", 0.01)
    assert mapper.cam_opt.param_groups[1]["lr"] == 0.01 and mapper.lrs["cam_trans"] == 0.01
    mapper.reset_optimizer()
    assert mapper.cam_opt.param_groups[1]["lr"] == 0.01


def test_sync_camera_style_replacement_is_adopted(gen, fx):
    """Camera tensors a caller puts into `cam` (tracking, sync_camera) are copied into the mapper's buffer before the
    next step, and that step refines them."""
    tag = "iso_"
    frames = _frames(gen, fx, tag)
    mapper = _mapper(gen, fx, tag, False)
    new = {k: v.detach().clone() for k, v in mapper.cam.items()}
    new["cam_trans"][..., 2] += 0.01
    mapper.cam = dict(new)
    _one(mapper, frames[2])
    assert mapper.cam["cam_trans"] is not new["cam_trans"]
    assert float((mapper.cam["cam_trans"].detach()[..., 2] - new["cam_trans"][..., 2]).abs().max()) < 0.01
    assert torch.equal(mapper.cam["cam_trans"][..., 0], new["cam_trans"][..., 0])


def _overlap_sequence(gen, T=6):
    """A 96x72 sequence whose camera moves far enough that the keyframes overlap each frame only in part (overlap
    fractions of 0.15-0.33), so keyframe selection's ranking depends on the stored est_w2c; the map starts
    perturbed."""
    import scenes
    from splatam_b200 import slam
    sc = scenes.config1(seed=8, P=240, w=96, h=72)
    gt = sc.splatam_params(opacity_clamp=(0.05, 0.95))
    rots, trans = slam.look_trajectory(T, "cpu", step=(0.12, -0.03, 0.02), rot_step=(0.004, 0.01, 0.002))
    cam = gen.camera(sc)
    frames = [slam.render_frame(gt, rots, trans, t, cam, render=gen.render) for t in range(T)]
    g = torch.Generator().manual_seed(9)
    init = {k: v + 0.02 * torch.randn(v.shape, generator=g) for k, v in gt.items()}
    K = torch.tensor([[sc.fx, 0.0, sc.cx], [0.0, sc.fy, sc.cy], [0.0, 0.0, 1.0]])
    return init, frames, cam, K


def test_run_slam_resumes_exactly_with_refinement_and_keyframe_selection(gen, tmp_path):
    """With refinement on and overlap keyframe selection, a run resumed from its middle checkpoint ends bit-equal to
    the uninterrupted run, keyframe list included: the sidecar carries each keyframe's stored est_w2c, which the
    refined camera columns no longer give.  Each keyframe stores its pose once, after its own mapping phase."""
    from splatam_b200 import formats, slam
    from splatam_b200.keyframes import get_pointcloud, overlap_fractions
    import numpy as np
    init, frames, cam, K = _overlap_sequence(gen)
    T = len(frames)
    torch.manual_seed(0); np.random.seed(0)     # keyframe selection draws from the global generators
    kw = dict(render=gen.render, tracking_iters=3, mapping_iters=3, keyframe_every=1, window=4, fused=False,
              select_keyframes=True, intrinsics=K, mapping_cam_lrs=(0.0004, 0.002))
    full = slam.run_slam(init, frames, cam, checkpoint_dir=str(tmp_path / "a"), checkpoint_every=1, **kw)
    # the keyframes overlap the last frame in part, at different fractions: selection's ranking reads the est_w2c
    last = frames[-1]
    pts = get_pointcloud(last["depth"], K, full["keyframe_est_w2c"][-1],
                         torch.stack(torch.where(last["depth"][0] > 0), dim=1))
    frac = overlap_fractions(pts, torch.stack(full["keyframe_est_w2c"][:-1]), K, cam.image_width, cam.image_height)
    assert ((frac > 0) & (frac < 1)).all() and len(set(frac.tolist())) >= 3, frac

    # insertion rule: keyframe k's est_w2c is column k as checkpoint k (after frame k's mapping phase) holds it ...
    cks = [formats.load_checkpoint(str(tmp_path / "a"), t, "cpu") for t in range(T)]
    assert torch.equal(full["keyframe_est_w2c"][0], torch.eye(4))
    for k in range(1, T):
        at_insertion = slam._curr_w2c(cks[k]["cam_unnorm_rots"], cks[k]["cam_trans"], k)
        assert torch.equal(full["keyframe_est_w2c"][k], at_insertion), k
    # ... and is not refreshed when later mapping phases move the column
    moved = [k for k in range(1, T - 1)
             if not torch.equal(full["keyframe_est_w2c"][k], slam._curr_w2c(full["rots"], full["trans"], k))]
    assert moved

    ck = cks[3]
    rebuilt = [slam._curr_w2c(ck["cam_unnorm_rots"], ck["cam_trans"], k) for k in ck["keyframe_time_indices"]]
    restored = slam.keyframes_from_checkpoint(frames, ck)
    assert any(not torch.equal(a, kf["est_w2c"]) for a, kf in zip(rebuilt, restored))     # the sidecar matters
    for kf, est in zip(restored, full["keyframe_est_w2c"]):
        assert torch.equal(kf["est_w2c"], est)
    res = slam.run_slam(None, frames, cam, checkpoint_dir=str(tmp_path / "b"), checkpoint_every=1, resume=ck, **kw)
    assert res["keyframe_time_indices"] == full["keyframe_time_indices"]
    for a, b in zip(res["keyframe_est_w2c"], full["keyframe_est_w2c"]):
        assert torch.equal(a, b)
    for k in ("rots", "trans"):
        assert torch.equal(full[k], res[k]), k
    for k in full["gauss"]:
        assert torch.equal(full["gauss"][k], res["gauss"][k]), k
    # the sidecar holds the keyframe poses only with refinement on
    off = slam.run_slam(init, frames, cam, checkpoint_dir=str(tmp_path / "c"), checkpoint_every=1,
                        **dict(kw, mapping_cam_lrs=(0.0, 0.0)))
    assert "keyframe_est_w2c" not in formats.load_checkpoint(str(tmp_path / "c"), 3, "cpu")["state"]
    assert not torch.equal(full["trans"][..., 1], off["trans"][..., 1])


def test_offline_drivers_reject_camera_rates(tmp_path):
    """The offline loops keep the poses fixed (the reference's post_splatam_opt renders with camera_grad=False): a
    non-zero camera rate is refused, zero ones are accepted."""
    from splatam_b200 import offline
    with pytest.raises(ValueError):
        offline._map_lrs(dict(offline.LRS, cam_trans=0.001))
    assert offline._map_lrs(dict(offline.LRS, cam_unnorm_rots=0.0, cam_trans=0.0)) == offline.LRS
