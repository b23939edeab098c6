"""CPU: checkpoints and exact resume of the SLAM loop (splatam_b200/slam.py, formats.py) and the per-Gaussian
`timestep` of the mapper's torch path, with the float32 brute-force composite from oracle/ standing in for the
rasterizer.  That renderer and the torch path are deterministic, so a resumed run must equal the uninterrupted one
bit for bit.  The GPU runs are tests/test_checkpoint_gpu.py."""
import os
import shutil
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import refsrc
import scenes
from util import cpu_render, load
from splatam_b200 import formats, mapping as M, slam

T = 8
# three mapping iterations per mapped frame: densification accumulates in iterations 0 and 1 and edits the map in
# iteration 0, pruning runs from iteration 2 -- never both in one iteration, where densify would index the step's
# statistic with the count from before the prune.  The statistic of iteration 1 carries into the next frame.
PRUNE = dict(start_after=2, remove_big_after=0, stop_after=20, prune_every=1, removal_opacity_threshold=0.06,
             final_removal_opacity_threshold=0.06, reset_opacities=False, reset_opacities_every=500)
DENSIFY = dict(start_after=0, remove_big_after=0, stop_after=1, densify_every=2, grad_thresh=2e-6, num_to_split_into=2,
               removal_opacity_threshold=0.06, final_removal_opacity_threshold=0.06, reset_opacities=False,
               reset_opacities_every=100)
REF_RECORD = dict(means3D=np.float32, rgb_colors=np.float32, unnorm_rotations=np.float32, logit_opacities=np.float32,
                  log_scales=np.float32, cam_unnorm_rots=np.float32, cam_trans=np.float32, timestep=np.float32,
                  intrinsics=np.float32, w2c=np.float32, org_width=np.int64, org_height=np.int64,
                  gt_w2c_all_frames=np.float32, keyframe_time_indices=np.int64)


@pytest.fixture(scope="module")
def problem():
    import splatam_b200 as S
    torch.set_num_threads(4)
    sc = scenes.config1(seed=8, P=160, w=48, h=32)
    cam = sc.settings(S.GaussianRasterizationSettings, "cpu")
    gt = sc.splatam_params(opacity_clamp=(0.05, 0.95))
    rots, trans = slam.look_trajectory(T, "cpu", step=(0.004, -0.002, 0.003), rot_step=(0.001, -0.001, 0.0005))
    frames = [slam.render_frame(gt, rots, trans, t, cam, render=cpu_render) for t in range(T)]
    K = torch.tensor([[sc.fx, 0, sc.cx], [0, sc.fy, sc.cy], [0, 0, 1]])
    init = dict(gt)
    init["rgb_colors"] = (gt["rgb_colors"] + 0.2).clamp(0, 1)          # a wrong map: densification has gradients
    kw = dict(render=cpu_render, fused=False, tracking_iters=3, mapping_iters=3, keyframe_every=2, window=3,
              intrinsics=K, prune_dict=PRUNE, densify_dict=DENSIFY, scene_radius=0.5, select_keyframes=True)
    return cam, frames, init, kw


@pytest.fixture(scope="module")
def full_run(problem, tmp_path_factory):
    """The uninterrupted run, checkpointing every second frame."""
    cam, frames, init, kw = problem
    d = str(tmp_path_factory.mktemp("ckpt"))
    torch.manual_seed(1); np.random.seed(1)
    out = slam.run_slam(init, frames, cam, checkpoint_dir=d, checkpoint_every=2, **kw)
    return out, d


def _assert_same_run(a, b):
    assert torch.equal(a["rots"], b["rots"]) and torch.equal(a["trans"], b["trans"])
    for k in M.GAUSSIAN_KEYS:
        assert torch.equal(a["gauss"][k], b["gauss"][k]), k
    assert torch.equal(a["timestep"], b["timestep"])
    assert a["keyframe_time_indices"] == b["keyframe_time_indices"]
    assert a["counts"] == b["counts"] and a["psnr"] == b["psnr"]


@pytest.mark.parametrize("t", [0, 2, 4, 6])
def test_resumed_run_equals_the_uninterrupted_one(problem, full_run, t):
    cam, frames, _, kw = problem
    out, d = full_run
    assert out["counts"][0] == 160 and len(set(out["counts"])) > 1          # the map was edited along the way
    torch.manual_seed(77); np.random.seed(77)                          # the sidecar restores every generator
    ckpt = formats.load_checkpoint(d, t, "cpu")
    assert ckpt["state"] is not None and ckpt["time_idx"] == t
    res = slam.run_slam(None, frames, cam, resume=ckpt, **kw)
    _assert_same_run(out, res)


def test_checkpoint_files(full_run, problem, tmp_path):
    out, d = full_run
    names = {"params%d.npz" % t for t in (0, 2, 4, 6)} | {"keyframe_time_indices%d.npy" % t for t in (0, 2, 4, 6)}
    names |= {"run_state%d.npz" % t for t in (0, 2, 4, 6)} | {"params.npz"}
    assert set(os.listdir(d)) == names
    for t in (0, 2, 4, 6):
        with np.load(os.path.join(d, "params%d.npz" % t)) as z:
            assert list(z.files) == list(formats.CHECKPOINT_KEYS)
            assert all(z[k].dtype == np.float32 for k in z.files)
            assert z["cam_unnorm_rots"].shape == (1, 4, T) and z["cam_trans"].shape == (1, 3, T)
        kti = np.load(os.path.join(d, "keyframe_time_indices%d.npy" % t))
        assert kti.dtype == np.int64 and kti.tolist() == [k for k in out["keyframe_time_indices"] if k <= t]
    with np.load(os.path.join(d, "run_state6.npz")) as z:
        assert z["counts"].dtype == np.int64 and z["counts"].tolist() == out["counts"][:4]
    # without checkpoint_every, checkpoint_dir writes what it always wrote: params<t>.npz per keyframe and params.npz
    cam, frames, init, kw = problem
    torch.manual_seed(1); np.random.seed(1)
    slam.run_slam(init, frames[:5], cam, checkpoint_dir=str(tmp_path), **kw)
    assert set(os.listdir(tmp_path)) == {"params2.npz", "params4.npz", "params.npz"}


def test_reference_style_checkpoint_resumes_at_the_next_frame(problem, full_run, tmp_path, monkeypatch):
    """A checkpoint without the sidecar, as the reference writes it: keyframes rebuilt from the stored camera columns
    as splatam.py:619-638 does, timestep zeros, and the loop starts at t + 1."""
    cam, frames, _, kw = problem
    out, d = full_run
    t = 4
    for name in ("params%d.npz" % t, "keyframe_time_indices%d.npy" % t):
        shutil.copy(os.path.join(d, name), tmp_path / name)
    ckpt = formats.load_checkpoint(str(tmp_path), t, "cpu")
    assert ckpt["state"] is None
    kfs = slam.keyframes_from_checkpoint(frames, ckpt)
    assert [f["id"] for f in kfs] == ckpt["keyframe_time_indices"] == [0, 2, 4]
    for f in kfs:
        k = f["id"]
        rot = F.normalize(ckpt["cam_unnorm_rots"][..., k].detach())
        w2c = torch.eye(4).float()
        w2c[:3, :3] = M.build_rotation(rot)
        w2c[:3, 3] = ckpt["cam_trans"][..., k].detach()
        assert torch.equal(f["est_w2c"], w2c), k
        assert f["im"] is frames[k]["im"] and "densify" not in f
    tracked = []
    track = M.track_frame
    monkeypatch.setattr(M, "track_frame", lambda params, frame, *a, **k: tracked.append(frame["id"]) or
                        track(params, frame, *a, **k))
    res = slam.run_slam(None, frames, cam, resume=ckpt, **kw)
    assert tracked == list(range(t + 1, T))
    assert torch.equal(res["timestep"], torch.zeros(res["gauss"]["means3D"].shape[0]))
    assert res["counts"][0] == ckpt["gauss"]["means3D"].shape[0]
    assert res["keyframe_time_indices"] == [0, 2, 4, 6]


def _record(out, frames, tmp_path, invalid=()):
    K = torch.tensor([[30.0, 0, 23.5], [0, 31.0, 15.5], [0, 0, 1]])
    gt = [torch.eye(4) if t not in invalid else torch.full((4, 4), float("nan")) for t in range(len(frames))]
    return formats.save_run_record(str(tmp_path), out["gauss"], out["rots"], out["trans"], out["timestep"], K,
                                   torch.eye(4), 48, 32, gt, out["keyframe_time_indices"])


def test_run_record_has_the_reference_keys(problem, full_run, tmp_path):
    cam, frames, _, _ = problem
    out, _ = full_run
    path = _record(out, frames, tmp_path, invalid=(3,))
    P = out["gauss"]["means3D"].shape[0]
    with np.load(path) as z:
        rec = {k: z[k] for k in z.files}
    assert list(rec) == list(REF_RECORD)
    for k, dt in REF_RECORD.items():
        assert rec[k].dtype == dt, k
    for k in M.GAUSSIAN_KEYS:
        assert np.array_equal(rec[k], out["gauss"][k].numpy()), k
    assert rec["timestep"].shape == (P,) and rec["intrinsics"].shape == (3, 3) and rec["w2c"].shape == (4, 4)
    assert rec["org_width"].shape == () and int(rec["org_width"]) == 48 and int(rec["org_height"]) == 32
    assert rec["gt_w2c_all_frames"].shape == (T, 4, 4) and np.isnan(rec["gt_w2c_all_frames"][3]).all()
    assert not np.isnan(rec["gt_w2c_all_frames"][[0, 1, 2, 4, 5, 6, 7]]).any()
    assert rec["keyframe_time_indices"].tolist() == [0, 2, 4, 6]
    # scripts/post_splatam_opt.py:94-102 pops the six non-Gaussian keys, then turns the rest into parameters and
    # reads `timestep`
    params = dict(np.load(path, allow_pickle=True))
    for k in ['intrinsics', 'w2c', 'org_width', 'org_height', 'gt_w2c_all_frames', 'keyframe_time_indices']:
        params.pop(k)
    assert set(params) == set(formats.CHECKPOINT_KEYS) | {"timestep"} and len(params["timestep"]) == P
    with pytest.raises(ValueError, match="timestep"):
        formats.save_run_record(str(tmp_path), out["gauss"], out["rots"], out["trans"], torch.zeros(P + 1),
                                torch.eye(3), torch.eye(4), 48, 32, [torch.eye(4)], [0])


def _final_recon():
    """The reference's viz_scripts/final_recon.py from the install in oracle/_ref, imported with this project's
    drop-in package as diff_gaussian_rasterization and open3d / matplotlib stubbed as refsrc stubs them."""
    root = refsrc.ref_root()
    path = None if root is None else os.path.join(root, "viz_scripts", "final_recon.py")
    if path is None or not os.path.isfile(path):
        pytest.skip("the reference's Python (viz_scripts) is not installed in oracle/_ref")
    from splatam_b200.compat import diff_gaussian_rasterization as pkg
    owned = lambda k: k in ("utils", "diff_gaussian_rasterization") or k.startswith("utils.")
    saved = {k: sys.modules.pop(k) for k in [k for k in sys.modules if owned(k)]}
    added = refsrc._stub_missing()
    sys.modules["diff_gaussian_rasterization"] = pkg
    path_before = list(sys.path)
    try:
        mod = load(path)
    finally:
        sys.path[:] = path_before
        for k in [k for k in sys.modules if owned(k)]:
            del sys.modules[k]
        for k in added:
            sys.modules.pop(k, None)
        sys.modules.update(saved)
    return mod


def test_reference_load_camera_reads_the_record(problem, full_run, tmp_path):
    cam, frames, _, _ = problem
    out, _ = full_run
    path = _record(out, frames, tmp_path)
    w2c, k = _final_recon().load_camera(dict(viz_w=96, viz_h=80), path)
    K = np.array([[30.0, 0, 23.5], [0, 31.0, 15.5], [0, 0, 1]], np.float32)
    assert np.array_equal(w2c, np.eye(4, dtype=np.float32))
    assert np.allclose(k, K * np.array([[96 / 48], [80 / 32], [1.0]]), rtol=1e-6)


def test_argument_checks(problem, full_run, tmp_path):
    cam, frames, init, kw = problem
    out, d = full_run
    ckpt = formats.load_checkpoint(d, 2, "cpu")
    with pytest.raises(ValueError, match="not both"):
        slam.run_slam(init, frames, cam, resume=ckpt, **kw)
    with pytest.raises(ValueError, match="cover 8 frames"):
        slam.run_slam(None, frames[:6], cam, resume=ckpt, **kw)
    for bad in (-1, 8):
        with pytest.raises(ValueError, match="outside"):
            slam.run_slam(None, frames, cam, resume=dict(ckpt, time_idx=bad), **kw)
    for bad in (0, -2, 1.5, True, "2"):
        with pytest.raises(ValueError, match="positive integer"):
            slam.run_slam(init, frames, cam, checkpoint_dir=str(tmp_path), checkpoint_every=bad, **kw)
    with pytest.raises(ValueError, match="checkpoint_dir"):
        slam.run_slam(init, frames, cam, checkpoint_every=2, **kw)
    with pytest.raises(FileNotFoundError, match="params3.npz"):
        formats.load_checkpoint(d, 3, "cpu")
    shutil.copy(os.path.join(d, "params2.npz"), tmp_path / "params2.npz")
    with pytest.raises(FileNotFoundError, match="keyframe_time_indices2.npy"):
        formats.load_checkpoint(str(tmp_path), 2, "cpu")
    assert os.listdir(tmp_path) == ["params2.npz"]               # the rejected runs wrote nothing


def test_tool_needs_out_for_checkpoints(monkeypatch, capsys):
    tool = load("tools/run_slam_dataset.py")
    for extra in (["--checkpoint-every", "5"], ["--resume", "10"]):
        monkeypatch.setattr(sys, "argv", ["run_slam_dataset.py", "--dataset", "replica", "--basedir", "x",
                                          "--sequence", "y"] + extra)
        with pytest.raises(SystemExit) as e:
            tool.main()
        assert e.value.code == 2 and "--out" in capsys.readouterr().err, extra


def _mapper(P=24, seed=0):
    g = torch.Generator().manual_seed(seed)
    gauss = dict(means3D=torch.randn(P, 3, generator=g), rgb_colors=torch.rand(P, 3, generator=g),
                 unnorm_rotations=torch.randn(P, 4, generator=g), logit_opacities=torch.randn(P, 1, generator=g),
                 log_scales=torch.randn(P, 1, generator=g) - 3.0)
    return M.ShardedMapper(gauss, torch.zeros(1, 4, 2), torch.zeros(1, 3, 2), render=cpu_render, fused=False), gauss


def test_mapper_timestep_follows_the_map_edits():
    m, gauss = _mapper()
    assert torch.equal(m.timestep, torch.zeros(24))
    new = {k: v[:5] for k, v in gauss.items()}
    m.add_gaussians(new, timestep=3)
    m.add_gaussians(new, timestep=torch.arange(5) + 10)
    m.add_gaussians(new)                                               # default: 0
    expect = torch.cat([torch.zeros(24), torch.full((5,), 3.0), torch.arange(5.0) + 10, torch.zeros(5)])
    assert m.timestep.dtype == torch.float32 and torch.equal(m.timestep, expect)
    drop = torch.zeros(39, dtype=torch.bool)
    drop[[0, 5, 25, 30, 31]] = True
    assert m.remove_points(drop) == 34 and torch.equal(m.timestep, expect[~drop])
    with pytest.raises(ValueError, match="timestep"):
        m.add_gaussians(new, timestep=torch.zeros(4))
    with pytest.raises(ValueError, match="timestep"):
        M.ShardedMapper(gauss, torch.zeros(1, 4, 2), torch.zeros(1, 3, 2), fused=False, timestep=torch.zeros(3))
    m2 = M.ShardedMapper(gauss, torch.zeros(1, 4, 2), torch.zeros(1, 3, 2), fused=False, timestep=torch.arange(24))
    assert torch.equal(m2.timestep, torch.arange(24.0))


def test_densify_children_inherit_the_parent_timestep():
    """Clones and split samples carry their parent's timestep (R/utils/gs_external.py:202-222)."""
    m, _ = _mapper(P=40, seed=3)
    m.timestep = torch.arange(40.0)
    with torch.no_grad():
        m.g.params["log_scales"][:20] = -6.0                            # small: cloned
        m.g.params["log_scales"][20:] = -1.0                            # big: split
        m.g.params["logit_opacities"].fill_(2.0)                        # nothing is transparent
    dd = dict(DENSIFY, grad_thresh=0.5, removal_opacity_threshold=0.01, final_removal_opacity_threshold=0.01,
              remove_big_after=100)
    grad = torch.zeros(40, 3)
    grad[[2, 7, 23, 31], 0] = 1.0
    P = m.densify(0, dd, scene_radius=1.0, means2D_grad=grad, seen=torch.ones(40, dtype=torch.bool),
                  generator=torch.Generator().manual_seed(0))
    # 2 clones appended, then the 2 split parents removed and 2 x 2 samples appended
    assert P == 40 + 2 - 2 + 4
    keep = torch.ones(42, dtype=torch.bool)
    keep[[23, 31]] = False
    expect = torch.cat([torch.arange(40.0), torch.tensor([2.0, 7.0])])[keep]
    assert torch.equal(m.timestep, torch.cat([expect, torch.tensor([23.0, 31.0, 23.0, 31.0])]))
