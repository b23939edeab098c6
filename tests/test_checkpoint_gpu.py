"""GPU: the per-Gaussian `timestep` through the fused map edits, end to end through the SLAM loop, checkpoint / resume
on the fused path (eager and graph), and the dataset tool's --checkpoint-every / --resume.  Two GPU runs are not
bit-equal (the backward uses float atomics), so resumed runs are held to test_slam_gpu.py's bounds between two arms."""
import os

import numpy as np
import pytest
import torch

import scenes
from util import load, run_tool
from test_slam_gpu import _opaque_sequence

pytestmark = pytest.mark.gpu

K = torch.tensor([[160.0, 0, 159.5], [0, 160.0, 95.5], [0, 0, 1]])
PRUNE = dict(start_after=0, remove_big_after=0, stop_after=20, prune_every=4, removal_opacity_threshold=0.005,
             final_removal_opacity_threshold=0.005, reset_opacities=False, reset_opacities_every=500)


def _map(dev, P=3000, seed=0):
    g = torch.Generator().manual_seed(seed)
    gauss = dict(means3D=torch.randn(P, 3, generator=g), rgb_colors=torch.rand(P, 3, generator=g),
                 unnorm_rotations=torch.randn(P, 4, generator=g), logit_opacities=torch.randn(P, 1, generator=g),
                 log_scales=torch.randn(P, 1, generator=g) - 3.0)        # isotropic, as SplaTAM's densify takes it
    return {k: v.to(dev) for k, v in gauss.items()}


def test_timestep_through_fused_map_edits(cuda_device):
    from splatam_b200 import mapping as M
    dev = cuda_device
    gauss = _map(dev)
    P = gauss["means3D"].shape[0]
    rots, trans = torch.zeros(1, 4, 2, device=dev), torch.zeros(1, 3, 2, device=dev)
    ts0 = torch.randint(0, 50, (P,), generator=torch.Generator().manual_seed(1)).float()
    arms = {f: M.ShardedMapper(gauss, rots, trans, fused=f, timestep=ts0) for f in (True, False)}
    g = torch.Generator().manual_seed(2)
    drop = (torch.rand(P, generator=g) < 0.3).to(dev)
    new = {k: v[:400] * 1.01 for k, v in gauss.items()}
    new_ts = torch.arange(400, device=dev) % 7 + 100
    grad = torch.rand(P, 3, generator=g).to(dev)
    seen = (torch.rand(P, generator=g) < 0.8).to(dev)
    dd = dict(start_after=0, remove_big_after=0, stop_after=10, densify_every=1, grad_thresh=0.5, num_to_split_into=2,
              removal_opacity_threshold=0.3, final_removal_opacity_threshold=0.3, reset_opacities=False,
              reset_opacities_every=100)
    for m in arms.values():
        m.remove_points(drop)
        m.add_gaussians(new, timestep=new_ts)
        m.add_gaussians({k: v[:5] for k, v in new.items()}, timestep=7)
        n = m.g.shapes["means3D"][0]                         # about 0.7 P + 405 < P
        m.densify(0, dd, scene_radius=2.0, means2D_grad=grad[:n], seen=seen[:n],
                  generator=torch.Generator(device=dev).manual_seed(3))
    a, b = arms[True], arms[False]
    assert a.timestep.device == b.timestep.device == dev
    assert torch.equal(a.timestep, b.timestep)
    assert a.timestep.shape[0] == a.g.shapes["means3D"][0] != P
    assert torch.equal(a.g.flat, b.g.flat)
    assert set(a.timestep.unique().tolist()) <= set(ts0.tolist()) | set(range(100, 107)) | {7.0}


def _sequence(dev):
    import splatam_b200 as S
    from splatam_b200 import slam
    cam, frames, rots_gt, trans_gt = _opaque_sequence(dev, S.GaussianRasterizationSettings)
    init, radius = slam.initialize_map(frames[0], K)
    return cam, frames, rots_gt, trans_gt, init, radius


def test_timestep_end_to_end(cuda_device):
    from splatam_b200 import slam
    dev = cuda_device
    cam, frames, _, _, init, radius = _sequence(dev)
    common = dict(fused=True, intrinsics=K, add_new_gaussians=True, sil_thres=0.5, scene_radius=radius, window=4,
                  mapping_iters=6, first_frame_iters=20, tracking_iters=20, map_every=1)
    torch.manual_seed(3); np.random.seed(3)
    out = slam.run_slam(init, frames, cam, **common)
    ts, counts = out["timestep"], out["counts"]
    assert ts.shape[0] == counts[-1] and counts[0] == init["means3D"].shape[0]
    assert int((ts == 0).sum()) == counts[0]
    for t in range(1, len(frames)):                          # no pruning: frame t's growth carries timestep t
        assert counts[t] - counts[t - 1] == int((ts == t).sum()), t
    assert counts[-1] > counts[0]
    torch.manual_seed(3); np.random.seed(3)
    out = slam.run_slam(init, frames, cam, prune_dict=PRUNE, **common)
    ts = out["timestep"]
    assert ts.shape[0] == out["counts"][-1]
    assert bool((ts[1:] >= ts[:-1]).all())                   # compaction keeps the row order, growth appends
    assert set(ts.unique().tolist()) <= {float(t) for t in range(len(frames))}


def test_resume_on_the_gpu(cuda_device, tmp_path, monkeypatch):
    from splatam_b200 import formats, slam
    dev = cuda_device
    cam, frames, rots_gt, trans_gt, init, radius = _sequence(dev)
    common = dict(fused=True, intrinsics=K, add_new_gaussians=True, sil_thres=0.5, prune_dict=PRUNE,
                  scene_radius=radius, select_keyframes=True, window=4, mapping_iters=12, tracking_iters=40)
    saved, est = {}, {}
    save = formats.save_checkpoint

    def recording_save(directory, t, params, kti, run_state=None):
        saved[t] = ({k: v.detach().clone() for k, v in params.items()}, list(kti),
                    {k: np.array(v, copy=True) for k, v in run_state.items()})
        return save(directory, t, params, kti, run_state)
    monkeypatch.setattr(formats, "save_checkpoint", recording_save)
    curr = slam._curr_w2c
    monkeypatch.setattr(slam, "_curr_w2c", lambda r, tr, t: est.setdefault(t, curr(r, tr, t)))
    torch.manual_seed(3); np.random.seed(3)
    full = slam.run_slam(init, frames, cam, checkpoint_dir=str(tmp_path), checkpoint_every=4, first_frame_iters=60,
                         **common)
    monkeypatch.undo()
    assert sorted(saved) == [0, 4, 8]
    t = 4
    ck = formats.load_checkpoint(str(tmp_path), t, dev)
    params, kti, state = saved[t]
    for k, v in ck["gauss"].items():
        assert torch.equal(v, params[k]), k
    assert torch.equal(ck["cam_unnorm_rots"], params["cam_unnorm_rots"])
    assert torch.equal(ck["cam_trans"], params["cam_trans"])
    assert ck["keyframe_time_indices"] == kti == [0, 2, 4]
    assert set(ck["state"]) == set(state) and "cuda_rng" in state
    for k in state:
        assert np.array_equal(ck["state"][k], state[k]), k
    assert state["timestep"].max() > 0                       # the map grew after frame 0
    for kf in slam.keyframes_from_checkpoint(frames, ck):
        if kf["id"] > 0:
            assert torch.equal(kf["est_w2c"], est[kf["id"]]), kf["id"]
    travelled = float(trans_gt[0, :, -1].norm())
    ate_full = slam.ate_rmse(full["rots"], full["trans"], rots_gt, trans_gt)
    for graph in (False, True):
        res = slam.run_slam(None, frames, cam, resume=formats.load_checkpoint(str(tmp_path), t, dev), graph=graph,
                            **common)
        ate = slam.ate_rmse(res["rots"], res["trans"], rots_gt, trans_gt)
        print("resume graph=%s: ATE %.5f (uninterrupted %.5f), PSNR %.2f (%.2f)" % (graph, ate, ate_full, res["psnr"],
                                                                                   full["psnr"]))
        assert torch.equal(res["rots"][..., :t + 1], full["rots"][..., :t + 1])
        assert res["keyframe_time_indices"] == full["keyframe_time_indices"]
        assert res["timestep"].shape[0] == res["counts"][-1] == res["gauss"]["means3D"].shape[0]
        assert abs(res["psnr"] - full["psnr"]) < 2.0
        assert abs(ate - ate_full) < 0.01 * travelled


def test_tool_checkpoints_and_resumes(cuda_device, tmp_path, monkeypatch, capsys):
    T = 12
    scenes.write_replica_sequence(str(tmp_path / "room0"), T, cuda_device)
    tool = load("tools/run_slam_dataset.py")
    out_dir = str(tmp_path / "run")
    base = ["run_slam_dataset.py", "--dataset", "replica", "--basedir", str(tmp_path), "--sequence", "room0",
            "--tracking-iters", "10", "--mapping-iters", "10", "--out", out_dir]
    lines = []
    for extra in (["--checkpoint-every", "5"], ["--resume", "10"]):
        lines.append(run_tool(tool, base + extra, monkeypatch, capsys))
        with np.load(os.path.join(out_dir, "params.npz")) as z:
            rec = {k: z[k] for k in z.files}
        if extra[0] == "--checkpoint-every":
            first = rec
            for t in (0, 5, 10):
                assert os.path.isfile(os.path.join(out_dir, "params%d.npz" % t))
                assert os.path.isfile(os.path.join(out_dir, "run_state%d.npz" % t))
    assert lines[0]["resumed_from"] is None and lines[1]["resumed_from"] == 10 and lines[1]["resume_s"] > 0
    assert list(rec) == list(first) and len(rec) == 14
    assert rec["timestep"].shape == (rec["means3D"].shape[0],)
    assert rec["gt_w2c_all_frames"].shape == (T, 4, 4) and int(rec["org_width"]) == 1200
    kti = np.load(os.path.join(out_dir, "keyframe_time_indices10.npy")).tolist()
    assert kti == [0, 5, 10] and rec["keyframe_time_indices"].tolist()[:len(kti)] == kti
    assert first["keyframe_time_indices"].tolist()[:len(kti)] == kti
    for line in lines:
        assert np.isfinite(line["ate_m"]) and np.isfinite(line["psnr_db"])
