"""GPU: the densification statistic kernel (sb_densify_accumulate), FusedAdam.set_lr, the fused offline loop against
the torch path, and tools/run_offline_opt.py end to end in both modes on a synthetic Replica-layout sequence."""
import importlib.util
import json
import os
import sys

import numpy as np
import pytest
import torch

import scenes
from splatam_b200 import evaluate, formats, map_ops, mapping as M, offline, slam
from splatam_b200.train_ops import FusedAdam

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_densify_accumulate_is_bit_equal_to_the_torch_statement(cuda_device):
    g = torch.Generator(device=cuda_device).manual_seed(3)
    P = 100_003
    grad = 1e-3 * torch.randn(P, 3, device=cuda_device, generator=g)
    grad[::7] = 0.0                                           # zero gradients
    seen = torch.rand(P, device=cuda_device, generator=g) < 0.6  # unseen rows stay untouched
    accum = torch.rand(P, device=cuda_device, generator=g)
    denom = torch.randint(0, 5, (P,), device=cuda_device, generator=g).float()
    a_ref, d_ref = accum.clone(), denom.clone()
    a_ref[seen] += torch.norm(grad[seen, :2], dim=-1)
    d_ref[seen] += 1
    map_ops.densify_accumulate(grad, seen, accum, denom)
    assert torch.equal(accum, a_ref) and torch.equal(denom, d_ref)
    with pytest.raises(Exception, match="bool"):
        map_ops.densify_accumulate(grad, seen.float(), accum, denom)


def test_set_lr_changes_only_its_segment(cuda_device):
    sizes = [5, 7, 3]
    flat = torch.zeros(sum(sizes), device=cuda_device)
    grad = torch.ones_like(flat)
    opt = FusedAdam(flat, grad, sizes, [0.1, 0.2, 0.3])
    opt.step()
    torch.testing.assert_close(flat, torch.cat([torch.full((n,), -lr, device=cuda_device)
                                                for n, lr in zip(sizes, (0.1, 0.2, 0.3))]))
    before = flat.clone()
    opt.set_lr(1, 0.05)
    opt.step()
    step = (flat - before).split(sizes)
    for s, lr in zip(step, (0.1, 0.05, 0.3)):
        torch.testing.assert_close(s, torch.full_like(s, -lr))
    with pytest.raises(IndexError):
        opt.set_lr(3, 0.1)


def _problem(dev, T=4):
    import splatam_b200 as S
    sc = scenes.config1(seed=8, P=2000, w=96, h=64)
    cam = sc.settings(S.GaussianRasterizationSettings, dev)
    gt = dict(means3D=sc.means3D, rgb_colors=sc.colors, unnorm_rotations=sc.rotations,
              logit_opacities=torch.logit(sc.opacities.clamp(0.05, 0.95)), log_scales=torch.log(sc.scales[:, :1]))
    gt = {k: v.to(dev) for k, v in gt.items()}
    rots, trans = slam.look_trajectory(T, dev)
    frames = [slam.render_frame(gt, rots, trans, t, cam) for t in range(T)]
    g = torch.Generator().manual_seed(5)
    init = {k: v + 0.02 * torch.randn(v.shape, generator=g).to(dev) for k, v in gt.items()}
    train = [dict(fr, pose=M.camera_w2c(rots[..., t], trans[..., t])) for t, fr in enumerate(frames)]
    return init, rots, trans, train


def test_fused_loop_matches_the_torch_path(cuda_device):
    init, rots, trans, train = _problem(cuda_device)
    dd = dict(offline.DENSIFY, start_after=50, densify_every=50, remove_big_after=100, reset_opacities_every=150)
    out = {}
    for fused in (True, False):
        torch.manual_seed(0)
        mapper = M.ShardedMapper(init, rots, trans, lrs=offline.LRS, fused=fused)
        before = offline.train_psnr(mapper, train)
        counts = offline.optimize_map(mapper, train, 300, offline.MEANS3D_LR_FINAL, dd, 1.5, seed=0)
        out[fused] = (before, offline.train_psnr(mapper, train), counts, mapper.lrs["means3D"])
    (b_f, a_f, c_f, lr_f), (b_t, a_t, c_t, lr_t) = out[True], out[False]
    assert abs(b_f - b_t) < 0.05 and a_f > b_f + 1.0 and a_t > b_t + 1.0
    # float atomics in the backward make the runs drift apart; the bound test_slam_gpu.py puts on fused vs torch PSNR
    assert abs(a_f - a_t) < 2.0
    assert abs(c_f[-1] - c_t[-1]) <= 0.05 * c_t[-1] and lr_f == lr_t


def _tool(name):
    spec = importlib.util.spec_from_file_location(name, os.path.join(ROOT, "tools", name + ".py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _run(tool, argv, monkeypatch, capsys):
    monkeypatch.setattr(sys, "argv", argv)
    tool.main()
    return json.loads(capsys.readouterr().out.strip().splitlines()[-1])


def test_tool_runs_both_modes_and_its_evaluation_is_evaluate(cuda_device, tmp_path, monkeypatch, capsys):
    T = 11
    scenes.write_replica_sequence(str(tmp_path / "room0"), T, cuda_device)
    data = ["--dataset", "replica", "--basedir", str(tmp_path), "--sequence", "room0"]
    slam_dir = str(tmp_path / "slam")
    _run(_tool("run_slam_dataset"), ["run_slam_dataset.py"] + data + ["--tracking-iters", "10", "--mapping-iters", "10",
                                                                       "--out", slam_dir], monkeypatch, capsys)
    opt = _tool("run_offline_opt")
    post_dir = str(tmp_path / "post")
    line = _run(opt, ["run_offline_opt.py", "--mode", "post_splatam", "--record", os.path.join(slam_dir, "params.npz"),
                      "--stride", "5", "--iters", "120", "--eval-frames", "3", "--out", post_dir] + data,
                monkeypatch, capsys)
    assert line["frames"] == 3 and line["iters"] == 120 and line["eval_frames"] == 3
    assert line["train_psnr_after_db"] >= line["train_psnr_before_db"]
    rec = formats.load_params(os.path.join(post_dir, "params.npz"))
    assert list(rec) == [k for k in formats.RECORD_KEYS if k != "keyframe_time_indices"]
    assert rec["means3D"].shape[0] == line["gaussians"] == rec["timestep"].shape[0]
    slam_rec = formats.load_params(os.path.join(slam_dir, "params.npz"))
    for t, k in enumerate((0, 5, 10)):         # trained at the SLAM camera column of the original index
        w2c = M.camera_w2c(torch.from_numpy(slam_rec["cam_unnorm_rots"][..., k]),
                           torch.from_numpy(slam_rec["cam_trans"][..., k]))[0]
        np.testing.assert_allclose(rec["gt_w2c_all_frames"][t], w2c.numpy(), atol=1e-6)
    # the final evaluation is evaluate() at the eval frames' ground-truth poses on the saved map
    from splatam_b200 import datasets
    with datasets.RGBDSequence("replica", str(tmp_path), "room0", stride=5, desired_height=680, desired_width=1200,
                               device=cuda_device) as seq:
        frames = [seq[t] for t in range(3)]
        gauss = {k: torch.from_numpy(rec[k]).to(cuda_device) for k in M.GAUSSIAN_KEYS}
        direct = evaluate.evaluate(gauss, frames, seq.cam, 0.5, 120, True, at_gt_pose=True)
    assert direct["psnr"] == line["psnr_db"] and direct["depth_l1"] == line["depth_l1_m"]
    np.testing.assert_array_equal(np.loadtxt(os.path.join(post_dir, "eval", "psnr.txt")), direct["psnr_per_frame"])
    # the intermediate evaluation (iteration 7000 in the shipped configs; 40 here) through the tool's scoring, on the
    # map as it stands inside the loop
    mapper, train, radius, _ = offline.from_record(os.path.join(slam_dir, "params.npz"), frames, [0, 5, 10],
                                                   cuda_device)
    seen = {}

    def on_eval(it, m):
        snap = {k: v.detach().clone() for k, v in m.g.params.items()}
        seen[it] = (opt.score(m.g.params, frames, seq.cam, 80, out_dir=str(tmp_path / "eval_7k")),
                    evaluate.evaluate(snap, frames, seq.cam, 0.5, 80, True, at_gt_pose=True))
    offline.optimize_map(mapper, train, 80, offline.MEANS3D_LR_FINAL, offline.DENSIFY, radius, eval_at=(40,),
                         on_eval=on_eval)
    assert list(seen) == [40]
    via_tool, direct_40 = seen[40]
    for k in ("psnr", "ms_ssim", "depth_l1", "depth_rmse"):
        assert via_tool[k] == direct_40[k]
    assert direct_40["psnr"] != direct["psnr"]
    np.testing.assert_array_equal(np.loadtxt(str(tmp_path / "eval_7k" / "psnr.txt")), direct_40["psnr_per_frame"])
    gt_dir = str(tmp_path / "gt")
    line = _run(opt, ["run_offline_opt.py", "--mode", "gt_poses", "--iters", "120", "--eval-frames", "2",
                      "--out", gt_dir] + data, monkeypatch, capsys)
    assert line["frames"] == T and line["initial_gaussians"] > 0 and np.isfinite(line["psnr_db"])
    assert line["train_psnr_after_db"] >= line["train_psnr_before_db"]
    assert line["width"] == 600 and line["height"] == 340
