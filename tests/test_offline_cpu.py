"""CPU: the offline all-frame loop (splatam_b200/offline.py) against tests/golden/offline/ref_offline.npz, which the
reference's own get_loss_gs, densify, get_expon_lr_func and update_learning_rate produced over the same map, frames
and float32 brute-force renderer; plus the record reader, the original-index pose lookup and the torch counterpart of
FusedAdam.set_lr.  The GPU runs are tests/test_offline_gpu.py."""
import importlib.util
import os

import numpy as np
import pytest
import torch

from splatam_b200 import formats, mapping as M, offline

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "offline")


def _generator():
    spec = importlib.util.spec_from_file_location("make_golden_offline", os.path.join(GOLDEN, "make_golden_offline.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


@pytest.fixture(scope="module")
def gen():
    torch.set_num_threads(4)
    mod = _generator()
    return mod, mod.problem()


def _write_record(pr, out_dir, keyframes=(0,)):
    return formats.save_run_record(out_dir, pr["init"], pr["rots"], pr["trans"], pr["timestep"], pr["K"], torch.eye(4),
                                   pr["sc"].w, pr["sc"].h, pr["w2c"], keyframes)


def _from_record(pr, path, index=None, lrs=offline.LRS):
    index = list(range(len(pr["frames"]))) if index is None else index
    return offline.from_record(path, pr["frames"], index, "cpu", lrs=lrs, render=pr["render"], fused=False)


def test_loop_matches_reference_fixture(gen, tmp_path, monkeypatch):
    mod, pr = gen
    G = np.load(os.path.join(GOLDEN, "ref_offline.npz"))
    lrs = {k: mod.LRS[k] for k in M.GAUSSIAN_KEYS}
    mapper, train, radius, _ = _from_record(pr, _write_record(pr, str(tmp_path)), lrs=lrs)
    assert radius == pytest.approx(float(G["scene_radius"]), rel=1e-6)
    monkeypatch.setattr(torch, "normal", mod.split_normal())      # the split samples the fixture drew
    trace = []
    counts = offline.optimize_map(mapper, train, mod.ITERS, mod.LR_FINAL, mod.DENSIFY, radius, seed=mod.SEED,
                                  trace=trace)
    assert [t["frame"] for t in trace] == G["frame_seq"].tolist()
    np.testing.assert_allclose([t["lr"] for t in trace], G["lr"], rtol=1e-12)
    np.testing.assert_allclose([float(t["loss"]) for t in trace], G["loss"], rtol=1e-5)
    # the Adam step is skipped exactly where densify edits the map (iterations 3 and 6)
    assert [t["stepped"] for t in trace] == [it not in (3, 6) for it in range(mod.ITERS)]
    assert counts == G["counts"].tolist()
    np.testing.assert_array_equal(mapper.timestep.numpy(), G["timestep"])
    assert mapper._adam_steps() == int(G["out_means3D_step"]) == mod.ITERS - 2
    for k, (m, v) in mapper.moments().items():
        np.testing.assert_allclose(mapper.g.params[k].detach().numpy(), G["out_" + k], rtol=1e-5, atol=1e-6)
        if k == "unnorm_rotations":     # moments of a rounding-noise gradient (see the generator's LRS)
            continue
        np.testing.assert_allclose(m.numpy(), G["out_" + k + "_exp_avg"], rtol=1e-3, atol=1e-7)
        np.testing.assert_allclose(v.numpy(), G["out_" + k + "_exp_avg_sq"], rtol=1e-3, atol=1e-12)
    assert mapper.lrs["means3D"] == pytest.approx(G["lr"][-1], rel=1e-12)


def test_from_record_reads_the_reference_layout(gen, tmp_path):
    _, pr = gen
    mine, _, _, _ = _from_record(pr, _write_record(pr, str(tmp_path / "here")))
    # the reference's save_params: np.savez of its dict, float64 intrinsics from the dataset, python ints, a list of
    # keyframe indices
    ref = {k: v.numpy() for k, v in pr["init"].items()}
    ref.update(cam_unnorm_rots=pr["rots"].numpy(), cam_trans=pr["trans"].numpy(), timestep=pr["timestep"].numpy(),
               intrinsics=pr["K"].double().numpy(), w2c=np.eye(4), org_width=pr["sc"].w, org_height=pr["sc"].h,
               gt_w2c_all_frames=np.stack([w.numpy() for w in pr["w2c"]]), keyframe_time_indices=np.array([0, 2]))
    path = str(tmp_path / "params.npz")
    np.savez(path, **ref)
    theirs, train, _, rec = _from_record(pr, path)
    assert set(rec) == set(formats.RECORD_KEYS)
    for k in M.GAUSSIAN_KEYS:
        assert torch.equal(mine.g.params[k], theirs.g.params[k])
    assert torch.equal(mine.timestep, theirs.timestep)
    for t, fr in enumerate(train):
        assert torch.allclose(fr["pose"][0], pr["w2c"][t], atol=1e-6)
    missing = {k: v for k, v in ref.items() if k != "timestep"}
    np.savez(path, **missing)
    with pytest.raises(ValueError, match="timestep"):
        _from_record(pr, path)


def test_pose_lookup_uses_the_original_frame_index(gen, tmp_path):
    _, pr = gen
    path = _write_record(pr, str(tmp_path))
    # frames read at stride 2 from a three-frame SLAM run: training frame 1 is image 2, trained at camera column 2
    _, train, _, _ = _from_record(pr, path, index=[0, 2, 1])
    for fr, k in zip(train, (0, 2, 1)):
        rel, q = M.camera_w2c(pr["rots"][..., k], pr["trans"][..., k])
        assert torch.equal(fr["pose"][0], rel) and torch.equal(fr["pose"][1], q)
    with pytest.raises(ValueError, match="3 camera columns; frame index 3"):
        _from_record(pr, path, index=[0, 3, 1])
    with pytest.raises(ValueError, match="3 camera columns; frame index -1"):
        _from_record(pr, path, index=[0, -1, 1])
    with pytest.raises(ValueError, match="2 frame indices for 3 frames"):
        _from_record(pr, path, index=[0, 1])


def test_record_without_keyframes_has_the_post_opt_keys(gen, tmp_path):
    _, pr = gen
    path = _write_record(pr, str(tmp_path), keyframes=None)
    rec = formats.load_params(path)
    assert list(rec) == [k for k in formats.RECORD_KEYS if k != "keyframe_time_indices"]
    assert len(rec) == 13 and rec["gt_w2c_all_frames"].shape == (3, 4, 4)


def test_expon_lr_is_the_log_linear_schedule():
    assert offline.expon_lr(0, 3.2e-4, 3.2e-6, 100) == pytest.approx(3.2e-4)
    assert offline.expon_lr(100, 3.2e-4, 3.2e-6, 100) == pytest.approx(3.2e-6)
    assert offline.expon_lr(50, 3.2e-4, 3.2e-6, 100) == pytest.approx(3.2e-5)
    assert offline.expon_lr(250, 3.2e-4, 3.2e-6, 100) == pytest.approx(3.2e-6)
    assert offline.expon_lr(-1, 3.2e-4, 3.2e-6, 100) == 0.0


def test_set_lr_torch_path_changes_one_group_and_survives_map_edits(gen):
    _, pr = gen
    mapper = M.ShardedMapper(pr["init"], pr["rots"], pr["trans"], lrs=offline.LRS, render=pr["render"], fused=False)
    mapper.set_lr("log_scales", 0.25)
    lrs = [g["lr"] for g in mapper.opt.param_groups]
    assert lrs == [offline.LRS[k] if k != "log_scales" else 0.25 for k in M.GAUSSIAN_KEYS]
    mapper.add_gaussians({k: v[:2] for k, v in pr["init"].items()})       # rebuilds the optimizer
    assert [g["lr"] for g in mapper.opt.param_groups] == lrs


def test_densify_due_schedule():
    d = dict(start_after=500, stop_after=15000, densify_every=100)
    assert not M.densify_due(400, d) and M.densify_due(500, d) and not M.densify_due(501, d)
    assert M.densify_due(15000, d) and not M.densify_due(15100, d)
