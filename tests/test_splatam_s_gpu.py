"""GPU: SplaTAM-S's densification resolution end to end -- the reader's second output bit for bit against the
reference's dataset classes (ref_datasets.npz) and the numpy restatement of the ingest kernel, with and without
prefetch; the initial map and add_new_gaussians on the densification-size frame against the reference's own
initialize_first_timestep / add_new_gaussians (ref_splatam_s.npz); and a SplaTAM-S run plus `evaluate` on a rendered
1200x680 Replica-layout sequence read from disk."""
import os

import numpy as np
import pytest
import torch

import scenes
from dataset_fixtures import sequence, sequence_fixtures
from util import GOLDEN
from splatam_b200 import datasets as D

pytestmark = pytest.mark.gpu

KEYS = ("means3D", "rgb_colors", "unnorm_rotations", "logit_opacities", "log_scales")
CAM_FIELDS = ("image_height", "image_width", "tanfovx", "tanfovy", "viewmatrix", "projmatrix", "campos")
# (desired read, densification read) of ref_datasets.npz: frames 1 and 6 of the 64x48 Replica sequence
PAIRS = [("replica_native", "replica_half"), ("replica_native", "replica_down"), ("replica_up", "replica_native")]
SELECT = dict(start=1, end=11, stride=5)
PRUNE = dict(start_after=0, remove_big_after=0, stop_after=20, prune_every=20, removal_opacity_threshold=0.005,
             final_removal_opacity_threshold=0.005, reset_opacities=False, reset_opacities_every=500)


gen, fx, root = sequence_fixtures("datasets")


@pytest.fixture(scope="module")
def sfx():
    return dict(np.load(os.path.join(GOLDEN, "slam_s", "ref_splatam_s.npz")))


def size(gen, read):
    kw = gen.READS[read][1]
    return kw["desired_height"], kw["desired_width"]


@pytest.mark.parametrize("prefetch", [0, 2])
@pytest.mark.parametrize("pair", PAIRS, ids=["%s+%s" % p for p in PAIRS])
def test_dual_read_bit_identical_to_reference(gen, fx, root, cuda_device, pair, prefetch):
    read, dread = pair
    h_d, w_d = size(gen, dread)
    with sequence(gen, root, read, cuda_device, prefetch, densify_height=h_d, densify_width=w_d) as seq, \
            sequence(gen, root, dread, cuda_device, 0) as single:
        assert len(seq) == 2 and (seq.densify_height, seq.densify_width) == (h_d, w_d)
        assert torch.equal(seq.densify_intrinsics, single.intrinsics)
        for t in range(len(seq)):
            fr = seq[t]
            assert torch.equal(fr["im"].cpu(), torch.from_numpy(fx[read + "_color"][t])), (pair, t)
            assert torch.equal(fr["depth"].cpu(), torch.from_numpy(fx[read + "_depth"][t])), (pair, t)
            dn = fr["densify"]
            assert set(dn) == {"id", "cam", "w2c", "im", "depth", "intrinsics"} and dn["id"] == t
            assert dn["cam"] is seq.densify_cam and dn["w2c"] is seq.w2c and dn["intrinsics"] is seq.densify_intrinsics
            assert dn["im"].shape == (3, h_d, w_d) and dn["depth"].shape == (1, h_d, w_d)
            assert torch.equal(dn["im"].cpu(), torch.from_numpy(fx[dread + "_color"][t])), (pair, t)
            assert torch.equal(dn["depth"].cpu(), torch.from_numpy(fx[dread + "_depth"][t])), (pair, t)
            other = single[t]
            assert torch.equal(dn["im"], other["im"]) and torch.equal(dn["depth"], other["depth"])
            again = seq[t]                              # cached: the same tensors, the densify entry included
            assert again is fr and again["densify"]["im"] is dn["im"] and again["densify"]["depth"] is dn["depth"]


@pytest.mark.parametrize("prefetch", [0, 2])
@pytest.mark.parametrize("read", ["tum_up", "scannet_mixed"])
def test_half_size_second_output_matches_numpy_ingest(gen, root, cuda_device, read, prefetch):
    from oracle import ingest_numpy
    h, w = size(gen, read)
    with sequence(gen, root, read, cuda_device, prefetch, densify_height=h // 2, densify_width=w // 2) as seq:
        for t in range(len(seq)):
            dn = seq[t]["densify"]
            rgb, raw = D.decode_color(seq.files.color_paths[t]), D.decode_depth(seq.files.depth_paths[t])
            ref_c, ref_d = ingest_numpy.ingest(rgb, raw, h // 2, w // 2, seq.files.png_depth_scale)
            assert torch.equal(dn["im"].cpu(), torch.from_numpy(ref_c)), (read, t)
            assert torch.equal(dn["depth"].cpu(), torch.from_numpy(ref_d)), (read, t)


@pytest.mark.parametrize("prefetch", [0, 2])
def test_no_densify_entry_at_the_desired_size(gen, root, cuda_device, prefetch):
    with sequence(gen, root, "replica_native", cuda_device, prefetch, densify_height=48, densify_width=64) as seq:
        assert all("densify" not in seq[t] for t in range(len(seq)))


def _reference_sequence(gen, root, dev):
    return D.RGBDSequence("replica", os.path.join(root, "replica"), gen.SEQUENCES["replica"], gen.config("replica"),
                          desired_height=48, desired_width=64, densify_height=24, densify_width=32, device=dev,
                          prefetch=0, **SELECT)


def test_initial_map_from_the_densify_frame_matches_reference(gen, sfx, root, cuda_device):
    from splatam_b200 import slam
    with _reference_sequence(gen, root, cuda_device) as seq:
        first = seq[0]["densify"]
        init, radius = slam.initialize_map(first, seq.densify_intrinsics.cpu())
    assert init["means3D"].shape[0] == sfx["init_means3D"].shape[0]
    assert np.float32(radius) == sfx["init_scene_radius"]
    for k in KEYS:
        a, b = init[k].cpu().numpy(), sfx["init_" + k]
        assert a.shape == b.shape and np.allclose(a, b, rtol=2e-6, atol=2e-6), (k, np.abs(a - b).max())


def test_add_new_gaussians_on_the_densify_frame_matches_reference(gen, sfx, root, cuda_device):
    """ShardedMapper.add_new_gaussians on the second frame's densify entry, through a stand-in render that returns the
    fixture's preset depth / silhouette: the raster settings it receives are the reference's densify_cam (the image
    size and fields of view exactly; the matrices, inverted on the GPU here and on the CPU there, to 1e-6), and the
    new rows match the reference's."""
    from splatam_b200 import mapping as M, slam
    dev = cuda_device
    t = int(sfx["add_time_idx"])
    seen = []
    preset = torch.from_numpy(sfx["add_depth_sil"]).to(dev)

    def render(settings, means3D, **rv):
        seen.append(settings)
        return preset.clone(), torch.zeros(means3D.shape[0], dtype=torch.int32, device=dev), None
    with _reference_sequence(gen, root, dev) as seq:
        init, _ = slam.initialize_map(seq[0]["densify"], seq.densify_intrinsics.cpu())
        P0 = init["means3D"].shape[0]
        rots = torch.from_numpy(sfx["add_cam_unnorm_rots"]).to(dev).contiguous()
        trans = torch.from_numpy(sfx["add_cam_trans"]).to(dev).contiguous()
        m = M.ShardedMapper(init, rots, trans, render=render, fused=False)
        dn = seq[t]["densify"]
        n = m.add_new_gaussians(dn, t, dn["intrinsics"], float(sfx["add_sil_thres"]))
        assert len(seen) == 1 and seen[0] is seq.densify_cam
    for k in CAM_FIELDS:
        a, b = getattr(seen[0], k), sfx["add_settings_" + k]
        if k.startswith("image_") or k.startswith("tanfov"):
            assert np.asarray(a) == b, k
        else:
            a = a.cpu().numpy()
            assert a.shape == b.shape and np.allclose(a, b, rtol=0, atol=1e-6), (k, np.abs(a - b).max())
    assert n == sfx["add_new_means3D"].shape[0] and m.g.shapes["means3D"][0] == P0 + n
    for k in KEYS:
        a, b = m.g.params[k].detach()[P0:].cpu().numpy(), sfx["add_new_" + k]
        assert a.shape == b.shape and np.allclose(a, b, rtol=2e-6, atol=2e-6), (k, np.abs(a - b).max())


def test_splatam_s_run_and_evaluate_on_a_sequence_read_from_disk(tmp_path, cuda_device, monkeypatch):
    """SplaTAM-S's row (R/configs/replica/splatam_s.py) on a rendered 1200x680 Replica-layout sequence read with
    densification at 340x600: the initial map is the back-projection of every valid pixel of the 600x340 frame 0, no
    stored keyframe holds a densify entry, and the run tracks and reconstructs."""
    from splatam_b200 import evaluate, keyframes, mapping as M, slam
    T = 8
    gt_w2c = scenes.write_replica_sequence(str(tmp_path / "room0"), T, cuda_device)
    stored = []
    select = keyframes.keyframe_selection_overlap
    monkeypatch.setattr(keyframes, "keyframe_selection_overlap",
                        lambda depth, w2c, K, kfs, k, *a, **kw: stored.append(list(kfs)) or select(depth, w2c, K, kfs, k,
                                                                                                 *a, **kw))
    step = M.ShardedMapper.step
    monkeypatch.setattr(M.ShardedMapper, "step", lambda self, win, *a, **kw: stored.append(list(win)) or step(self, win, *a, **kw))
    with D.RGBDSequence("replica", str(tmp_path), "room0", device=cuda_device, prefetch=2, densify_height=340,
                        densify_width=600) as seq:
        assert (seq.height, seq.width, seq.densify_height, seq.densify_width) == (680, 1200, 340, 600)
        first = seq[0]["densify"]
        init, radius = slam.initialize_map(first, seq.densify_intrinsics.cpu())
        assert init["means3D"].shape[0] == int((first["depth"] > 0).sum())
        assert radius == float(first["depth"].max()) / 3.0
        K = seq.intrinsics.cpu()
        out = slam.run_slam(init, seq, seq.cam, seed=3, tracking_iters=10, mapping_iters=15, keyframe_every=5,
                            map_every=1, window=32, sil_thres=0.5, intrinsics=K, add_new_gaussians=True,
                            prune_dict=PRUNE, scene_radius=radius, select_keyframes=True, first_frame_iters=15)
        params = dict(out["gauss"], cam_unnorm_rots=out["rots"], cam_trans=out["trans"])
        res = evaluate.evaluate(params, seq, seq.cam, 0.5, 15, True, gt_w2c=seq.gt_w2c)
        gt = seq.gt_w2c
    assert stored and all("densify" not in f for frames in stored for f in frames)
    for k in ("psnr", "ms_ssim", "depth_rmse", "depth_l1", "ate"):
        assert np.isfinite(res[k]), (k, res[k])
    assert res["psnr"] > 15.0
    hold = slam.ate_horn(gt, [gt[0]] * T)              # never moving from the first pose
    assert res["ate"] < hold, (res["ate"], hold)
    assert torch.allclose(torch.stack([g.cpu().double() for g in gt]), gt_w2c, atol=1e-5)
