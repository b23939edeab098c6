"""GPU: the ingest kernel (csrc/ingest.cu) and the dataset readers (splatam_b200/datasets.py) against the reference's
own dataset classes (tests/golden/datasets/ref_datasets.npz): colour and depth bit for bit in every resize case
(native, downscale, upscale, exact 2x, ScanNet's mixed colour / depth sizes); the prefetching reader against the
synchronous one; and SplaTAM's loop plus `evaluate` on a rendered 1200x680 Replica-layout sequence read from disk."""
import numpy as np
import pytest
import torch

import scenes
from dataset_fixtures import sequence, sequence_fixtures
from splatam_b200 import datasets as D

pytestmark = pytest.mark.gpu

PIXEL_READS = ["replica_native", "replica_down", "replica_up", "replica_half", "tum_up", "scannet_mixed"]


gen, fx, root = sequence_fixtures("datasets")


@pytest.mark.parametrize("prefetch", [0, 2])
@pytest.mark.parametrize("read", PIXEL_READS)
def test_frames_bit_identical_to_reference(gen, fx, root, cuda_device, read, prefetch):
    with sequence(gen, root, read, cuda_device, prefetch) as seq:
        for t in range(len(seq)):
            fr = seq[t]
            assert fr["im"].dtype == torch.float32 and fr["im"].shape == (3, seq.height, seq.width)
            assert torch.equal(fr["im"].cpu(), torch.from_numpy(fx[read + "_color"][t])), (read, t)
            assert torch.equal(fr["depth"].cpu(), torch.from_numpy(fx[read + "_depth"][t])), (read, t)
            assert fr["id"] == t and fr["cam"] is seq.cam and fr["w2c"] is seq.w2c
            pose_ok = bool(np.isfinite(fx[read + "_poses"][t]).all())
            assert bool(torch.isfinite(fr["gt_w2c"]).all()) == pose_ok     # ScanNet's -inf pose: an all-NaN gt_w2c


def test_kernel_matches_numpy_restatement_on_random_frames(cuda_device):
    from oracle import ingest_numpy
    g = np.random.default_rng(5)
    cases = [((680, 1200), (680, 1200), 680, 1200), ((968, 1296), (480, 640), 480, 640), ((680, 1200), (680, 1200), 340, 600),
             ((97, 130), (48, 64), 200, 77), ((5, 7), (3, 2), 33, 17), ((480, 640), (480, 640), 481, 639)]
    for (hc, wc), (hd, wd), H, W in cases:
        rgb = g.integers(0, 256, (hc, wc, 3), dtype=np.uint8)
        raw = g.integers(0, 65536, (hd, wd), dtype=np.uint16)
        color, depth = D.ingest_rgbd(torch.from_numpy(rgb).to(cuda_device), torch.from_numpy(raw).to(cuda_device),
                                     H, W, 5000.0)
        ref_c, ref_d = ingest_numpy.ingest(rgb, raw, H, W, 5000.0)
        assert torch.equal(color.cpu(), torch.from_numpy(ref_c)), ((hc, wc), (H, W))
        assert torch.equal(depth.cpu(), torch.from_numpy(ref_d)), ((hd, wd), (H, W))


def test_prefetch_matches_synchronous_read(gen, root, cuda_device):
    """12 frames through a ring of 3 staging slots (4 refills of each), every frame held; interleaved GPU work on the
    consumer stream.  Repeated indexing returns the same tensors."""
    with sequence(gen, root, "replica_all", cuda_device, 0, desired_height=70, desired_width=100) as ref_seq:
        ref = [ref_seq[t] for t in range(len(ref_seq))]
    held = []
    with sequence(gen, root, "replica_all", cuda_device, 3, desired_height=70, desired_width=100, cache=2) as seq:
        assert len(seq) == 12
        for t in range(len(seq)):
            fr = seq[t]
            assert seq[t] is fr and seq[t]["im"] is fr["im"]
            held.append(fr)
            torch.cuda._sleep(200_000)                 # the consumer stream is busy while the next frames load
        for t, fr in enumerate(held):
            assert torch.equal(fr["im"], ref[t]["im"]) and torch.equal(fr["depth"], ref[t]["depth"]), t
            assert torch.equal(fr["gt_w2c"], ref[t]["gt_w2c"])
        back = seq[2]                                  # out of the cache window: read again, same pixels
        assert back is not held[2] and torch.equal(back["im"], ref[2]["im"])
        assert [f["id"] for f in seq[3:6]] == [3, 4, 5]


def test_run_slam_and_evaluate_on_a_sequence_read_from_disk(tmp_path, cuda_device):
    from splatam_b200 import evaluate, slam
    T = 6
    gt_w2c = scenes.write_replica_sequence(str(tmp_path / "room0"), T, cuda_device)
    with D.RGBDSequence("replica", str(tmp_path), "room0", device=cuda_device, prefetch=2) as seq:
        assert (seq.height, seq.width) == (680, 1200) and len(seq) == T
        K = seq.intrinsics.cpu()
        init, radius = slam.initialize_map(seq[0], K)
        prune = dict(start_after=0, remove_big_after=0, stop_after=20, prune_every=20, removal_opacity_threshold=0.005,
                     final_removal_opacity_threshold=0.005, reset_opacities=False, reset_opacities_every=500)
        out = slam.run_slam(init, seq, seq.cam, seed=3, tracking_iters=20, mapping_iters=10, keyframe_every=5,
                            map_every=1, window=24, sil_thres=0.5, intrinsics=K, add_new_gaussians=True,
                            prune_dict=prune, scene_radius=radius, select_keyframes=True, first_frame_iters=10)
        params = dict(out["gauss"], cam_unnorm_rots=out["rots"], cam_trans=out["trans"])
        res = evaluate.evaluate(params, seq, seq.cam, 0.5, 10, True, gt_w2c=seq.gt_w2c)
        gt = seq.gt_w2c
    for k in ("psnr", "ms_ssim", "depth_rmse", "depth_l1", "ate"):
        assert np.isfinite(res[k]), (k, res[k])
    assert res["psnr"] > 15.0
    hold = slam.ate_horn(gt, [gt[0]] * T)              # never moving from the first pose
    assert res["ate"] < hold, (res["ate"], hold)
    assert torch.allclose(torch.stack([g.cpu().double() for g in gt]), gt_w2c, atol=1e-5)
