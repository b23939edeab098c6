"""CPU: the ScanNet++ and ReplicaV2 readers of splatam_b200/datasets.py, both splits, against the reference's own
ScannetPPDataset and ReplicaV2Dataset run unmodified on tiny synthetic sequences
(tests/golden/datasets/ref_nvs_datasets.npz, written by make_golden_nvs_datasets.py): file order, split assembly,
is_bad filtering, start / end / stride on the test split, poses, intrinsics and retained indices bit for bit, colour
and depth through the float64 restatement of the ingest kernel; and the error cases."""
import json
import os
import shutil

import pytest
import torch

from dataset_fixtures import files_of, sequence_fixtures
from util import GOLDEN, bits_equal
from splatam_b200 import datasets as D

FIX = os.path.join(GOLDEN, "datasets", "ref_nvs_datasets.npz")


gen, fx, root = sequence_fixtures("nvs_datasets")


READS = ["scannetpp_train", "scannetpp_train_bad", "scannetpp_test", "scannetpp_test_bad", "replicav2_train",
         "replicav2_test", "replicav2_test_sel"]


def test_fixture_covers_every_case(gen, fx):
    assert os.path.getsize(FIX) < 1 << 20
    assert set(gen.READS) == set(READS) == {k[:-len("_retained")] for k in fx if k.endswith("_retained")}
    # ScanNet++: the JSON lists the frames in another order than train_test_lists.json
    meta = json.loads(bytes(fx["file_blobs"][slice(*fx["file_blobs_offsets"][
        fx["file_names"].tolist().index("scannetpp/8b5caf3398/dslr/nerfstudio/transforms_undistorted.json")])]))
    assert [f["file_path"] for f in meta["frames"]] != gen.SCANNETPP_TRAIN
    assert sum(f["is_bad"] for f in meta["frames"]) == 1 and sum(f["is_bad"] for f in meta["test_frames"]) == 1
    # ReplicaV2: more than 10 frames, so natural and lexical order differ
    names = fx["replicav2_train_color_names"].tolist()
    assert len(names) == 12 and names != sorted(names)


@pytest.mark.parametrize("read", READS)
def test_files_and_selection_match_reference(gen, fx, root, read):
    f = files_of(gen, root, read)
    base = os.path.join(root, gen.READS[read][0], gen.SEQUENCES[gen.READS[read][0]])
    assert [os.path.relpath(p, base) for p in f.color_paths] == fx[read + "_color_names"].tolist()
    assert [os.path.relpath(p, base) for p in f.depth_paths] == fx[read + "_depth_names"].tolist()
    assert f.retained_inds.tolist() == fx[read + "_retained"].tolist()
    assert len(f) == len(fx[read + "_retained"])


@pytest.mark.parametrize("read", READS)
def test_poses_and_intrinsics_bit_equal_to_reference(gen, fx, root, read):
    f = files_of(gen, root, read)
    assert f.poses.dtype == torch.float32
    assert bits_equal(f.poses.numpy(), fx[read + "_poses"])
    assert bits_equal(f.intrinsics.numpy(), fx[read + "_intrinsics"])


@pytest.mark.parametrize("read", READS)
def test_numpy_ingest_matches_reference_pixels(gen, fx, root, read):
    from oracle import ingest_numpy
    f = files_of(gen, root, read)
    for t in range(len(f)):
        rgb, depth = D.decode_color(f.color_paths[t]), D.decode_depth(f.depth_paths[t])
        color, d = ingest_numpy.ingest(rgb, depth, f.height, f.width, f.png_depth_scale)
        assert bits_equal(color, fx[read + "_color"][t]), (read, t)
        assert bits_equal(d, fx[read + "_depth"][t]), (read, t)


def test_test_split_starts_with_the_first_train_frame(gen, root):
    for dataset in ("scannetpp", "replicav2"):
        train, test = (files_of(gen, root, dataset + s) for s in ("_train", "_test"))
        assert test.color_paths[0] == train.color_paths[0] and test.depth_paths[0] == train.depth_paths[0]
        assert torch.equal(test.poses[0], train.poses[0]) and torch.allclose(test.poses[0], torch.eye(4), atol=1e-6)
    # the first train frame is is_bad: ignore_bad drops it from the train split but never from the test split
    bad_train, bad_test = files_of(gen, root, "scannetpp_train_bad"), files_of(gen, root, "scannetpp_test_bad")
    first = files_of(gen, root, "scannetpp_train").color_paths[0]
    assert first not in bad_train.color_paths and bad_test.color_paths[0] == first


def test_scannetpp_camera_comes_from_the_sequence(gen, root):
    cfg = D.scannetpp_config(os.path.join(root, "scannetpp", gen.SEQUENCES["scannetpp"]))["camera_params"]
    assert (cfg["image_height"], cfg["image_width"], cfg["fx"], cfg["fy"], cfg["cx"], cfg["cy"],
            cfg["png_depth_scale"]) == (48, 64, 50.25, 51.5, 31.75, 23.25, 1000.0)
    with pytest.raises(ValueError, match="no shipped data config"):
        D.default_config("scannetpp")
    v2 = D.default_config("replicav2")["camera_params"]
    assert (v2["image_height"], v2["image_width"], v2["fx"], v2["png_depth_scale"]) == (680, 1200, 600.0, 1000.0)


def test_error_cases(gen, root, tmp_path):
    seq = os.path.join(str(tmp_path), "scannetpp", "s")
    shutil.copytree(os.path.join(root, "scannetpp", gen.SEQUENCES["scannetpp"]), seq)
    os.remove(os.path.join(seq, "dslr", "train_test_lists.json"))
    with pytest.raises(FileNotFoundError, match="train_test_lists.json"):
        D.SequenceFiles("scannetpp", os.path.join(str(tmp_path), "scannetpp"), "s")
    with open(os.path.join(seq, "dslr", "train_test_lists.json"), "w") as f:
        json.dump(dict(train=gen.SCANNETPP_TRAIN, test=gen.SCANNETPP_TEST + ["DSC09999.JPG"]), f)
    D.SequenceFiles("scannetpp", os.path.join(str(tmp_path), "scannetpp"), "s")         # the train split is fine
    with pytest.raises(ValueError, match="DSC09999.JPG"):
        D.SequenceFiles("scannetpp", os.path.join(str(tmp_path), "scannetpp"), "s", split="test")
    # a test split only where the dataset has one; ignore_bad only for ScanNet++
    replica = os.path.join(str(tmp_path), "replica", "room0")
    os.makedirs(replica)
    for dataset in ("replica", "tum", "scannet"):
        with pytest.raises(ValueError, match="no 'test' split"):
            D.SequenceFiles(dataset, os.path.join(str(tmp_path), "replica"), "room0", split="test")
    with pytest.raises(ValueError, match="split must be"):
        files_of(gen, root, "replicav2_train").__class__("replicav2", os.path.join(root, "replicav2"),
                                                         gen.SEQUENCES["replicav2"], split="val")
    with pytest.raises(ValueError, match="ignore_bad"):
        D.SequenceFiles("replicav2", os.path.join(root, "replicav2"), gen.SEQUENCES["replicav2"], ignore_bad=True)
