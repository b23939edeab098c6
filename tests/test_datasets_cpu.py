"""CPU: the host side of the dataset readers (splatam_b200/datasets.py) and the float64 restatement of the ingest
kernel (oracle/ingest_numpy.py) against the reference's own dataset classes, run unmodified on tiny synthetic Replica,
TUM and ScanNet sequences (tests/golden/datasets/ref_datasets.npz, written by make_golden_datasets.py): file discovery
and natural order, start / end / stride, TUM's association and 1/32 s subsampling, poses and intrinsics bit for bit,
colour and depth bit for bit; argument checks of sb_ingest_rgbd; no CPU fallback."""
import os

import numpy as np
import pytest
import torch

from dataset_fixtures import files_of, sequence_fixtures
from util import GOLDEN, bits_equal
from splatam_b200 import _lib
from splatam_b200 import datasets as D

FIX = os.path.join(GOLDEN, "datasets", "ref_datasets.npz")


gen, fx, root = sequence_fixtures("datasets")


def test_fixture_covers_every_case(gen, fx):
    assert os.path.getsize(FIX) < 1 << 20
    assert set(gen.READS) == {k[:-len("_retained")] for k in fx if k.endswith("_retained")}
    assert fx["replica_all_color_names"].size == 12
    assert np.isinf(fx["scannet_mixed_poses"]).any() or np.isnan(fx["scannet_mixed_poses"]).any()


@pytest.mark.parametrize("read", ["replica_all", "replica_native", "replica_down", "replica_up", "replica_half",
                                  "tum_up", "scannet_mixed"])
def test_discovery_order_and_selection_match_reference(gen, fx, root, read):
    f = files_of(gen, root, read)
    base = os.path.join(root, gen.READS[read][0], gen.SEQUENCES[gen.READS[read][0]])
    assert [os.path.relpath(p, base) for p in f.color_paths] == fx[read + "_color_names"].tolist()
    assert [os.path.relpath(p, base) for p in f.depth_paths] == fx[read + "_depth_names"].tolist()
    assert f.retained_inds.tolist() == fx[read + "_retained"].tolist()
    assert len(f) == len(fx[read + "_retained"])


def test_natural_order_differs_from_lexical(gen, fx, root):
    names = fx["replica_all_color_names"].tolist()
    assert names[:3] == ["results/frame0.jpg", "results/frame1.jpg", "results/frame2.jpg"]
    assert names != sorted(names)
    assert D.natsorted(["a10.png", "a9.png", "a100.png"]) == ["a9.png", "a10.png", "a100.png"]


def test_tum_association_drops_unpaired_and_too_close_frames(gen, fx, root):
    t_img = np.array([float(r.split()[0]) for r in open(os.path.join(root, "tum", gen.SEQUENCES["tum"], "rgb.txt"))
                      if not r.startswith("#")])
    f = D.SequenceFiles("tum", os.path.join(root, "tum"), gen.SEQUENCES["tum"], gen.config("tum"))
    assert 0 < len(f) <= t_img.size - 3           # a pose gap and sub-1/32 s steps drop frames
    kept = np.array([float(os.path.basename(p)[:-4]) for p in f.color_paths])
    assert (np.diff(kept) > 1.0 / 32).all()
    assert D.tum_associate(np.array([0.0, 0.01, 0.05, 0.2]), np.array([0.0, 0.05, 0.21]),
                           np.array([0.0, 0.06, 0.19])) == [(0, 0, 0), (2, 1, 1), (3, 2, 2)]


@pytest.mark.parametrize("read", ["replica_all", "replica_native", "replica_down", "replica_up", "replica_half",
                                  "tum_up", "scannet_mixed"])
def test_poses_and_intrinsics_bit_equal_to_reference(gen, fx, root, read):
    f = files_of(gen, root, read)
    assert f.poses.dtype == torch.float32
    assert bits_equal(f.poses.numpy(), fx[read + "_poses"])
    assert bits_equal(f.intrinsics.numpy(), fx[read + "_intrinsics"])


@pytest.mark.parametrize("read", ["replica_native", "replica_down", "replica_up", "replica_half", "tum_up",
                                  "scannet_mixed"])
def test_numpy_ingest_matches_reference_pixels(gen, fx, root, read):
    from oracle import ingest_numpy
    f = files_of(gen, root, read)
    for t in range(len(f)):
        rgb, depth = D.decode_color(f.color_paths[t]), D.decode_depth(f.depth_paths[t])
        color, d = ingest_numpy.ingest(rgb, depth, f.height, f.width, f.png_depth_scale)
        assert bits_equal(color, fx[read + "_color"][t]), (read, t)
        assert bits_equal(d, fx[read + "_depth"][t]), (read, t)


def test_selection_arguments_are_checked(gen, root):
    args = ("replica", os.path.join(root, "replica"), gen.SEQUENCES["replica"], gen.config("replica"))
    with pytest.raises(ValueError, match="start"):
        D.SequenceFiles(*args, start=-1)
    with pytest.raises(ValueError, match="end"):
        D.SequenceFiles(*args, start=4, end=4)
    with pytest.raises(FileNotFoundError, match="no such sequence"):
        D.SequenceFiles("replica", os.path.join(root, "replica"), "missing", gen.config("replica"))


def test_default_configs_are_the_shipped_ones():
    r = D.default_config("replica")["camera_params"]
    assert (r["image_height"], r["image_width"], r["fx"], r["cx"], r["png_depth_scale"]) == (680, 1200, 600.0, 599.5,
                                                                                              6553.5)
    assert D.default_config("tum", "rgbd_dataset_freiburg1_desk")["camera_params"]["fx"] == 517.3
    assert D.default_config("tum", "rgbd_dataset_freiburg2_xyz")["camera_params"]["fx"] == 520.9
    assert D.default_config("tum", "rgbd_dataset_freiburg3_long_office_household")["camera_params"]["fy"] == 539.2
    s = D.default_config("scannet")["camera_params"]
    assert (s["image_height"], s["image_width"], s["png_depth_scale"]) == (968, 1296, 1000.0)
    with pytest.raises(ValueError, match="unknown dataset"):
        D.default_config("icl")


def test_yaml_config_of_the_reference_shape(tmp_path):
    p = tmp_path / "data.yaml"
    p.write_text("dataset_name: 'tum'\ncamera_params:\n  image_height: 480\n  image_width: 640\n  fx: 535.4\n"
                 "  fy: 539.2\n  cx: 320.1\n  cy: 247.6\n  crop_edge: 8\n  png_depth_scale: 5000.0\n")
    cfg = D.load_config(str(p))
    assert cfg["camera_params"]["fx"] == 535.4 and cfg["camera_params"]["crop_edge"] == 8
    p.write_text("camera_params:\n  image_height: 480\n")
    with pytest.raises(ValueError, match="lacks"):
        D.load_config(str(p))


def test_non_rgb_colour_is_rejected(tmp_path):
    from PIL import Image
    p = str(tmp_path / "gray.png")
    Image.fromarray(np.zeros((4, 5), np.uint8)).save(p)
    with pytest.raises(ValueError, match="3-channel"):
        D.decode_color(p)
    p = str(tmp_path / "rgba.png")
    Image.fromarray(np.zeros((4, 5, 4), np.uint8)).save(p)
    with pytest.raises(ValueError, match="3-channel"):
        D.decode_color(p)


def test_ingest_bad_arguments_are_rejected_before_any_launch():
    lib = _lib.load()
    f = lib.sb_ingest_rgbd
    assert f(None, 4, 4, 1, 4, 4, 4, 4, 1000.0, 1, 1, None) == 1              # null colour
    assert f(1, 4, 4, None, 4, 4, 4, 4, 1000.0, 1, 1, None) == 1              # null depth
    assert f(1, 4, 4, 1, 4, 4, 4, 4, 1000.0, None, 1, None) == 1              # null output
    assert f(1, 4, 4, 1, 4, 4, 4, 4, 1000.0, 1, None, None) == 1
    assert f(1, 0, 4, 1, 4, 4, 4, 4, 1000.0, 1, 1, None) == 1                 # non-positive sizes
    assert f(1, 4, 4, 1, 4, -1, 4, 4, 1000.0, 1, 1, None) == 1
    assert f(1, 4, 4, 1, 4, 4, 0, 4, 1000.0, 1, 1, None) == 1
    assert f(1, 4, 4, 1, 4, 4, 4, 4, 0.0, 1, 1, None) == 1                    # depth scale must be positive
    assert lib.sb_status_string(1) == b"SB_ERR_BAD_ARG"


def test_no_cpu_fallback(gen, root):
    rgb, depth = torch.zeros(4, 4, 3, dtype=torch.uint8), torch.zeros(4, 4, dtype=torch.uint16)
    with pytest.raises(_lib.SplatamB200Error, match="no CPU fallback"):
        D.ingest_rgbd(rgb, depth, 4, 4, 1000.0)
    seq = D.RGBDSequence("replica", os.path.join(root, "replica"), gen.SEQUENCES["replica"], gen.config("replica"),
                         device="cpu", prefetch=0)
    assert len(seq) == 12 and seq.cam.image_width == 64
    with pytest.raises(_lib.SplatamB200Error, match="no CPU fallback"):
        seq[0]
