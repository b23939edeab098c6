"""CPU: formats.read_record, the one checked reader of a run record, driven with the `need` of each of its callers: a
valid record reads as np.load gives it, and each malformed one raises the same message whichever tool opens it --
offline.from_record, tools/eval_record.py and tools/render_record.py --camera-from included."""
import os

import numpy as np
import pytest
import torch

from util import load
from splatam_b200 import formats, offline


NEEDS = {
    "viewer": formats.CHECKPOINT_KEYS + formats.CAMERA_KEYS,      # viewer.load_record, mesh.RecordFusion, extract_mesh
    "offline": formats.CHECKPOINT_KEYS + ("timestep",),            # offline.from_record
    "eval_train": formats.CHECKPOINT_KEYS,                         # tools/eval_record.py --split train
    "eval_test": formats.GAUSSIAN_KEYS,                            # tools/eval_record.py --split test
    "camera_from": formats.CAMERA_KEYS,                            # tools/render_record.py --camera-from
}
WITH_CAMERAS = ("viewer", "offline", "eval_train")


def _record(out_dir, T=4, P=6, **override):
    """A save_run_record record with T cameras and P Gaussians; override: key -> array, or None to drop the key."""
    g = np.random.default_rng(0)
    gauss = {k: g.normal(size=(P, w)) for k, w in zip(formats.GAUSSIAN_KEYS, (3, 3, 4, 1, 1))}
    rots = np.zeros((1, 4, T), np.float32)
    rots[0, 0] = 1
    path = formats.save_run_record(str(out_dir), gauss, rots, g.normal(size=(1, 3, T)), np.arange(P) % T, np.eye(3),
                                   np.eye(4), 64, 48, [np.eye(4)] * T, list(range(T)))
    if override:
        raw = dict(np.load(path))
        for k, v in override.items():
            if v is None:
                raw.pop(k)
            else:
                raw[k] = v
        np.savez(path, **raw)
    return path


@pytest.mark.parametrize("caller", sorted(NEEDS))
def test_a_valid_record_reads_as_np_load_gives_it(tmp_path, caller):
    path = _record(tmp_path)
    ref = dict(np.load(path, allow_pickle=True))
    rec = formats.read_record(path, NEEDS[caller])
    assert list(rec) == list(ref)
    for k in ref:
        assert rec[k].dtype == ref[k].dtype and np.array_equal(rec[k], ref[k]), k
    cam = formats.read_record(path, NEEDS[caller], camera=dict(org_width=640, intrinsics=2 * np.eye(3)))
    assert cam["org_width"] == 640 and np.array_equal(cam["intrinsics"], 2 * np.eye(3))
    assert np.array_equal(cam["w2c"], ref["w2c"])


@pytest.mark.parametrize("caller", sorted(NEEDS))
def test_a_missing_key_is_named(tmp_path, caller):
    need = NEEDS[caller]
    for i, k in enumerate((need[0], need[-1])):
        path = _record(tmp_path / str(i), **{k: None})
        with pytest.raises(ValueError, match="params.npz lacks %s" % k) as e:
            formats.read_record(path, need)
        assert ("a checkpoint holds no camera" in str(e.value)) == (k in formats.CAMERA_KEYS), k


def test_a_checkpoint_needs_the_camera_given(tmp_path):
    formats.save_checkpoint(str(tmp_path / "ckpt"), 3, dict(np.load(_record(tmp_path))), [0])
    path = str(tmp_path / "ckpt" / "params3.npz")
    with pytest.raises(ValueError, match="lacks intrinsics, w2c, org_width, org_height .a checkpoint holds no camera"):
        formats.read_record(path, NEEDS["viewer"])
    camera = dict(intrinsics=np.eye(3), w2c=np.eye(4), org_width=64, org_height=48)
    rec = formats.read_record(path, NEEDS["viewer"], camera=camera)
    assert set(rec) == set(formats.CHECKPOINT_KEYS + formats.CAMERA_KEYS)
    with pytest.raises(ValueError, match="lacks timestep$"):
        formats.read_record(path, NEEDS["offline"])


BAD_CAMERAS = {
    "fewer cam_trans columns": dict(cam_trans=np.zeros((1, 3, 3), np.float32)),
    "fewer cam_unnorm_rots columns": dict(cam_unnorm_rots=np.zeros((1, 4, 2), np.float32)),
    "cam_unnorm_rots not [1,4,T]": dict(cam_unnorm_rots=np.zeros((4, 4), np.float32)),
    "cam_trans not [1,3,T]": dict(cam_trans=np.zeros((1, 4, 4), np.float32)),
    "no camera": dict(cam_unnorm_rots=np.zeros((1, 4, 0), np.float32), cam_trans=np.zeros((1, 3, 0), np.float32)),
}


@pytest.mark.parametrize("caller", sorted(NEEDS))
@pytest.mark.parametrize("bad", sorted(BAD_CAMERAS))
def test_camera_shapes_are_checked_where_the_cameras_are_needed(tmp_path, caller, bad):
    path = _record(tmp_path, **BAD_CAMERAS[bad])
    if caller in WITH_CAMERAS:
        with pytest.raises(ValueError, match=r"camera count mismatch: cam_unnorm_rots .* must be \[1,4,T\]"):
            formats.read_record(path, NEEDS[caller])
    else:
        formats.read_record(path, NEEDS[caller])


@pytest.mark.parametrize("caller", sorted(NEEDS))
def test_row_counts_follow_means3d(tmp_path, caller):
    for k in formats.GAUSSIAN_KEYS[1:] + ("timestep",):
        path = _record(tmp_path / k, **{k: np.zeros((7, 1), np.float32)})
        with pytest.raises(ValueError, match="%s has 7 rows for 6 Gaussians" % k):
            formats.read_record(path, NEEDS[caller])
    path = _record(tmp_path / "no_timestep", timestep=None)
    if caller == "offline":
        with pytest.raises(ValueError, match="lacks timestep"):
            formats.read_record(path, NEEDS[caller])
    else:
        assert "timestep" not in formats.read_record(path, NEEDS[caller])


def test_camera_columns(tmp_path):
    path = _record(tmp_path, T=4)
    rec = formats.read_record(path, formats.CHECKPOINT_KEYS)
    formats.check_camera_columns(path, rec, [0, 3, 1])
    for idx, first in (([0, 4, 9], 4), ([2, -1, 7], -1)):
        with pytest.raises(ValueError, match="params.npz has 4 camera columns; frame index %d has none" % first):
            formats.check_camera_columns(path, rec, idx)


def test_record_tensors_are_contiguous_float32():
    rec = dict(a=np.arange(12, dtype=np.float64).reshape(3, 4).T / 3, b=np.ones((2, 1), np.float32))
    t = formats.record_tensors(rec, ("a",), "cpu")
    assert list(t) == ["a"] and t["a"].dtype == torch.float32 and t["a"].is_contiguous()
    assert np.array_equal(t["a"].numpy(), rec["a"].astype(np.float32))


def test_offline_from_record_rejects_a_malformed_record_at_read_time(tmp_path):
    frames, idx = [dict(), dict()], [0, 3]
    path = _record(tmp_path / "cams", cam_trans=np.zeros((1, 3, 3), np.float32))
    with pytest.raises(ValueError, match="camera count mismatch"):
        offline.from_record(path, frames, idx, "cpu")
    path = _record(tmp_path / "rows", rgb_colors=np.zeros((5, 3), np.float32))
    with pytest.raises(ValueError, match="rgb_colors has 5 rows for 6 Gaussians"):
        offline.from_record(path, frames, idx, "cpu")


def _replica_layout(root, T):
    """The file layout of a Replica sequence with T tiny frames (the reader's file discovery needs no pixels)."""
    from PIL import Image
    d = os.path.join(root, "room0", "results")
    os.makedirs(d)
    for t in range(T):
        Image.fromarray(np.zeros((8, 8, 3), np.uint8)).save(os.path.join(d, "frame%06d.jpg" % t))
        Image.fromarray(np.zeros((8, 8), np.uint16)).save(os.path.join(d, "depth%06d.png" % t))
    with open(os.path.join(root, "room0", "traj.txt"), "w") as f:
        f.write("".join(" ".join(str(v) for v in np.eye(4).reshape(-1)) + "\n" for _ in range(T)))


def test_eval_record_rejects_a_malformed_record_at_read_time(tmp_path):
    tool = load("tools/eval_record.py")
    _replica_layout(str(tmp_path), 12)
    base = ["--dataset", "replica", "--basedir", str(tmp_path), "--sequence", "room0", "--record"]
    # 12 cameras with one cam_trans column short: each evaluated frame (0, 4, 9) still has a column in both tensors
    path = _record(tmp_path / "cams", T=12, cam_trans=np.zeros((1, 3, 11), np.float32))
    with pytest.raises(ValueError, match="camera count mismatch"):
        tool.main(base + [path])
    path = _record(tmp_path / "rows", T=12, timestep=np.zeros(5, np.float32))
    with pytest.raises(ValueError, match="timestep has 5 rows for 6 Gaussians"):
        tool.main(base + [path])


def test_render_record_camera_from_names_what_it_lacks(tmp_path):
    tool = load("tools/render_record.py")
    path = _record(tmp_path / "run")
    formats.save_checkpoint(str(tmp_path / "ckpt"), 3, dict(np.load(path)), [0])
    ckpt = str(tmp_path / "ckpt" / "params3.npz")
    with pytest.raises(ValueError, match="params3.npz lacks intrinsics, w2c, org_width, org_height"):
        tool.main(["--record", ckpt, "--out", str(tmp_path / "viz"), "--camera-from", ckpt])
