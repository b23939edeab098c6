"""CPU: the saved-frame pixel rules of csrc/eval_frames.cu restated in numpy against the reference's own files
(tests/golden/eval/ref_eval_frames.npz), the JET table against cv2's, argument checks of sb_eval_frames_u8 before any
launch, no CPU fallback, save_frames without out_dir, and the argument and record checks of tools/eval_record.py."""
import ctypes
import os

import numpy as np
import pytest
import torch

from splatam_b200 import _lib, evaluate as EV, formats
from util import GOLDEN, load


@pytest.fixture(scope="module")
def gen():
    return load("tests/golden/eval/make_golden_eval_frames.py")


@pytest.fixture(scope="module")
def tool():
    return load("tools/eval_record.py")


def test_jet_table_is_cv2s():
    cv2 = pytest.importorskip("cv2")
    ref = cv2.applyColorMap(np.arange(256, dtype=np.uint8)[:, None], cv2.COLORMAP_JET)[:, 0, ::-1]
    assert EV.JET_RGB.shape == (256, 3) and EV.JET_RGB.dtype == np.uint8
    assert np.array_equal(EV.JET_RGB, ref)


def _rgb_rule(x):
    """round_half_even(clamp(x, 0, 1) * 255f), NaN -> 0, on [3,H,W] -> HWC."""
    x = x.numpy().transpose(1, 2, 0)
    with np.errstate(invalid="ignore"):
        v = np.clip(x, 0, 1) * np.float32(255)
    v[np.isnan(v)] = 0
    return np.rint(v).astype(np.uint8)


def _depth_rule(d):
    """JET_RGB[trunc(clip(d / 6f, 0, 1) * 255f)], NaN -> index 0, on [H,W]."""
    with np.errstate(invalid="ignore"):
        n = d.numpy() / np.float32(6)
        v = np.clip(n, 0, 1) * np.float32(255)
    v[np.isnan(v)] = 0
    return EV.JET_RGB[v.astype(np.uint8)]


def test_pixel_rules_reproduce_the_reference_files(gen):
    """The rules the kernel implements, restated in numpy, give every pixel of every file the reference wrote."""
    fx = np.load(os.path.join(GOLDEN, "eval", "ref_eval_frames.npz"))
    for name in gen.CASES:
        case = gen.frames_case(name)
        files = [str(f) for f in fx[name + "_files"]]
        assert len(files) == 4 * len(evaluate_ids(case))
        for f, px in zip(files, fx[name + "_pixels"]):
            sub, fname = f.split("/")
            i = int(fname.split("_")[1][:4])
            t = i if case["kind"] == "eval" else i + 1
            im, depth_sil = case["renders"][t]
            color, depth = case["dataset"][t][:2]
            want = {"rendered_rgb": lambda: _rgb_rule(im), "rgb": lambda: _rgb_rule(color.permute(2, 0, 1) / 255),
                    "rendered_depth": lambda: _depth_rule(depth_sil[0]),
                    "depth": lambda: _depth_rule(depth[..., 0])}[sub]()
            assert np.array_equal(want, px), (name, f)


def evaluate_ids(case):
    if case["kind"] == "eval":
        return EV.select_frames(len(case["dataset"]), case["eval_every"])
    return EV.select_nvs_frames(len(case["dataset"]), case["eval_every"])


def test_fixture_covers_the_special_values(gen):
    case = gen.frames_case("eval")
    im, depth_sil = case["renders"][0]
    gd = case["dataset"][0][1]
    for x in (im, depth_sil[0]):
        assert torch.isnan(x).any() and torch.isposinf(x).any() and torch.isneginf(x).any()
    assert (im < 0).any() and (im > 1).any()
    assert (np.float32(gen.tie_values().numpy()) * np.float32(255) % 1 == 0.5).all()
    for d in (depth_sil[0], gd):
        assert (d < 0).any() and (d == 0).any() and (d > 6).any()
        assert np.isin(((torch.arange(256) * 6.0) / 255).float().numpy(), d.numpy()).all()


def test_bad_arguments_are_rejected_before_any_launch():
    lib = _lib.load()
    ok = (1, 1, 1, 1, 4, 4, 1, 1, None)
    for i in (0, 1, 2, 3, 6, 7):                                   # a null pointer
        args = list(ok)
        args[i] = None
        assert lib.sb_eval_frames_u8(*args) == 1, i
    for H, W in ((0, 4), (4, 0), (-1, 4), (4, -3), (1 << 16, 1 << 16)):
        assert lib.sb_eval_frames_u8(1, 1, 1, 1, H, W, 1, 1, None) == 1, (H, W)
    assert _lib._SIGNATURES["sb_eval_frames_u8"][1][-1] is ctypes.c_void_p


def test_no_cpu_fallback():
    im, ds, d = torch.rand(3, 8, 8), torch.rand(3, 8, 8), torch.rand(1, 8, 8)
    with pytest.raises(_lib.SplatamB200Error, match="no CPU fallback"):
        EV.eval_frames_u8(im, ds, im, d)


def test_save_frames_needs_out_dir():
    frames = [dict(id=0, im=torch.rand(3, 8, 8), depth=torch.rand(1, 8, 8))]
    params = dict(means3D=torch.zeros(1, 3))
    with pytest.raises(ValueError, match="save_frames=True needs out_dir"):
        EV.evaluate(params, frames, None, 0.5, 30, True, save_frames=True)
    with pytest.raises(ValueError, match="save_frames=True needs out_dir"):
        EV.evaluate_nvs(params, frames, None, 0.5, 30, True, save_frames=True)


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


def _record(out_dir, T_cam, P=5):
    g = torch.Generator().manual_seed(0)
    gauss = dict(means3D=torch.randn(P, 3, generator=g), rgb_colors=torch.rand(P, 3, generator=g),
                 unnorm_rotations=torch.randn(P, 4, generator=g), logit_opacities=torch.zeros(P, 1),
                 log_scales=torch.full((P, 1), -3.0))
    rots = torch.zeros(1, 4, T_cam)
    rots[:, 0] = 1.0
    return formats.save_run_record(out_dir, gauss, rots, torch.zeros(1, 3, T_cam), torch.zeros(P), torch.eye(3),
                                   torch.eye(4), 1200, 680, [torch.eye(4)] * T_cam, list(range(T_cam)))


def test_eval_record_argument_errors(tool, tmp_path, capsys):
    rec = _record(str(tmp_path / "run"), 3)
    base = ["--dataset", "replica", "--basedir", str(tmp_path), "--sequence", "room0"]
    for argv, msg in ((base, "--record"),
                      (base + ["--record", str(tmp_path / "none.npz")], "no such file"),
                      (base + ["--record", rec, "--split", "test"], "--split test needs"),
                      (base + ["--record", rec, "--lpips-alexnet", "a.pth"], "go together"),
                      (base + ["--record", rec, "--frames", "-1"], "--frames"),
                      (["--dataset", "kitti", "--basedir", "x", "--sequence", "y", "--record", rec], "invalid choice")):
        with pytest.raises(SystemExit):
            tool.parse_args(argv)
        assert msg in capsys.readouterr().err, argv
    a = tool.parse_args(base + ["--record", rec])
    assert a.out == os.path.join(str(tmp_path / "run"), "eval_train") and not a.no_frames
    a = tool.parse_args(["--dataset", "replicav2", "--basedir", "b", "--sequence", "s", "--record", rec,
                         "--split", "test"])
    assert a.out == os.path.join(str(tmp_path / "run"), "eval_nvs")


def test_eval_record_checks_its_record_with_the_formats_reader(tool, tmp_path):
    """tools/eval_record.py reads the record with formats.read_record (the Gaussians, and the cameras on the train
    split) and names the first evaluated frame without a camera column (formats.check_camera_columns)."""
    _replica_layout(str(tmp_path), 12)
    rec = _record(str(tmp_path / "run"), 9)
    base = ["--dataset", "replica", "--basedir", str(tmp_path), "--sequence", "room0", "--record", rec]
    # Replica evaluates every 5th frame: 0, 4, 9 of 12 frames; the record has columns 0 .. 8
    with pytest.raises(ValueError, match="has 9 camera columns; frame index 9 has none"):
        tool.main(base)
    train = formats.read_record(rec, formats.CHECKPOINT_KEYS)
    with pytest.raises(ValueError, match="has 9 camera columns; frame index 9 has none"):
        formats.check_camera_columns(rec, train, EV.select_frames(10, 5))
    formats.check_camera_columns(rec, train, EV.select_frames(9, 5))
    assert train["cam_trans"].shape[-1] == 9
    assert formats.read_record(rec, formats.GAUSSIAN_KEYS)["means3D"].shape == (5, 3)
    partial = str(tmp_path / "partial.npz")
    np.savez(partial, **{k: v for k, v in np.load(rec).items() if k != "cam_trans"})
    with pytest.raises(ValueError, match="lacks cam_trans"):
        tool.main(base[:-1] + [partial])
