"""CPU: SplaTAM-S's densification resolution on the host side -- the reader's size arguments, its densification
intrinsics and camera against the reference's own initialize_first_timestep (tests/golden/slam_s/ref_splatam_s.npz,
written by make_golden_splatam_s.py), the SLAM loop's choice of frame for map growth, and the tool's variant check."""
import importlib.util
import os
import sys

import numpy as np
import pytest
import torch

import scenes
from util import GOLDEN
from oracle import bruteforce_torch as BF
from splatam_b200 import datasets as D
from splatam_b200 import mapping as M
from splatam_b200 import slam

ROOT = os.path.dirname(os.path.dirname(GOLDEN))
FIX = os.path.join(GOLDEN, "slam_s", "ref_splatam_s.npz")
CAM_FIELDS = ("image_height", "image_width", "tanfovx", "tanfovy", "viewmatrix", "projmatrix", "campos")


def _load(name, path):
    spec = importlib.util.spec_from_file_location(name, path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


@pytest.fixture(scope="module")
def gen():
    return _load("make_golden_datasets", os.path.join(GOLDEN, "datasets", "make_golden_datasets.py"))


@pytest.fixture(scope="module")
def sgen():
    return _load("make_golden_splatam_s", os.path.join(GOLDEN, "slam_s", "make_golden_splatam_s.py"))


@pytest.fixture(scope="module")
def fx():
    return dict(np.load(FIX))


@pytest.fixture(scope="module")
def root(gen, tmp_path_factory):
    d = str(tmp_path_factory.mktemp("sequences"))
    gen.write_sequences(d, np.load(os.path.join(GOLDEN, "datasets", "ref_datasets.npz")))
    return d


def replica(gen, root, kw, **extra):
    return D.RGBDSequence("replica", os.path.join(root, "replica"), gen.SEQUENCES["replica"], gen.config("replica"),
                          device="cpu", prefetch=0, **dict(kw, **extra))


def bits_equal(a, b):
    a, b = np.asarray(a), np.asarray(b)
    return a.shape == b.shape and a.dtype == b.dtype and a.tobytes() == b.tobytes()


def field(cam, k):
    v = getattr(cam, k)
    return v.cpu().numpy() if torch.is_tensor(v) else np.asarray(v)


@pytest.mark.parametrize("bad", [dict(densify_height=24), dict(densify_width=32), dict(densify_height=0, densify_width=32),
                                 dict(densify_height=24, densify_width=-32), dict(densify_height=24.0, densify_width=32),
                                 dict(densify_height=True, densify_width=32), dict(densify_height="24", densify_width=32)])
def test_densify_size_arguments_are_checked(gen, sgen, root, bad):
    with pytest.raises(ValueError, match="densify"):
        replica(gen, root, sgen.DESIRED, **bad)


def test_densify_intrinsics_and_camera_bit_equal_to_reference(gen, sgen, fx, root):
    seq = replica(gen, root, sgen.DESIRED, densify_height=24, densify_width=32)
    assert (seq.densify_height, seq.densify_width) == (24, 32)
    assert bits_equal(seq.densify_intrinsics.numpy(), fx["init_densify_intrinsics"])
    assert bits_equal(seq.intrinsics.numpy(), fx["init_intrinsics"])
    assert bits_equal(seq.w2c.numpy(), fx["init_first_frame_w2c"])
    for tag, cam in (("densify_cam", seq.densify_cam), ("cam", seq.cam)):
        for k in CAM_FIELDS:
            a, b = field(cam, k), fx["init_%s_%s" % (tag, k)]
            if k.startswith("image_"):
                assert int(a) == int(b), (tag, k)
            else:
                assert bits_equal(a.astype(b.dtype), b) and a.dtype == b.dtype, (tag, k, a, b)
    # the reference's densification dataset at 24x32 is the replica_half read of ref_datasets.npz
    half = np.load(os.path.join(GOLDEN, "datasets", "ref_datasets.npz"))["replica_half_intrinsics"]
    assert bits_equal(half[:3, :3], fx["init_densify_intrinsics"])


def test_no_separate_resolution_at_the_desired_size(gen, sgen, root):
    for extra in ({}, dict(densify_height=48, densify_width=64)):
        seq = replica(gen, root, sgen.DESIRED, **extra)
        assert seq.densify_height is None and seq.densify_width is None
        assert seq.densify_cam is None and seq.densify_intrinsics is None


def test_default_desired_size_is_the_config_size(gen, root):
    seq = replica(gen, root, dict(start=1, end=11, stride=5), densify_height=24, densify_width=32)
    assert (seq.height, seq.width) == (48, 64) and seq.densify_cam.image_height == 24
    seq = replica(gen, root, dict(start=1, end=11, stride=5), densify_height=48, densify_width=64)
    assert seq.densify_cam is None


def _cpu_render(settings, means3D, means2D, opacities, colors_precomp, scales, rotations):
    out = BF.render(means3D, colors_precomp, opacities, scales, rotations, width=settings.image_width,
                    height=settings.image_height, tanfovx=settings.tanfovx, tanfovy=settings.tanfovy, bg=settings.bg,
                    viewmatrix=settings.viewmatrix[0], projmatrix=settings.projmatrix[0], means2D=means2D,
                    dtype=torch.float32)
    return out["color"], out["radii"], out["depth"]


def test_run_slam_grows_the_map_from_the_densify_entry(monkeypatch):
    """Mapped frames that carry ``densify`` are grown from it with its own intrinsics; frames without it from
    themselves with the `intrinsics` argument; no mapping window ever holds a ``densify`` entry.  (Map growth itself is
    CUDA only: here it is recorded, not run.)"""
    import splatam_b200 as S
    torch.set_num_threads(4)
    sc = scenes.config1(seed=8, P=120, w=48, h=32)
    cam = sc.settings(S.GaussianRasterizationSettings, "cpu")
    gt = dict(means3D=sc.means3D, rgb_colors=sc.colors, unnorm_rotations=sc.rotations,
              logit_opacities=torch.logit(sc.opacities.clamp(0.05, 0.95)), log_scales=torch.log(sc.scales[:, :1]))
    T = 5
    rots, trans = slam.look_trajectory(T, "cpu", step=(0.004, -0.002, 0.003), rot_step=(0.001, -0.001, 0.0005))
    frames = [slam.render_frame(gt, rots, trans, t, cam, render=_cpu_render) for t in range(T)]
    K = torch.tensor([[sc.fx, 0, sc.cx], [0, sc.fy, sc.cy], [0, 0, 1]])
    K_d = K.clone()
    K_d[:2] *= 0.5
    for t in (0, 1, 2, 4):                        # frame 3 has no densification copy
        frames[t]["densify"] = dict(id=t, cam=None, w2c=frames[t]["w2c"], im=frames[t]["im"][:, ::2, ::2],
                                    depth=frames[t]["depth"][:, ::2, ::2], intrinsics=K_d)
    grown, windows = [], []
    monkeypatch.setattr(M.ShardedMapper, "add_new_gaussians",
                        lambda self, frame, t, intrinsics, sil: grown.append((frame, t, intrinsics)) or 0)
    step = M.ShardedMapper.step

    def recording_step(self, window, *a, **k):
        windows.append(window)
        return step(self, window, *a, **k)
    monkeypatch.setattr(M.ShardedMapper, "step", recording_step)
    torch.manual_seed(1); np.random.seed(1)
    slam.run_slam(gt, frames, cam, render=_cpu_render, fused=False, tracking_iters=2, mapping_iters=1,
                  keyframe_every=2, map_every=1, window=3, intrinsics=K, add_new_gaussians=True,
                  select_keyframes=True, first_frame_iters=1)
    assert [t for _, t, _ in grown] == [1, 2, 3, 4]
    for frame, t, intrinsics in grown:
        if t == 3:
            assert frame is frames[3] and intrinsics is K
        else:
            assert frame is frames[t]["densify"] and intrinsics is K_d
    assert windows and all("densify" not in f for w in windows for f in w)
    assert all("densify" in frames[t] for t in (0, 1, 2, 4))          # the caller's frames are left as they were


def test_tool_accepts_splatam_s_for_replica_only(monkeypatch, capsys):
    tool = _load("run_slam_dataset", os.path.join(ROOT, "tools", "run_slam_dataset.py"))
    assert set(tool.HYPER_S) == {"replica"}
    row = tool.HYPER_S["replica"]
    assert (row["height"], row["width"], row["densify_height"], row["densify_width"]) == (680, 1200, 340, 600)
    assert (row["tracking_iters"], row["mapping_iters"], row["window"]) == (10, 15, 32)
    for dataset in ("tum", "scannet", "scannetpp", "replicav2"):
        monkeypatch.setattr(sys, "argv", ["run_slam_dataset.py", "--dataset", dataset, "--basedir", "x",
                                          "--sequence", "y", "--variant", "splatam_s"])
        with pytest.raises(SystemExit) as e:
            tool.main()
        assert e.value.code == 2 and "splatam_s" in capsys.readouterr().err, dataset
