"""CPU: the float64 metric oracle (oracle/metrics_torch.py) and the host side of splatam_b200.evaluate against the
reference's own final `eval`, run unmodified with preset renders (tests/golden/eval/ref_eval.npz, written by
tests/golden/eval/make_golden_eval.py); argument checks of the metric entry points; no CPU fallback."""
import ctypes
import os

import numpy as np
import pytest
import torch

from util import GOLDEN, load

FIX = os.path.join(GOLDEN, "eval", "ref_eval.npz")


@pytest.fixture(scope="module")
def gen():
    return load("tests/golden/eval/make_golden_eval.py")


@pytest.fixture(scope="module")
def fx():
    return np.load(FIX)


def frame_inputs(case, t):
    """(im, depth_sil, gt_im [3,H,W], gt_depth [1,H,W]) of frame t as the reference's eval forms them."""
    color, depth, _, _ = case["dataset"][t]
    im, depth_sil = case["renders"][t]
    return im, depth_sil, color.permute(2, 0, 1) / 255, depth.permute(2, 0, 1)


@pytest.mark.parametrize("name", ["masked", "unmasked_every3"])
def test_oracle_reproduces_reference_eval(gen, fx, name):
    from oracle import metrics_torch as O
    from splatam_b200.evaluate import select_frames
    case = gen.eval_case(name)
    ids = select_frames(len(case["dataset"]), case["eval_every"])
    assert ids == fx[name + "_ids"].tolist()
    use_presence = case["mapping_iters"] == 0 and not case["add_new_gaussians"]
    for k, t in enumerate(ids):
        m = O.frame_metrics(*frame_inputs(case, t), case["sil_thres"], use_presence)
        assert abs(float(m["psnr"]) - fx[name + "_psnr"][k]) < 1e-4, (t, float(m["psnr"]))
        for key, ref in (("depth_rmse", "rmse"), ("depth_l1", "l1")):
            assert abs(float(m[key]) / fx[name + "_" + ref][k] - 1) < 1e-5, (t, key)
        assert int(m["n_valid"]) == fx[name + "_n_valid"][k] and int(m["n_mask"]) == fx[name + "_n_mask"][k]
        s = O.ms_ssim(m["weighted_im"][None], m["weighted_gt"][None])
        assert abs(float(s) - fx[name + "_ssim"][k]) < 1e-12, t
    if not use_presence:
        assert (fx[name + "_n_mask"] == fx[name + "_n_valid"]).all()


@pytest.mark.parametrize("name", ["masked", "unmasked_every3"])
def test_trajectory_ate_matches_reference(gen, fx, name):
    """Estimated frame 0 is the first frame's w2c; the frame whose ground-truth pose holds NaN is skipped."""
    from splatam_b200.evaluate import trajectory_ate
    case = gen.eval_case(name)
    gt_w2c = [torch.linalg.inv(pose) for _, _, _, pose in case["dataset"]]
    assert sum(bool(torch.isnan(m).any()) for m in gt_w2c) == 1
    ate = trajectory_ate(case["params"], gt_w2c[0], gt_w2c)
    # the reference centres the float32 point arrays in float32 (eval_helpers.py:37-38); slam.ate_horn works in double,
    # so the two agree to float32 rounding of those means (1.5e-9 of 0.013 m here), not to the last double bit
    assert abs(ate - float(fx[name + "_ate"])) < 1e-6 * float(fx[name + "_ate"]), ate


def test_select_frames():
    from splatam_b200.evaluate import select_frames
    assert select_frames(7, 1) == list(range(7))
    assert select_frames(7, 3) == [0, 2, 5]
    assert select_frames(1, 5) == [0]


def test_oracle_ms_ssim_of_identical_images_is_one():
    from oracle import metrics_torch as O
    g = torch.Generator().manual_seed(0)
    x = torch.rand(2, 3, 171, 199, generator=g)
    assert float(O.ms_ssim(x, x.clone())) == 1.0
    assert torch.equal(O.ms_ssim(x, x.clone(), size_average=False), torch.ones(2, 3, dtype=torch.float64))
    with pytest.raises(ValueError):
        O.ms_ssim(x[..., :160, :], x[..., :160, :])


def test_metric_entry_points_reject_bad_arguments_before_any_launch():
    from splatam_b200 import _lib
    lib = _lib.load()
    n = ctypes.c_size_t(0)
    assert lib.sb_frame_metrics_workspace_bytes(171, 199, ctypes.byref(n)) == 0 and n.value > 0
    assert lib.sb_frame_metrics_workspace_bytes(0, 199, ctypes.byref(n)) == 1
    assert lib.sb_frame_metrics_workspace_bytes(171, 199, None) == 1
    assert lib.sb_ms_ssim_workspace_bytes(1, 3, 171, 199, ctypes.byref(n)) == 0 and n.value > 0
    for N, C, H, W in ((0, 3, 171, 199), (1, 0, 171, 199), (1, 3, 160, 199), (1, 3, 199, 160), (1, 3, -5, 199)):
        assert lib.sb_ms_ssim_workspace_bytes(N, C, H, W, ctypes.byref(n)) == 1, (N, C, H, W)
    big = 1 << 30
    # non-null dummy pointers are never dereferenced: every check comes before the first CUDA call
    assert lib.sb_frame_metrics(None, 1, 1, 1, 8, 8, 0.5, 1, 1, 1, 1, big, 1, None) == 1
    assert lib.sb_frame_metrics(1, 1, 1, 1, 8, 8, 0.5, 1, 1, None, 1, big, 1, None) == 1
    assert lib.sb_frame_metrics(1, 1, 1, 1, 8, 8, 0.5, 1, 1, 1, 1, big, None, None) == 1
    assert lib.sb_frame_metrics(1, 1, 1, 1, 0, 8, 0.5, 1, 1, 1, 1, big, 1, None) == 1
    assert lib.sb_frame_metrics(1, 1, 1, 1, 8, -1, 0.5, 1, 1, 1, 1, big, 1, None) == 1
    assert lib.sb_frame_metrics(1, 1, 1, 1, 8, 8, 0.5, 1, 1, 1, 1, 0, 1, None) == 2          # SB_ERR_WORKSPACE
    assert lib.sb_ms_ssim(None, 1, 1, 3, 171, 199, 1.0, 1, big, 1, 1, None) == 1
    assert lib.sb_ms_ssim(1, 1, 1, 3, 171, 199, 1.0, None, big, 1, 1, None) == 1
    assert lib.sb_ms_ssim(1, 1, 1, 3, 171, 199, 1.0, 1, big, None, None, None) == 1        # nowhere to write
    assert lib.sb_ms_ssim(1, 1, 1, 3, 160, 199, 1.0, 1, big, 1, 1, None) == 1              # smaller side of 160
    assert lib.sb_ms_ssim(1, 1, 1, 3, 171, 160, 1.0, 1, big, 1, 1, None) == 1
    assert lib.sb_ms_ssim(1, 1, 0, 3, 171, 199, 1.0, 1, big, 1, 1, None) == 1
    assert lib.sb_ms_ssim(1, 1, 1, 3, 171, 199, 1.0, 1, 16, 1, 1, None) == 2               # SB_ERR_WORKSPACE


def test_no_cpu_fallback(gen):
    import splatam_b200 as S
    from splatam_b200 import evaluate as EV
    x = torch.rand(1, 3, 171, 199)
    with pytest.raises(S.SplatamB200Error, match="no CPU fallback"):
        EV.ms_ssim(x, x)
    case = gen.eval_case("masked")
    frames = [dict(id=t, im=f[2], depth=f[3], w2c=torch.eye(4)) for t, f in
              enumerate(frame_inputs(case, t) for t in range(len(case["dataset"])))]
    with pytest.raises(S.SplatamB200Error, match="no CPU fallback"):
        EV.evaluate(case["params"], frames, None, 0.5, 0, False)
