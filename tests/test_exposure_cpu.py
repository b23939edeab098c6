"""CPU: per-frame exposure (train_ops.exposure_torch, oracle/exposure_numpy.py, slam.run_slam's `exposure`,
formats.save_exposure / load_exposure) on the torch path, with the float32 brute-force composite from oracle/ standing
in for the rasterizer.  The kernels themselves and the fused and captured paths are tests/test_exposure_gpu.py."""
import numpy as np
import pytest
import torch

import scenes
from oracle import exposure_numpy as XN
from util import cpu_render
from splatam_b200 import formats, mapping as M, slam
from splatam_b200.train_ops import exposure_torch

T = 8


def _ab(seed):
    g = np.random.default_rng(seed)
    return np.concatenate([g.uniform(-0.4, 0.4, 3), g.uniform(-0.1, 0.1, 3)]).astype(np.float32)


def test_oracle_agrees_with_the_torch_statement_and_its_autograd_in_float64():
    g = np.random.default_rng(0)
    x = g.uniform(-0.2, 1.2, (3, 17, 13)).astype(np.float32)
    gy = g.normal(size=x.shape).astype(np.float32)
    ab = _ab(1)
    y = XN.apply(x, ab)
    yt = exposure_torch(torch.from_numpy(x).double(), torch.from_numpy(ab).double()).numpy()
    np.testing.assert_allclose(y, yt, rtol=2e-7, atol=2e-7)
    back = XN.apply(y, ab, inverse=True)
    np.testing.assert_allclose(back, x, rtol=1e-6, atol=1e-6)
    np.testing.assert_allclose(exposure_torch(torch.from_numpy(y).double(), torch.from_numpy(ab).double(),
                                              inverse=True).numpy(), back, rtol=1e-6, atol=1e-6)
    xt = torch.from_numpy(x).double().requires_grad_(True)
    abt = torch.from_numpy(ab).double().requires_grad_(True)
    exposure_torch(xt, abt).backward(torch.from_numpy(gy).double())
    gx, g_ab = XN.backward(x, ab, gy)
    np.testing.assert_allclose(gx, xt.grad.numpy(), rtol=2e-7, atol=1e-7)
    # the oracle's gain is exp(a) of the float32 a in double; the torch statement's is the same in float64
    np.testing.assert_allclose(g_ab, abt.grad.numpy(), rtol=1e-12, atol=1e-12)


def test_identity_correction_is_exact():
    x = np.random.default_rng(2).uniform(0, 1, (3, 5, 7)).astype(np.float32)
    zero = np.zeros(6, np.float32)
    assert np.array_equal(XN.apply(x, zero), x) and np.array_equal(XN.apply(x, zero, inverse=True), x)
    gy = np.random.default_rng(3).normal(size=x.shape).astype(np.float32)
    assert np.array_equal(XN.backward(x, zero, gy)[0], gy)


@pytest.fixture(scope="module")
def problem():
    import splatam_b200 as S
    torch.set_num_threads(4)
    sc = scenes.config1(seed=8, P=256, w=64, h=64)
    cam = sc.settings(S.GaussianRasterizationSettings, "cpu")
    gt = sc.splatam_params(opacity_clamp=(0.05, 0.95))
    rots, trans = slam.look_trajectory(T, "cpu", step=(0.004, -0.002, 0.003), rot_step=(0.001, -0.001, 0.0005))
    table = scenes.exposure_profile(T, gain=0.1, bias=0.01, period=8.0)
    frames = []
    for t in range(T):
        f = slam.render_frame(gt, rots, trans, t, cam, render=cpu_render)
        f["im"] = exposure_torch(f["im"], torch.from_numpy(table[t]))
        frames.append(f)
    K = torch.tensor([[sc.fx, 0, sc.cx], [0, sc.fy, sc.cy], [0, 0, 1]])
    kw = dict(render=cpu_render, fused=False, tracking_iters=30, mapping_iters=2, keyframe_every=2, window=3,
              intrinsics=K)
    return cam, frames, dict(gt), kw, table


@pytest.fixture(scope="module")
def full_run(problem, tmp_path_factory):
    cam, frames, init, kw, _ = problem
    d = str(tmp_path_factory.mktemp("ckpt"))
    torch.manual_seed(1); np.random.seed(1)
    out = slam.run_slam(init, frames, cam, checkpoint_dir=d, checkpoint_every=2, exposure={}, **kw)
    return out, d


def test_run_recovers_the_frames_gains_relative_to_frame_0(full_run, problem):
    out, _ = full_run
    table = problem[4]
    est = out["exposure"][0].numpy()                              # [6, T]
    assert out["exposure"].shape == (1, 6, T)
    assert np.array_equal(est[:, 0], np.zeros(6, np.float32))      # frame 0 is the gauge and is never stepped
    err = np.abs(est[:3].T - table[:, :3])
    # measured on this problem at the default rates: the largest log-gain error is 0.040, over log-gains down to -0.14
    assert err.max() < 0.05, err


def test_exact_resume_with_exposure(problem, full_run):
    cam, frames, _, kw, _ = problem
    out, d = full_run
    torch.manual_seed(77); np.random.seed(77)
    ckpt = formats.load_checkpoint(d, 4, "cpu")
    assert ckpt["state"]["cam_exposure"].shape == (1, 6, T)
    with np.load("%s/params4.npz" % d) as z:
        assert sorted(z.files) == sorted(formats.CHECKPOINT_KEYS)
    res = slam.run_slam(None, frames, cam, resume=ckpt, exposure={}, **kw)
    assert torch.equal(out["exposure"], res["exposure"])
    assert torch.equal(out["rots"], res["rots"]) and torch.equal(out["trans"], res["trans"])
    for k in M.GAUSSIAN_KEYS:
        assert torch.equal(out["gauss"][k], res["gauss"][k]), k
    assert out["psnr"] == res["psnr"]


def test_resume_without_saved_exposure_and_relocalise_raise(problem, tmp_path):
    cam, frames, init, kw, _ = problem
    d = str(tmp_path)
    slam.run_slam(init, frames[:3], cam, checkpoint_dir=d, checkpoint_every=2, **dict(kw, tracking_iters=1))
    ckpt = formats.load_checkpoint(d, 2, "cpu")
    with pytest.raises(ValueError, match="exposure"):
        slam.run_slam(None, frames[:3], cam, resume=ckpt, exposure={}, **kw)
    with pytest.raises(ValueError, match="relocalise"):
        slam.run_slam(init, frames, cam, exposure={}, relocalise={}, **kw)
    for bad in (dict(lr_gain=0.1), dict(lr_bias=-1.0), dict(lr_log_gain=float("nan")), [0.1]):
        with pytest.raises(ValueError):
            slam.run_slam(init, frames, cam, exposure=bad, **kw)


def test_exposure_npz_round_trips_and_params_keep_their_14_keys(full_run, problem, tmp_path):
    out, _ = full_run
    K = problem[3]["intrinsics"]
    d = str(tmp_path)
    path = formats.save_exposure(d, out["exposure"])
    assert path.endswith("exposure.npz")
    back = formats.load_exposure(path, num_frames=T)
    assert back.dtype == np.float32 and np.array_equal(back, out["exposure"].numpy())
    assert torch.equal(formats.load_exposure(path, device="cpu"), out["exposure"])
    with pytest.raises(ValueError):
        formats.load_exposure(path, num_frames=T + 1)
    with pytest.raises(ValueError):
        formats.save_exposure(d, out["exposure"][0])
    rec = formats.save_run_record(d, out["gauss"], out["rots"], out["trans"], out["timestep"], K, torch.eye(4), 64, 64,
                                  [torch.eye(4)] * T, out["keyframe_time_indices"])
    with np.load(rec) as z:
        assert len(z.files) == 14 and "cam_exposure" not in z.files


def test_exposure_lives_only_where_it_is_given(problem):
    """_render_pair corrects only with an exposure: params without cam_exposure render as before."""
    cam, frames, gt, _, table = problem
    rots, trans = slam.look_trajectory(T, "cpu", step=(0.004, -0.002, 0.003), rot_step=(0.001, -0.001, 0.0005))
    p = dict(gt, cam_unnorm_rots=rots, cam_trans=trans)
    fr = dict(frames[3], cam=cam)
    plain, _, _, _ = M._render_pair(p, fr, cpu_render, False, camera_grad=False)
    expo = torch.from_numpy(np.ascontiguousarray(table.T[None]))
    corr, _, _, _ = M._render_pair(dict(p, cam_exposure=expo), fr, cpu_render, False, camera_grad=False)
    assert torch.equal(corr, exposure_torch(plain, expo[0, :, 3]))
    given, _, _, _ = M._render_pair(p, dict(fr, exposure=expo[0, :, 5]), cpu_render, False, camera_grad=False)
    assert torch.equal(given, exposure_torch(plain, expo[0, :, 5]))
