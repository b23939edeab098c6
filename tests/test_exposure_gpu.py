"""GPU: per-frame exposure (csrc/exposure.cu through train_ops.exposure; tracking, mapping, map growth, evaluation and
the tools through slam.run_slam's `exposure`).  The kernels against oracle/exposure_numpy.py, graph and eager tracking,
fused and torch paths, the identity correction that changes no bit of a run, and SLAM on written sequences whose
frames change exposure and white balance."""
import os

import numpy as np
import pytest
import torch

import scenes
from oracle import exposure_numpy as XN
from util import load, run_tool
from splatam_b200 import _lib, formats, mapping as M, slam
from splatam_b200.train_ops import exposure, exposure_torch

pytestmark = pytest.mark.gpu

SIZES = [(1, 1), (17, 1), (97, 45), (1200, 680), (1920, 1440)]          # (W, H)


def _inputs(W, H, seed, dev):
    g = np.random.default_rng(seed)
    x = g.uniform(-0.1, 1.1, (3, H, W)).astype(np.float32)
    gy = g.normal(size=(3, H, W)).astype(np.float32)
    ab = np.concatenate([g.uniform(-0.5, 0.5, 3), g.uniform(-0.1, 0.1, 3)]).astype(np.float32)
    return x, gy, ab, [torch.from_numpy(a).to(dev) for a in (x, gy, ab)]


@pytest.mark.parametrize("W,H", SIZES)
def test_apply_and_inverse_are_bit_equal_to_the_oracle(cuda_device, W, H):
    x, _, ab, (xd, _, abd) = _inputs(W, H, W + H, cuda_device)
    y = exposure(xd, abd)
    assert np.array_equal(y.cpu().numpy(), XN.apply(x, ab))
    assert np.array_equal(exposure(xd, abd, inverse=True).cpu().numpy(), XN.apply(x, ab, inverse=True))
    # a view that starts one float into its storage takes the unaligned path
    buf = torch.empty(3 * H * W + 1, device=cuda_device)
    buf[1:].copy_(xd.reshape(-1))
    xo, yo = buf[1:].view(3, H, W), torch.empty(3 * H * W + 1, device=cuda_device)[1:].view(3, H, W)
    _lib.call("sb_exposure_apply", H, W, xo, abd, 0, yo, device=cuda_device)
    assert np.array_equal(yo.cpu().numpy(), XN.apply(x, ab))


@pytest.mark.parametrize("W,H", SIZES)
def test_backward_matches_the_oracle_and_repeats_bit_for_bit(cuda_device, W, H):
    x, gy, ab, (xd, gyd, abd) = _inputs(W, H, 7 * W + H, cuda_device)
    gx_ref, g_ref = XN.backward(x, ab, gy)
    ws = torch.empty(_lib.nbytes("sb_exposure_workspace_bytes", H, W), dtype=torch.uint8, device=cuda_device)
    outs = []
    for _ in range(2):
        gx = torch.empty_like(xd)
        g = torch.empty(6, dtype=torch.float64, device=cuda_device)
        _lib.call("sb_exposure_backward", H, W, xd, abd, gyd, gx, g, ws, ws.numel(), device=cuda_device)
        outs.append((gx.cpu().numpy(), g.cpu().numpy()))
    assert np.array_equal(outs[0][0], gx_ref)
    assert np.array_equal(outs[0][1], outs[1][1]) and np.array_equal(outs[0][0], outs[1][0])
    # relative to the sum of the terms' magnitudes: a sum of signed terms can cancel to far below them
    x64, g64 = x.astype(np.float64).reshape(3, -1), gy.astype(np.float64).reshape(3, -1)
    scale = np.concatenate([np.exp(ab[:3].astype(np.float64)) * np.abs(x64 * g64).sum(1), np.abs(g64).sum(1)])
    assert (np.abs(outs[0][1] - g_ref) <= 1e-12 * scale).all(), (outs[0][1], g_ref)
    # the autograd Function returns the same numbers
    xg, abg = xd.clone().requires_grad_(True), abd.clone().requires_grad_(True)
    exposure(xg, abg).backward(gyd)
    assert np.array_equal(xg.grad.cpu().numpy(), gx_ref)
    assert np.array_equal(abg.grad.cpu().numpy(), outs[0][1].astype(np.float32))


def test_bad_arguments_are_rejected(cuda_device):
    x = torch.zeros(3, 4, 4, device=cuda_device)
    ab = torch.zeros(6, device=cuda_device)
    for args in ((0, 4, x, ab, 0, x), (4, 4, None, ab, 0, x), (4, 4, x, ab, 2, x)):
        with pytest.raises(_lib.SplatamB200Error):
            _lib.call("sb_exposure_apply", *args, device=cuda_device)
    g = torch.zeros(6, dtype=torch.float64, device=cuda_device)
    ws = torch.zeros(8, dtype=torch.uint8, device=cuda_device)
    with pytest.raises(_lib.SplatamB200Error, match="WORKSPACE"):
        _lib.call("sb_exposure_backward", 4, 4, x, ab, x, x, g, ws, ws.numel(), device=cuda_device)
    with pytest.raises(_lib.SplatamB200Error):
        exposure(x.cpu(), ab.cpu())


# ---- tracking ------------------------------------------------------------------------------------------------------

TABLE = scenes.exposure_profile(6, gain=0.12, bias=0.02, period=6.0)


@pytest.fixture(scope="module")
def track_problem(cuda_device):
    import splatam_b200 as S
    sc = scenes.config1(seed=5, P=4000, w=320, h=240)
    cam = sc.settings(S.GaussianRasterizationSettings, cuda_device)
    gt = {k: v.to(cuda_device) for k, v in sc.splatam_params(opacity_clamp=(0.3, 0.95)).items()}
    rots, trans = slam.look_trajectory(6, cuda_device)
    frames = []
    for t in range(6):
        f = slam.render_frame(gt, rots, trans, t, cam)
        f["im"] = exposure(f["im"], torch.from_numpy(TABLE[t]).to(cuda_device))
        frames.append(f)
    return gt, rots, trans, frames


def _track(track_problem, t, graph, fused=True, lr_exposure=(0.01, 0.002), iters=100):
    gt, rots, trans, frames = track_problem
    r, tr = rots.clone(), trans.clone()
    r[..., t], tr[..., t] = rots[..., t - 1], trans[..., t - 1]
    expo = torch.zeros(1, 6, rots.shape[-1], device=rots.device)
    expo[0, :, t - 1] = torch.from_numpy(TABLE[t - 1]).to(rots.device)
    expo[..., t] = expo[..., t - 1]
    params = dict({k: v.detach() for k, v in gt.items()}, cam_unnorm_rots=r, cam_trans=tr, cam_exposure=expo)
    M._TRACK_GRAPHS.clear()
    losses = M.track_frame(params, frames[t], num_iters=iters, fused=fused, graph=graph, lr_exposure=lr_exposure)
    return params, losses


def test_graph_and_eager_tracking_agree_on_pose_and_exposure(track_problem):
    t = 3
    pg, lg = _track(track_problem, t, graph=True)
    pe, le = _track(track_problem, t, graph=False)
    assert len(lg) == len(le) == 100
    ex_g, ex_e = pg["cam_exposure"][0, :, t], pe["cam_exposure"][0, :, t]
    # both paths sum pose gradients with float atomics, so each run keeps a slightly different best iteration:
    # measured on an H100 up to 2.2e-3 apart in a log-gain
    assert float((ex_g - ex_e).abs().max()) < 5e-3
    # test_tracking_gpu's tolerances between tracking paths: 1e-3 on the quaternion, 2e-3 on the translation
    assert float((pg["cam_unnorm_rots"][..., t] - pe["cam_unnorm_rots"][..., t]).detach().abs().max()) < 1e-3
    assert float((pg["cam_trans"][..., t] - pe["cam_trans"][..., t]).detach().abs().max()) < 2e-3
    assert float((ex_g[:3].cpu() - torch.from_numpy(TABLE[t][:3])).abs().max()) < 0.02


def test_fused_and_torch_paths_agree(track_problem):
    t = 2
    pf, _ = _track(track_problem, t, graph=False, fused=True, iters=40)
    pt, _ = _track(track_problem, t, graph=False, fused=False, iters=40)
    assert float((pf["cam_exposure"][0, :, t] - pt["cam_exposure"][0, :, t]).abs().max()) < 2e-3
    assert float((pf["cam_trans"][..., t] - pt["cam_trans"][..., t]).detach().abs().max()) < 2e-3
    assert float((pf["cam_unnorm_rots"][..., t] - pt["cam_unnorm_rots"][..., t]).detach().abs().max()) < 1e-3


def test_identity_correction_is_exact_in_the_kernels(cuda_device):
    """ab = 0: apply, inverse and the backward's gx give their inputs back bit for bit, so zero rates change no value
    a render, a loss or an image gradient carries."""
    x, gy, _, (xd, gyd, _) = _inputs(1200, 680, 11, cuda_device)
    zero = torch.zeros(6, device=cuda_device)
    assert torch.equal(exposure(xd, zero), xd) and torch.equal(exposure(xd, zero, inverse=True), xd)
    xg = xd.clone().requires_grad_(True)
    exposure(xg, zero).backward(gyd)
    assert torch.equal(xg.grad, gyd)


@pytest.mark.parametrize("graph", [False, True])
def test_zero_rates_change_nothing_in_a_run(track_problem, cuda_device, graph):
    """exposure with zero rates: every correction stays the identity, so the run is the run without exposure --
    tracking (graphed when `graph`), mapping (captured when `graph`), map growth and the final PSNR.  The renders
    match bit for bit; the rasterizer's backward sums gradients with float atomics, so two runs without exposure need
    not end bit-equal either: the run with exposure must stay within their run-to-run spread."""
    import splatam_b200 as S
    gt, rots, trans, frames = track_problem
    sc = scenes.config1(seed=5, P=4000, w=320, h=240)
    cam = sc.settings(S.GaussianRasterizationSettings, cuda_device)
    p = dict(gt, cam_unnorm_rots=rots, cam_trans=trans)
    fr = dict(frames[2], cam=cam)
    plain, _, _, _ = M._render_pair(p, fr, M.default_render, True, camera_grad=False)
    ident, _, _, _ = M._render_pair(dict(p, cam_exposure=torch.zeros(1, 6, 6, device=cuda_device)), fr,
                                    M.default_render, True, camera_grad=False)
    assert torch.equal(plain, ident)
    K = torch.tensor([[sc.fx, 0, sc.cx], [0, sc.fy, sc.cy], [0, 0, 1]])
    init = {k: v.clone() for k, v in gt.items()}
    init["rgb_colors"] = (init["rgb_colors"] * 0.9).contiguous()
    kw = dict(tracking_iters=100 if graph else 20, mapping_iters=10, keyframe_every=2, window=3, graph=graph,
              intrinsics=K, add_new_gaussians=True, sil_thres=0.5)
    outs = []
    for expo in (None, None, dict(lr_log_gain=0.0, lr_bias=0.0)):
        M._TRACK_GRAPHS.clear()
        torch.manual_seed(0); np.random.seed(0)
        outs.append(slam.run_slam(dict(init), frames, cam, exposure=expo, **kw))
    a, a2, b = outs
    assert torch.equal(b["exposure"], torch.zeros_like(b["exposure"]))
    ate = lambda o: slam.ate_rmse(o["rots"], o["trans"], rots, trans)
    spread_ate, spread_psnr = abs(ate(a) - ate(a2)), abs(a["psnr"] - a2["psnr"])
    assert abs(ate(b) - ate(a)) <= 2 * spread_ate + 2e-4, (ate(a), ate(a2), ate(b))
    assert abs(b["psnr"] - a["psnr"]) <= 2 * spread_psnr + 0.2, (a["psnr"], a2["psnr"], b["psnr"])


# ---- SLAM on written sequences -------------------------------------------------------------------------------------

T_SEQ = 16
VARYING = scenes.exposure_profile(T_SEQ)


def _run(tool, basedir, out_dir, exposure, monkeypatch, capsys):
    argv = ["run_slam_dataset.py", "--dataset", "replica", "--basedir", basedir, "--sequence", "room0",
            "--tracking-iters", "40", "--mapping-iters", "30", "--out", out_dir] + (["--exposure"] if exposure else [])
    return run_tool(tool, argv, monkeypatch, capsys)


@pytest.fixture(scope="module")
def written(cuda_device, tmp_path_factory):
    root = tmp_path_factory.mktemp("expo")
    for name, table in (("varying", VARYING), ("constant", None)):
        scenes.write_replica_sequence(str(root / name / "room0"), T_SEQ, cuda_device, exposure=table)
    return root


def test_exposure_beats_no_exposure_on_a_varying_sequence(written, monkeypatch, capsys):
    tool = load("tools/run_slam_dataset.py")
    base = str(written / "varying")
    off = _run(tool, base, str(written / "run_off"), False, monkeypatch, capsys)
    on = _run(tool, base, str(written / "run_on"), True, monkeypatch, capsys)
    assert on["exposure"] and not off["exposure"]
    assert on["ate_m"] < off["ate_m"] and on["psnr_db"] > off["psnr_db"], (on, off)
    est = formats.load_exposure(os.path.join(str(written / "run_on"), "exposure.npz"), num_frames=T_SEQ)[0]
    err = np.abs(est[:3].T - VARYING[:, :3])
    # measured on an H100: at most 0.012 over log-gains down to -0.43
    assert err.max() < 0.04, err
    # the record evaluator scores the saved run through exposure.npz as the run did
    ev = load("tools/eval_record.py")
    rec = str(written / "run_on" / "params.npz")
    argv = ["eval_record.py", "--dataset", "replica", "--basedir", base, "--sequence", "room0", "--record", rec,
            "--no-frames", "--out", str(written / "eval_on")]
    with_expo = run_tool(ev, argv + ["--exposure", str(written / "run_on" / "exposure.npz")], monkeypatch, capsys)
    plain = run_tool(ev, argv, monkeypatch, capsys)
    assert abs(with_expo["psnr_db"] - on["psnr_db"]) < 1e-6 and with_expo["psnr_db"] > plain["psnr_db"]


def test_constant_exposure_stays_near_the_identity(written, monkeypatch, capsys):
    tool = load("tools/run_slam_dataset.py")
    base = str(written / "constant")
    offs = [_run(tool, base, str(written / ("c_off%d" % i)), False, monkeypatch, capsys)["ate_m"] for i in range(2)]
    on = _run(tool, base, str(written / "c_on"), True, monkeypatch, capsys)
    est = formats.load_exposure(os.path.join(str(written / "c_on"), "exposure.npz"), num_frames=T_SEQ)[0]
    assert np.abs(est[:3]).max() < 0.02 and np.abs(est[3:]).max() < 0.01, est
    spread = abs(offs[0] - offs[1])
    assert on["ate_m"] <= max(offs) + max(2 * spread, 5e-4), (on["ate_m"], offs)


def test_iphone_demo_runs_with_exposure(cuda_device, tmp_path, monkeypatch, capsys):
    demo = load("tools/run_iphone_demo.py")
    out = str(tmp_path / "demo")
    line = run_tool(demo, ["run_iphone_demo.py", "--source", "synthetic", "--frames", "5", "--out", out,
                           "--tracking-iters", "5", "--mapping-iters", "5", "--exposure"], monkeypatch, capsys)
    assert line["exposure"] and np.isfinite(line["ate_m"])
    assert formats.load_exposure(os.path.join(out, "exposure.npz"), num_frames=5).shape == (1, 6, 5)
    with np.load(os.path.join(out, "params.npz")) as z:
        assert len(z.files) == 14
