"""GPU: sb_lpips (csrc/lpips.cu) through evaluate.lpips against the float64 oracle (oracle/lpips_torch.py) with seeded
random weights in the real key layout, and LPIPS inside evaluate / evaluate_nvs on rendered sequences.

Bound per image pair: max(1e-5, 2 x the distance of the float32 restatement of the same definition from float64, both
on the CPU) -- the kernel has to be at least as close to the definition as a float32 PyTorch implementation of it (the
rule of the MS-SSIM tests)."""
import numpy as np
import pytest
import torch

from oracle import lpips_torch as OL
from test_evaluate_gpu import _slam_sequence

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def weights():
    alex, lin = OL.random_state_dicts(seed=7)
    return alex, lin, dict(alex, **lin)


@pytest.fixture(scope="module")
def net(weights, cuda_device):
    from splatam_b200.evaluate import LpipsAlex
    return LpipsAlex.from_state_dicts(weights[0], weights[1], cuda_device)


def lpips_bound(x, y, w):
    """[N] float64 tolerance of the kernel on CPU images x, y (see the module docstring), and the float64 values."""
    ref = OL.lpips(x, y, w)
    f32 = OL.lpips(x.float(), y.float(), w, dtype=torch.float32).double()
    return torch.clamp(2 * (f32 - ref).abs(), min=1e-5), ref


def _pair(kind, N, H, W, seed):
    """Image pairs, partly outside [0, 1] so the clamp matters."""
    g = torch.Generator().manual_seed(seed)
    x = 1.4 * torch.rand(N, 3, H, W, generator=g) - 0.2
    if kind == "random":
        y = 1.4 * torch.rand(N, 3, H, W, generator=g) - 0.2
    elif kind == "correlated":
        y = x + 0.1 * torch.randn(N, 3, H, W, generator=g)
    elif kind == "inverted":
        y = 1 - x
    elif kind == "constant":
        x, y = torch.full((N, 3, H, W), 0.3), torch.full((N, 3, H, W), 1.3)
    elif kind == "masked":              # weighted images: both zero where the mask is off
        y = x + 0.05 * torch.randn(N, 3, H, W, generator=g)
        keep = (torch.rand(N, 1, H, W, generator=g) > 0.2) & (torch.arange(W) > W // 3)
        x, y = x * keep, y * keep
    return x, y


CASES = [("random", 1, 31, 31), ("inverted", 2, 31, 31), ("correlated", 2, 45, 97), ("constant", 2, 45, 97),
         ("masked", 1, 45, 97), ("masked", 2, 480, 640), ("inverted", 1, 480, 640), ("correlated", 2, 584, 876),
         ("random", 1, 584, 876), ("masked", 1, 680, 1200), ("correlated", 2, 680, 1200)]


@pytest.mark.parametrize("kind,N,H,W", CASES)
def test_lpips_matches_float64_definition(cuda_device, weights, net, kind, N, H, W):
    from splatam_b200.evaluate import lpips
    x, y = _pair(kind, N, H, W, seed=H + W + N)
    bound, ref = lpips_bound(x, y, weights[2])
    got = lpips(x.to(cuda_device), y.to(cuda_device), net, size_average=False).cpu()
    assert got.shape == (N,) and got.dtype == torch.float64
    err = (got - ref).abs()
    print("%s N=%d %dx%d: lpips %s, |err| %.3g, bound %.3g" % (kind, N, W, H, ref.tolist(), err.max(), bound.min()))
    assert (err <= bound).all(), (err.tolist(), bound.tolist())
    mean = lpips(x.to(cuda_device), y.to(cuda_device), net)
    assert mean.shape == () and abs(mean.item() - ref.mean().item()) <= bound.max().item()
    assert (ref > 0).all()


def test_strided_inputs(cuda_device, weights, net):
    from splatam_b200.evaluate import lpips
    x, y = _pair("correlated", 2, 97, 45, seed=5)
    xt, yt = x.transpose(-1, -2), y.transpose(-1, -2)                      # [2,3,45,97] views
    bound, ref = lpips_bound(xt.contiguous(), yt.contiguous(), weights[2])
    xg, yg = x.to(cuda_device).transpose(-1, -2), y.to(cuda_device).transpose(-1, -2)
    assert not xg.is_contiguous()
    assert ((lpips(xg, yg, net, size_average=False).cpu() - ref).abs() <= bound).all()
    both = torch.stack([xt, yt], 2).reshape(2, 6, 45, 97).to(cuda_device)   # x and y channels interleaved
    assert ((lpips(both[:, 0::2], both[:, 1::2], net, size_average=False).cpu() - ref).abs() <= bound).all()


def test_identical_images_and_determinism(cuda_device, net):
    from splatam_b200.evaluate import lpips
    x, y = _pair("correlated", 2, 680, 1200, seed=11)
    x, y = x.to(cuda_device), y.to(cuda_device)
    assert lpips(x, x.clone(), net).item() == 0.0
    assert torch.equal(lpips(x, x.clone(), net, size_average=False), torch.zeros(2, dtype=torch.float64, device=cuda_device))
    a, b = lpips(x, y, net, size_average=False), lpips(x, y, net, size_average=False)
    assert torch.equal(a, b) and (a > 0).all()
    with pytest.raises(Exception, match="H and W >= 31"):
        lpips(x[..., :30, :], y[..., :30, :], net)


def _check_per_frame(out, frames_and_renders, weights, use_presence, sil_thres):
    from oracle import metrics_torch as O
    for k, (fr, im, ds) in enumerate(frames_and_renders):
        m = O.frame_metrics(im.cpu(), ds.cpu(), fr["im"].cpu(), fr["depth"].cpu(), sil_thres, use_presence)
        bound, ref = lpips_bound(m["weighted_im"][None], m["weighted_gt"][None], weights[2])
        assert abs(out["lpips_per_frame"][k] - ref.item()) <= bound.item(), (k, out["lpips_per_frame"][k], ref.item())


def _same_except_lpips(with_lp, without, tmp_with, tmp_without):
    assert "lpips_per_frame" not in without and without["lpips"] is None
    assert set(with_lp) == set(without) | {"lpips_per_frame"}
    for key, v in without.items():
        if key == "lpips":
            continue
        if isinstance(v, np.ndarray):
            assert np.array_equal(with_lp[key], v), key
        elif isinstance(v, float) and np.isnan(v):
            assert np.isnan(with_lp[key]), key
        else:
            assert with_lp[key] == v, key
    files = sorted(p.name for p in tmp_without.iterdir())
    assert sorted(p.name for p in tmp_with.iterdir()) == sorted(files + ["lpips.txt"])
    for name in files:
        assert (tmp_with / name).read_bytes() == (tmp_without / name).read_bytes(), name
    lp = np.atleast_1d(np.loadtxt(tmp_with / "lpips.txt"))
    assert lp.shape == (len(with_lp["frame_ids"]),) and np.array_equal(lp, with_lp["lpips_per_frame"])


def test_evaluate_with_lpips(cuda_device, weights, net, tmp_path):
    from splatam_b200 import mapping as M
    from splatam_b200.evaluate import evaluate
    dev = cuda_device
    cam, frames, params, gt_w2c = _slam_sequence(dev)
    for mapping_iters, add_new in ((0, False), (40, True)):
        a, b = tmp_path / ("with%d" % mapping_iters), tmp_path / ("without%d" % mapping_iters)
        out = evaluate(params, frames, cam, 0.5, mapping_iters, add_new, eval_every=2, gt_w2c=gt_w2c, out_dir=str(a),
                       lpips=net)
        ref = evaluate(params, frames, cam, 0.5, mapping_iters, add_new, eval_every=2, gt_w2c=gt_w2c, out_dir=str(b))
        _same_except_lpips(out, ref, a, b)
        assert out["lpips"] == float(out["lpips_per_frame"].mean()) and out["lpips"] > 0
        rendered = []
        for t in out["frame_ids"]:
            with torch.no_grad():
                im, ds, _, _ = M._render_pair(params, dict(frames[t], cam=cam), M.default_render, True, False)
            rendered.append((frames[t], im, ds))
        _check_per_frame(out, rendered, weights, mapping_iters == 0 and not add_new, 0.5)
        print("evaluate (mapping_iters=%d): LPIPS %.5f" % (mapping_iters, out["lpips"]))


def test_evaluate_nvs_with_lpips_averages_valid_views(cuda_device, weights, net, tmp_path):
    from splatam_b200 import mapping as M
    from splatam_b200.evaluate import evaluate_nvs
    dev = cuda_device
    cam, frames, est, _ = _slam_sequence(dev, T=6)
    params = {k: v for k, v in est.items() if not k.startswith("cam_")}
    away = torch.eye(4, device=dev)
    away[2, 3] = -50.0                   # the map lies behind this camera: every valid-depth pixel is a hole
    for t, fr in enumerate(frames):
        fr["gt_w2c"] = away if t == 3 else M.camera_w2c(est["cam_unnorm_rots"][..., t], est["cam_trans"][..., t])[0]
        if t != 3:                       # no holes: ground-truth depth only where the map's silhouette covers
            with torch.no_grad():
                _, ds, _, _ = M._render_pair(params, dict(fr, cam=cam, pose=M.gt_pose(fr["gt_w2c"])), M.default_render,
                                             True, False)
            fr["depth"] = fr["depth"] * (ds[1:2] > 0.5)
    a, b = tmp_path / "with", tmp_path / "without"
    out = evaluate_nvs(params, frames, cam, 0.5, 30, True, out_dir=str(a), lpips=net)
    ref = evaluate_nvs(params, frames, cam, 0.5, 30, True, out_dir=str(b))
    _same_except_lpips(out, ref, a, b)
    valid = out["valid_nvs_frames"]
    assert out["frame_ids"] == [1, 2, 3, 4, 5] and valid.tolist() == [True, True, False, True, True]
    assert out["lpips"] == float(out["lpips_per_frame"][valid].mean())
    assert out["lpips"] != float(out["lpips_per_frame"].mean())
    rendered = []
    for t in out["frame_ids"]:
        with torch.no_grad():
            fr = dict(frames[t], cam=cam, pose=M.gt_pose(frames[t]["gt_w2c"].float()))
            im, ds, _, _ = M._render_pair(params, fr, M.default_render, True, False)
        rendered.append((frames[t], im, ds))
    _check_per_frame(out, rendered, weights, False, 0.5)
    # no valid view: the average is NaN, the per-frame values are still written
    for fr in frames:
        fr["gt_w2c"] = away
    none = evaluate_nvs(params, frames, cam, 0.5, 30, True, lpips=net)
    assert not none["valid_nvs_frames"].any() and np.isnan(none["lpips"])
    assert np.isfinite(none["lpips_per_frame"]).all()
