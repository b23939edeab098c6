"""GPU: the saved evaluation frames (csrc/eval_frames.cu, evaluate(..., save_frames=True)) against the files the
reference's own `eval` / `eval_nvs` wrote (tests/golden/eval/ref_eval_frames.npz), the kernel against the reference's
numpy / cv2 statements at 1200x680, save_frames leaving every metric unchanged, and tools/eval_record.py end to end
against the run that wrote the record."""
import importlib.util
import json
import os
import sys

import numpy as np
import pytest
import torch

import scenes
from util import GOLDEN, ROOT

pytestmark = pytest.mark.gpu


def _load(path, name):
    spec = importlib.util.spec_from_file_location(name, path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _gen():
    return _load(os.path.join(GOLDEN, "eval", "make_golden_eval_frames.py"), "make_golden_eval_frames")


@pytest.mark.parametrize("name", ["eval", "eval_nvs"])
def test_saved_frames_equal_the_reference_files(cuda_device, tmp_path, name):
    from splatam_b200.evaluate import evaluate, evaluate_nvs
    gen = _gen()
    fx = np.load(os.path.join(GOLDEN, "eval", "ref_eval_frames.npz"))
    dev = cuda_device
    case = gen.frames_case(name)
    params = {k: v.to(dev) for k, v in case["params"].items()}
    renders = {t: (im.to(dev), ds.to(dev)) for t, (im, ds) in case["renders"].items()}
    dev_case = dict(case, params=params, gt_w2c=case["gt_w2c"].to(dev))

    def render(settings, means3D, colors_precomp, **rv):
        t = gen.render_frame_of(dev_case, means3D)
        depth_call = bool((colors_precomp[:, 1] == 1).all())
        return renders[t][1 if depth_call else 0].clone(), torch.zeros(means3D.shape[0], dtype=torch.int32), None
    w2c0 = torch.linalg.inv(case["dataset"][0][3]).to(dev)
    frames = [dict(id=t, im=(c.permute(2, 0, 1) / 255).to(dev), depth=d.permute(2, 0, 1).to(dev), w2c=w2c0,
                   gt_w2c=dev_case["gt_w2c"][t]) for t, (c, d, _, _) in enumerate(case["dataset"])]
    args = (params, frames, None, case["sil_thres"], case["mapping_iters"], case["add_new_gaussians"])
    kw = dict(eval_every=case["eval_every"], fused=False, render=render, out_dir=str(tmp_path), save_frames=True)
    if name == "eval":
        evaluate(*args, **kw)
    else:
        evaluate_nvs(*args, **kw)
    names, pixels = gen.read_frames(str(tmp_path))
    assert names == [str(f) for f in fx[name + "_files"]]
    for n, got, ref in zip(names, pixels, fx[name + "_pixels"]):
        assert np.array_equal(got, ref), n


def _special(g, shape, lo, hi):
    x = lo + (hi - lo) * torch.rand(shape, generator=g)
    flat = x.view(-1)
    idx = torch.randperm(flat.numel(), generator=g)[:3000]
    flat[idx[:1000]] = float("nan")
    flat[idx[1000:1500]] = float("inf")
    flat[idx[1500:2000]] = -float("inf")
    return x


def test_kernel_equals_the_reference_statements_at_1200x680(cuda_device, tmp_path):
    """eval_helpers.py:509-528 verbatim on the CPU (torch.clamp, numpy, cv2.applyColorMap, cv2.imwrite of the float32
    image decoded by Pillow) against one sb_eval_frames_u8 launch, on random inputs with NaN, +-inf, colours outside
    [0, 1], depths below 0 and above 6 m and every 6 * k / 255 boundary with its float32 neighbours."""
    cv2 = pytest.importorskip("cv2")
    from PIL import Image
    from splatam_b200.evaluate import eval_frames_u8
    gen = _gen()
    H, W = 680, 1200
    g = torch.Generator().manual_seed(17)
    im, gt = _special(g, (3, H, W), -0.3, 1.3), _special(g, (3, H, W), -0.1, 1.1)
    ties = gen.tie_values()
    im.view(-1)[:ties.numel()] = ties
    gt.view(-1)[-ties.numel():] = ties
    depth_sil = torch.stack([_special(g, (H, W), -1.0, 8.0), torch.rand(H, W, generator=g), torch.rand(H, W, generator=g)])
    gd = (-1.0 + 9.0 * torch.rand(1, H, W, generator=g))
    b = gen.depth_boundaries()
    depth_sil[0].view(-1)[:b.numel()] = b
    gd.view(-1)[-b.numel():] = b
    gd.view(-1)[:1000] = 0.0
    got = eval_frames_u8(*(t.to(cuda_device) for t in (im, depth_sil, gt, gd))).cpu().numpy()
    vmin, vmax = 0, 6

    def rgb(x, path):
        v = torch.clamp(x, 0, 1).detach().cpu().permute(1, 2, 0).numpy()
        cv2.imwrite(path, cv2.cvtColor(v * 255, cv2.COLOR_RGB2BGR))
        with Image.open(path) as f:
            return np.array(f)

    def depth(d):
        with np.errstate(invalid="ignore"):
            n = np.clip((d - vmin) / (vmax - vmin), 0, 1)
            return cv2.applyColorMap((n * 255).astype(np.uint8), cv2.COLORMAP_JET)[..., ::-1]
    want = [rgb(im, str(tmp_path / "a.png")), depth(depth_sil[0].numpy()), rgb(gt, str(tmp_path / "b.png")),
            depth(gd[0].numpy())]
    for k in range(4):
        assert np.array_equal(got[k], want[k]), (k, int((got[k] != want[k]).any(-1).sum()))


def test_save_frames_changes_no_result(cuda_device, tmp_path):
    """On the fused path evaluate with and without save_frames gives identical result dicts and .txt files; without
    it no image directory is made."""
    import splatam_b200 as S
    from splatam_b200 import evaluate as EV, slam
    dev = cuda_device
    sc = scenes.room(seed=31, P=30_000, cam=dict(w=320, h=192, fx=160.0, fy=160.0, cx=159.5, cy=95.5))
    cam = sc.settings(S.GaussianRasterizationSettings, dev)
    gt = dict(means3D=sc.means3D, rgb_colors=sc.colors, unnorm_rotations=sc.rotations,
              logit_opacities=torch.logit(sc.opacities.clamp(0.02, 0.98)), log_scales=torch.log(sc.scales[:, :1]))
    gt = {k: v.to(dev) for k, v in gt.items()}
    T = 9
    rots, trans = slam.look_trajectory(T, dev)
    frames = [slam.render_frame(gt, rots, trans, t, cam) for t in range(T)]
    g = torch.Generator().manual_seed(5)
    params = dict(gt, cam_unnorm_rots=rots, cam_trans=trans)
    params["rgb_colors"] = (gt["rgb_colors"] + 0.08 * torch.randn(gt["rgb_colors"].shape, generator=g).to(dev)).clamp(0, 1)
    gt_w2c = slam.w2c_list(rots, trans)
    plain, saved = str(tmp_path / "plain"), str(tmp_path / "saved")
    a = EV.evaluate(params, frames, cam, 0.5, 40, True, eval_every=2, gt_w2c=gt_w2c, fused=True, out_dir=plain)
    b = EV.evaluate(params, frames, cam, 0.5, 40, True, eval_every=2, gt_w2c=gt_w2c, fused=True, out_dir=saved,
                    save_frames=True)
    assert a.keys() == b.keys()
    for k in a:
        if isinstance(a[k], np.ndarray):
            assert np.array_equal(a[k], b[k]), k
        else:
            assert a[k] == b[k], k
    assert sorted(os.listdir(plain)) == ["l1.txt", "psnr.txt", "rmse.txt", "ssim.txt"]
    for f in os.listdir(plain):
        with open(os.path.join(plain, f), "rb") as x, open(os.path.join(saved, f), "rb") as y:
            assert x.read() == y.read(), f
    ids = a["frame_ids"]
    assert ids == [0, 1, 3, 5, 7]
    for d in ("rendered_rgb", "rendered_depth"):
        assert sorted(os.listdir(os.path.join(saved, d))) == ["gs_%04d.png" % t for t in ids]
    for d in ("rgb", "depth"):
        assert sorted(os.listdir(os.path.join(saved, d))) == ["gt_%04d.png" % t for t in ids]
    # the saved frames are the kernel's images of the frame's renders
    from PIL import Image
    from splatam_b200 import mapping as M
    with torch.no_grad():
        im, ds, _, _ = M._render_pair(params, dict(frames[3], cam=cam), M.default_render, True, False)
    want = EV.eval_frames_u8(im, ds, frames[3]["im"], frames[3]["depth"]).cpu().numpy()
    for k, (d, n) in enumerate((("rendered_rgb", "gs"), ("rendered_depth", "gs"), ("rgb", "gt"), ("depth", "gt"))):
        with Image.open(os.path.join(saved, d, "%s_0003.png" % n)) as f:
            assert np.array_equal(np.array(f), want[k]), d
    with pytest.raises(FileNotFoundError):            # a writer's error reaches the caller, after every thread ends
        EV.evaluate(params, frames[:2], cam, 0.5, 40, True, fused=True, out_dir=str(tmp_path / "gone"),
                    save_frames=True, render=_removing_render(str(tmp_path / "gone")))


def _removing_render(path):
    """M.default_render that first deletes `path`'s rendered_rgb directory, so the writers cannot save there."""
    import shutil
    from splatam_b200 import mapping as M

    def render(settings, **rv):
        shutil.rmtree(os.path.join(path, "rendered_rgb"), ignore_errors=True)
        return M.default_render(settings, **rv)
    return render


def _run(tool, argv, monkeypatch, capsys):
    monkeypatch.setattr(sys, "argv", argv)
    tool.main()
    return json.loads(capsys.readouterr().out.strip().splitlines()[-1])


def test_eval_record_reproduces_the_run(cuda_device, tmp_path, monkeypatch, capsys):
    from splatam_b200 import datasets, evaluate, formats
    T = 6
    scenes.write_replica_sequence(str(tmp_path / "room0"), T, cuda_device)
    data = ["--dataset", "replica", "--basedir", str(tmp_path), "--sequence", "room0"]
    run_dir = str(tmp_path / "run")
    run = _run(_load(os.path.join(ROOT, "tools", "run_slam_dataset.py"), "run_slam_dataset"),
               ["run_slam_dataset.py"] + data + ["--tracking-iters", "10", "--mapping-iters", "10", "--out", run_dir,
                                                 "--save-frames"], monkeypatch, capsys)
    for d, n in (("rendered_rgb", "gs"), ("rendered_depth", "gs"), ("rgb", "gt"), ("depth", "gt")):
        assert sorted(os.listdir(os.path.join(run_dir, d))) == ["%s_0000.png" % n, "%s_0004.png" % n]
    tool = _load(os.path.join(ROOT, "tools", "eval_record.py"), "eval_record")
    rec_path = os.path.join(run_dir, "params.npz")
    line = _run(tool, ["eval_record.py"] + data + ["--record", rec_path], monkeypatch, capsys)
    assert line["out"] == os.path.join(run_dir, "eval_train") and line["evaluated_frames"] == 2
    for k in ("psnr_db", "ms_ssim", "depth_l1_m", "ate_m"):
        assert line[k] == run[k], k
    for d in ("rendered_rgb", "rendered_depth", "rgb", "depth"):
        for f in os.listdir(os.path.join(run_dir, d)):
            from PIL import Image
            with Image.open(os.path.join(run_dir, d, f)) as x, Image.open(os.path.join(line["out"], d, f)) as y:
                assert np.array_equal(np.array(x), np.array(y)), (d, f)
    rec = formats.load_params(rec_path, cuda_device)
    with datasets.RGBDSequence("replica", str(tmp_path), "room0", desired_height=680, desired_width=1200,
                               device=cuda_device) as seq:
        frames = [seq[t] for t in range(T)]
        gt_w2c = [torch.linalg.inv(seq.files.poses[t].to(cuda_device)) for t in range(T)]
        direct = evaluate.evaluate({k: rec[k] for k in formats.CHECKPOINT_KEYS}, frames, seq.cam, 0.5, 60, True,
                                   eval_every=5, gt_w2c=gt_w2c)
    assert direct["psnr"] == line["psnr_db"] and direct["ms_ssim"] == line["ms_ssim"]
    assert direct["depth_l1"] == line["depth_l1_m"] and direct["ate"] == line["ate_m"]
    no_frames = str(tmp_path / "no_frames")
    _run(tool, ["eval_record.py"] + data + ["--record", rec_path, "--out", no_frames, "--no-frames"], monkeypatch,
         capsys)
    assert sorted(os.listdir(no_frames)) == ["l1.txt", "psnr.txt", "rmse.txt", "ssim.txt"]


def test_eval_record_test_split(cuda_device, tmp_path, monkeypatch, capsys):
    from test_evaluate_nvs_gpu import _write_replicav2
    from splatam_b200 import datasets, evaluate, formats
    _write_replicav2(str(tmp_path), 11, cuda_device)
    data = ["--dataset", "replicav2", "--basedir", str(tmp_path), "--sequence", "room_0"]
    run_dir = str(tmp_path / "run")
    run = _run(_load(os.path.join(ROOT, "tools", "run_slam_dataset.py"), "run_slam_dataset"),
               ["run_slam_dataset.py"] + data + ["--tracking-iters", "10", "--mapping-iters", "10", "--out", run_dir,
                                                 "--nvs", "--save-frames"], monkeypatch, capsys)
    nvs_dir = os.path.join(run_dir, "eval_nvs")
    views = ["0000", "0004"]                             # test views k = t - 1 for t = 1 and 5 (eval_every 5)
    for d, n in (("rendered_rgb", "splatam"), ("rendered_depth", "splatam"), ("rgb", "gt"), ("depth", "gt")):
        assert sorted(os.listdir(os.path.join(nvs_dir, d))) == ["%s_%s.png" % (n, k) for k in views]
    tool = _load(os.path.join(ROOT, "tools", "eval_record.py"), "eval_record")
    rec_path = os.path.join(run_dir, "params.npz")
    out = str(tmp_path / "nvs")
    line = _run(tool, ["eval_record.py"] + data + ["--record", rec_path, "--split", "test", "--out", out],
                monkeypatch, capsys)
    assert line["psnr_db"] == run["nvs_psnr_db"] and line["ms_ssim"] == run["nvs_ms_ssim"]
    assert line["depth_l1_m"] == run["nvs_depth_l1_m"] and line["valid_frames"] == run["nvs_valid_frames"]
    for d, n in (("rendered_rgb", "splatam"), ("rendered_depth", "splatam"), ("rgb", "gt"), ("depth", "gt")):
        assert sorted(os.listdir(os.path.join(out, d))) == ["%s_%s.png" % (n, k) for k in views]
    rec = formats.load_params(rec_path, cuda_device)
    with datasets.RGBDSequence("replicav2", str(tmp_path), "room_0", desired_height=680, desired_width=1200,
                               device=cuda_device, split="test") as test:
        direct = evaluate.evaluate_nvs({k: rec[k] for k in formats.GAUSSIAN_KEYS}, test, test.cam, 0.5, 60, True,
                                       eval_every=5)
    assert direct["psnr"] == line["psnr_db"] and direct["depth_l1"] == line["depth_l1_m"]
    np.testing.assert_array_equal(np.loadtxt(os.path.join(out, "psnr.txt")), direct["psnr_per_frame"])
