"""Generates tests/golden/eval/ref_eval_nvs.npz by running the reference's UNMODIFIED novel-view evaluation, `eval_nvs`
(R/utils/eval_helpers.py:626-841, imported through refsrc.load), on the CPU over synthetic test splits, with the
stand-ins of make_golden_eval.py: preset renders, pytorch_msssim bound to the float64 oracle, LPIPS 0, no plots,
Tensor.cuda the identity.

A test split is a list in the reference's format (HWC colour x 255, HWC depth, 4x4 intrinsics, c2w pose) whose frame 0
is the first train frame.  `Renderer` tells the frame of a call by the transformed position of Gaussian 0, which sits
at the world origin and therefore lands on the translation of the frame's ground-truth w2c, and the depth/silhouette
call from the RGB call by the colours.  The cases:
* unmasked_every1: mapping_iters > 0, every test view; the views have 0, exactly H*W/1000, H*W/1000 + 1 and many
  holes (gt depth > 0, silhouette <= sil_thres), so the first two are valid and the others are not;
* masked_every2: mapping_iters == 0 and no new Gaussians (presence-masked images and depth), eval_every 2;
* none_valid: every view has too many holes, so the averages are NaN.
`nvs_case` builds every input from one seeded CPU torch.Generator; the tests call it too, so only the outputs are
stored: psnr / rmse / l1 / ssim per evaluated view as the reference writes them, valid_nvs_frames.npy, the evaluated
frame indices and the valid-depth, weighting-mask and hole pixel counts (the reference's mask expressions).
Run:  python tests/golden/eval/make_golden_eval_nvs.py   (needs the reference installed by oracle/reference.py)
"""
import importlib.util
import os
import sys
import tempfile
import warnings

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(os.path.dirname(HERE)))


def _base():
    spec = importlib.util.spec_from_file_location("make_golden_eval", os.path.join(HERE, "make_golden_eval.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


B = _base()

H, W = 200, 250                                        # H * W = 50000: 50 holes are exactly 0.1 %
SIL_THRES = 0.5
# name: (frames incl. the first train frame, eval_every, mapping_iters, add_new_gaussians, holes per frame, seed)
CASES = {
    "unmasked_every1": (5, 1, 30, True, [0, 0, 50, 51, 400], 80),
    "masked_every2": (6, 2, 0, False, [0, 10, 50, 0, 3000, 20], 81),
    "none_valid": (3, 1, 30, True, [0, 60, 200], 82),
}


def nvs_case(name):
    """Inputs of one case: dict(dataset=[(color HWC x255, depth HWC, K 4x4, c2w 4x4)], params (2 isotropic Gaussians),
    renders={t: (im [3,H,W], depth_sil [3,H,W])}, gt_w2c [T,4,4], sil_thres, mapping_iters, add_new_gaussians,
    eval_every).  Frame t has exactly holes[t] hole pixels; other low-silhouette pixels lie where gt depth is 0."""
    T, eval_every, mapping_iters, add_new, holes, seed = CASES[name]
    g = torch.Generator().manual_seed(seed)
    rnd = lambda *s: torch.rand(*s, generator=g)
    K = torch.tensor([[180.0, 0, (W - 1) / 2, 0], [0, 180.0, (H - 1) / 2, 0], [0, 0, 1, 0], [0, 0, 0, 1]])
    yy, xx = torch.meshgrid(torch.arange(H, dtype=torch.float32), torch.arange(W, dtype=torch.float32), indexing="ij")
    dataset, renders, gt_w2c = [], {}, []
    for t in range(T):
        w2c = B._quat_w2c(torch.tensor([1.0, 0.02 * t, -0.01 * t, 0.015 * t]), torch.tensor([0.1 * t, -0.05 * t, 0.2]))
        gt_w2c.append(w2c)
        gt_im = 0.5 + 0.4 * torch.sin(xx / (9.0 + t) + torch.tensor([0.0, 1.0, 2.0])[:, None, None] + yy / 13.0)
        gt_im = (gt_im + 0.05 * rnd(3, H, W)).clamp(0, 1)
        gt_d = 1.0 + 2.0 * rnd(1, H, W)
        gt_d[:, 20:40, 30:80] = 0.0                                           # a hole in the gt depth
        im = gt_im + 0.1 * torch.randn(3, H, W, generator=g)
        im[:, 120:150, 150:200] += 0.4                                        # rendered colours above 1
        sil = 0.55 + 0.45 * rnd(H, W)
        sil[20:40, 30:80] = 0.2 * rnd(20, 50)                                 # uncovered, but no valid gt depth
        flat = torch.nonzero((gt_d[0] > 0).reshape(-1)).reshape(-1)
        pick = flat[torch.randperm(flat.numel(), generator=g)[:holes[t]]]
        sil.view(-1)[pick] = SIL_THRES * rnd(pick.numel())                    # the holes: <= sil_thres
        sil.view(-1)[pick[:1]] = SIL_THRES                                    # one exactly at the threshold
        d = gt_d[0] + 0.05 * torch.randn(H, W, generator=g)
        d[gt_d[0] == 0] = 2.0
        renders[t] = (im, torch.stack([d, sil, d * d + 0.01]))
        dataset.append(((gt_im * 255).permute(1, 2, 0).contiguous(), gt_d.permute(1, 2, 0).contiguous(), K,
                        torch.linalg.inv(w2c)))
    params = dict(means3D=torch.tensor([[0.0, 0.0, 0.0], [0.3, -0.2, 2.0]]), rgb_colors=torch.tensor([[0.2, 0.4, 0.6],
                  [0.7, 0.1, 0.3]]), unnorm_rotations=torch.tensor([[1.0, 0, 0, 0], [1.0, 0, 0, 0]]),
                  logit_opacities=torch.zeros(2, 1), log_scales=torch.full((2, 1), -3.0))
    return dict(dataset=dataset, params=params, renders=renders, gt_w2c=torch.stack(gt_w2c), sil_thres=SIL_THRES,
                mapping_iters=mapping_iters, add_new_gaussians=add_new, eval_every=eval_every)


def frame_from_render_call(gt_w2c, means3D):
    """The frame a render call belongs to: Gaussian 0 sits at the origin, so it lands on the translation of the
    frame's ground-truth w2c."""
    d = (gt_w2c[:, :3, 3] - means3D[0].detach().reshape(1, 3).to(gt_w2c)).norm(dim=1)
    return int(d.argmin())


def run_reference(R, case):
    from oracle import metrics_torch
    E = R.eval_helpers
    rec = dict(ids=[])

    class Renderer:
        def __init__(self, raster_settings=None):
            pass

        def __call__(self, means3D, colors_precomp, **rv):
            t = frame_from_render_call(case["gt_w2c"], means3D)
            im, depth_sil = case["renders"][t]
            if bool((colors_precomp[:, 1] == 1).all()):
                rec["ids"].append(t)
                return depth_sil.clone(), torch.zeros(means3D.shape[0], dtype=torch.int32), None
            return im.clone(), torch.zeros(means3D.shape[0], dtype=torch.int32), None

    E.Renderer = Renderer
    E.ms_ssim = metrics_torch.ms_ssim
    E.loss_fn_alex = lambda a, b: torch.tensor(0.0)
    E.plot_rgbd_silhouette = lambda *a, **k: None
    E.plt = B._NoPlot()
    with tempfile.TemporaryDirectory() as d, B.cpu_only(), warnings.catch_warnings():
        warnings.simplefilter("ignore", RuntimeWarning)               # the mean over no valid view
        E.eval_nvs(case["dataset"], case["params"], len(case["dataset"]), d, case["sil_thres"], case["mapping_iters"],
                   case["add_new_gaussians"], eval_every=case["eval_every"])
        out = {n: np.atleast_1d(np.loadtxt(os.path.join(d, n + ".txt"))) for n in ("psnr", "rmse", "l1", "ssim")}
        out["valid"] = np.load(os.path.join(d, "valid_nvs_frames.npy"))
    out["ids"] = np.array(rec["ids"], np.int64)
    use_presence = case["mapping_iters"] == 0 and not case["add_new_gaussians"]
    n_valid, n_mask, holes = [], [], []
    for t in rec["ids"]:
        valid = case["dataset"][t][1].permute(2, 0, 1) > 0
        presence = case["renders"][t][1][1] > case["sil_thres"]
        n_valid.append(int(valid.sum()))
        n_mask.append(int((presence * valid).sum() if use_presence else valid.sum()))
        holes.append(int((~(presence | ~valid)).sum()))
    out["n_valid"], out["n_mask"], out["holes"] = (np.array(v, np.int64) for v in (n_valid, n_mask, holes))
    return out


def main():
    sys.path.insert(0, ROOT)
    import types
    import refsrc
    pkg = types.ModuleType("fake_rasterizer_pkg")
    pkg.GaussianRasterizer = object
    pkg.GaussianRasterizationSettings = B._Camera
    R = refsrc.load(pkg)
    out = {}
    for name in CASES:
        for k, v in run_reference(R, nvs_case(name)).items():
            out[name + "_" + k] = v
    path = os.path.join(HERE, "ref_eval_nvs.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, "%d arrays, %.1f KB" % (len(out), os.path.getsize(path) / 1024))
    for k, v in out.items():
        print(k, v)


if __name__ == "__main__":
    main()
