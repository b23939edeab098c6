"""Generates tests/golden/eval/ref_eval.npz by running the reference's UNMODIFIED final evaluation, `eval`
(R/utils/eval_helpers.py:408-623, imported through refsrc.load), on the CPU over synthetic inputs.

Stand-ins for what the CPU run lacks:
* the dataset is a list in the reference's format: HWC colour x 255, HWC depth, 4x4 intrinsics, c2w pose;
* `Renderer` returns preset images: it tells the depth/silhouette call from the RGB call by the colours (the
  silhouette column of [depth, 1, depth^2] is all ones) and the frame by the transformed position of Gaussian 0, which
  sits at the world origin and therefore lands on the frame's camera translation;
* pytorch_msssim.ms_ssim is bound to the float64 oracle (oracle/metrics_torch.py), so ssim.txt holds the oracle's value
  on exactly the tensors the reference hands to pytorch_msssim;
* LPIPS returns 0 and plotting is a no-op;
* Tensor.cuda is the identity and device="cuda" is dropped while the call runs (without that the ATE block fails on
  the CPU and `eval` silently reports 100).

`eval_case` builds every input from one seeded CPU torch.Generator; the tests call it too, so only the outputs are
stored: psnr / rmse / l1 / ssim per evaluated frame as the reference writes them, its ATE, the evaluated frame ids and
the valid / weighting-mask pixel counts (the reference's mask expressions, eval_helpers.py:467-480).
Run:  python tests/golden/eval/make_golden_eval.py   (needs the reference installed by oracle/reference.py)
"""
import contextlib
import os
import sys
import tempfile

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(os.path.dirname(HERE)))

# name: (H, W, frames, eval_every, mapping_iters, add_new_gaussians, frame with a NaN ground-truth pose, seed)
CASES = {
    "masked": (171, 199, 5, 1, 0, False, 3, 70),
    "unmasked_every3": (171, 199, 7, 3, 30, True, 4, 71),
}
SIL_THRES = 0.5


def _quat_w2c(q, t):
    q = q / q.norm()
    r, x, y, z = q.tolist()
    m = torch.eye(4)
    m[:3, :3] = torch.tensor([[1 - 2 * (y * y + z * z), 2 * (x * y - r * z), 2 * (x * z + r * y)],
                              [2 * (x * y + r * z), 1 - 2 * (x * x + z * z), 2 * (y * z - r * x)],
                              [2 * (x * z - r * y), 2 * (y * z + r * x), 1 - 2 * (x * x + y * y)]])
    m[:3, 3] = t
    return m


def eval_case(name):
    """Inputs of one case: dict(dataset=[(color HWC x255, depth HWC, K 4x4, c2w 4x4)], params (2 Gaussians plus
    cam_unnorm_rots [1,4,T] / cam_trans [1,3,T]), renders={t: (im [3,H,W], depth_sil [3,H,W])}, sil_thres,
    mapping_iters, add_new_gaussians, eval_every).  Rendered colours exceed 1 in a patch, the ground-truth depth has
    zero holes and part of each silhouette lies below the threshold."""
    H, W, T, eval_every, mapping_iters, add_new, nan_frame, seed = CASES[name]
    g = torch.Generator().manual_seed(seed)
    rnd = lambda *s: torch.rand(*s, generator=g)
    K = torch.tensor([[160.0, 0, (W - 1) / 2, 0], [0, 160.0, (H - 1) / 2, 0], [0, 0, 1, 0], [0, 0, 0, 1]])
    rots = torch.zeros(1, 4, T)
    trans = torch.zeros(1, 3, T)
    rots[0, 0] = 1.0
    dataset, renders = [], {}
    yy, xx = torch.meshgrid(torch.arange(H, dtype=torch.float32), torch.arange(W, dtype=torch.float32), indexing="ij")
    for t in range(T):
        gt_q = torch.tensor([1.0, 0.01 * t, -0.02 * t, 0.005 * t])
        gt_t = torch.tensor([0.05 * t, -0.02 * t, 0.03 * t])
        if t > 0:
            rots[0, :, t] = gt_q + 0.01 * torch.randn(4, generator=g)
            trans[0, :, t] = gt_t + 0.01 * torch.randn(3, generator=g)
        pose = torch.linalg.inv(_quat_w2c(gt_q, gt_t))
        if t == nan_frame:
            pose[1, 3] = float("nan")
        gt_im = 0.5 + 0.4 * torch.sin(xx / (7.0 + t) + torch.tensor([0.0, 1.0, 2.0])[:, None, None] + yy / 11.0)
        gt_im = (gt_im + 0.05 * rnd(3, H, W)).clamp(0, 1)
        gt_d = 1.0 + 2.0 * rnd(1, H, W)
        gt_d[:, 10:30, 20:60] = 0.0                                           # a hole
        gt_d[rnd(1, H, W) < 0.05] = 0.0                                       # scattered invalid pixels
        im = gt_im + 0.1 * torch.randn(3, H, W, generator=g)
        im[:, 100:140, 120:180] += 0.4                                        # rendered colours above 1
        sil = (0.3 + 0.7 * rnd(H, W)) * (0.5 + 0.5 * torch.sin(xx / 15.0 + t) ** 2)
        d = gt_d[0] + 0.05 * torch.randn(H, W, generator=g)
        d[gt_d[0] == 0] = 2.0
        depth_sil = torch.stack([d, sil, d * d + 0.01])
        renders[t] = (im, depth_sil)
        dataset.append(((gt_im * 255).permute(1, 2, 0).contiguous(), gt_d.permute(1, 2, 0).contiguous(), K, pose))
    params = dict(means3D=torch.tensor([[0.0, 0.0, 0.0], [0.3, -0.2, 2.0]]), rgb_colors=torch.tensor([[0.2, 0.4, 0.6],
                  [0.7, 0.1, 0.3]]), unnorm_rotations=torch.tensor([[1.0, 0, 0, 0], [1.0, 0, 0, 0]]),
                  logit_opacities=torch.zeros(2, 1), log_scales=torch.full((2, 1), -3.0), cam_unnorm_rots=rots,
                  cam_trans=trans)
    return dict(dataset=dataset, params=params, renders=renders, sil_thres=SIL_THRES, mapping_iters=mapping_iters,
                add_new_gaussians=add_new, eval_every=eval_every)


def frame_from_render_call(params, means3D):
    """The frame a render call belongs to: Gaussian 0 sits at the origin, so it lands on the frame's translation."""
    d = (params["cam_trans"][0].T - means3D[0].detach().reshape(1, 3)).norm(dim=1)
    return int(d.argmin())


@contextlib.contextmanager
def cpu_only():
    """Tensor.cuda is the identity and device="cuda" arguments are dropped while the block runs."""
    saved = {n: getattr(torch, n) for n in ("zeros", "zeros_like", "ones", "eye", "tensor")}
    cuda = torch.Tensor.cuda

    def strip(fn):
        return lambda *a, **k: fn(*a, **{kk: vv for kk, vv in k.items()
                                         if not (kk == "device" and str(vv).startswith("cuda"))})
    torch.Tensor.cuda = lambda self, *a, **k: self
    for n, fn in saved.items():
        setattr(torch, n, strip(fn))
    try:
        yield
    finally:
        torch.Tensor.cuda = cuda
        for n, fn in saved.items():
            setattr(torch, n, fn)


class _NoPlot:
    def subplots(self, *a, **k):
        return self, [self, self]

    def __getattr__(self, name):
        return lambda *a, **k: None


def run_reference(R, case):
    from oracle import metrics_torch
    E = R.eval_helpers
    rec = dict(ids=[], ate=[])

    class Renderer:
        def __init__(self, raster_settings=None):
            pass

        def __call__(self, means3D, colors_precomp, **rv):
            t = frame_from_render_call(case["params"], means3D)
            im, depth_sil = case["renders"][t]
            if bool((colors_precomp[:, 1] == 1).all()):
                rec["ids"].append(t)
                return depth_sil.clone(), torch.zeros(means3D.shape[0], dtype=torch.int32), None
            return im.clone(), torch.zeros(means3D.shape[0], dtype=torch.int32), None

    def ate(gt, est):
        v = evaluate_ate(gt, est)
        rec["ate"].append(v)
        return v
    evaluate_ate = E.evaluate_ate
    E.Renderer, E.evaluate_ate = Renderer, ate
    E.ms_ssim = metrics_torch.ms_ssim
    E.loss_fn_alex = lambda a, b: torch.tensor(0.0)
    E.plot_rgbd_silhouette = lambda *a, **k: None
    E.plt = _NoPlot()
    with tempfile.TemporaryDirectory() as d, cpu_only():
        E.eval(case["dataset"], case["params"], len(case["dataset"]), d, case["sil_thres"], case["mapping_iters"],
               case["add_new_gaussians"], eval_every=case["eval_every"])
        out = {n: np.atleast_1d(np.loadtxt(os.path.join(d, n + ".txt"))) for n in ("psnr", "rmse", "l1", "ssim")}
    assert len(rec["ate"]) == 1, "the reference's ATE block failed"
    out["ate"], out["ids"] = np.float64(rec["ate"][0]), np.array(rec["ids"], np.int64)
    use_presence = case["mapping_iters"] == 0 and not case["add_new_gaussians"]
    n_valid, n_mask = [], []
    for t in rec["ids"]:
        depth = case["dataset"][t][1].permute(2, 0, 1)
        valid = depth > 0
        presence = case["renders"][t][1][1] > case["sil_thres"]
        n_valid.append(int(valid.sum()))
        n_mask.append(int((presence * valid).sum() if use_presence else valid.sum()))
    out["n_valid"], out["n_mask"] = np.array(n_valid, np.int64), np.array(n_mask, np.int64)
    return out


class _Camera:
    def __init__(self, **kw):
        self.__dict__.update(kw)


def main():
    sys.path.insert(0, ROOT)
    import types
    import refsrc
    pkg = types.ModuleType("fake_rasterizer_pkg")
    pkg.GaussianRasterizer = object
    pkg.GaussianRasterizationSettings = _Camera
    R = refsrc.load(pkg)
    out = {}
    for name in CASES:
        for k, v in run_reference(R, eval_case(name)).items():
            out[name + "_" + k] = v
    path = os.path.join(HERE, "ref_eval.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, "%d arrays, %.1f KB" % (len(out), os.path.getsize(path) / 1024))
    for k, v in out.items():
        print(k, v)


if __name__ == "__main__":
    main()
