"""Generates tests/golden/eval/ref_eval_frames.npz by running the reference's UNMODIFIED `eval` and `eval_nvs`
(R/utils/eval_helpers.py:408-623, 626-841, imported through refsrc.load) with save_frames=True on the CPU, with the real
cv2 and the stand-ins of make_golden_eval.py / make_golden_eval_nvs.py (preset renders told apart by the transformed
position of Gaussian 0, pytorch_msssim bound to the float64 oracle, LPIPS 0, no plots, Tensor.cuda the identity).

`frames_case` builds every input from one seeded CPU torch.Generator; the tests call it too, so only the outputs are
stored: for each case the names of the files the reference wrote under rendered_rgb/, rendered_depth/, rgb/ and depth/
(`<case>_files`, sorted) and their pixels as Pillow decodes them (`<case>_pixels`, uint8 [files, H, W, 3], same
order).  The images are smooth, so the archive stays small, and carry the values the pixel rules must get right:
rendered and ground-truth colours below 0 and above 1, float32 products that land exactly on k + 0.5, NaN and +-inf in
the render; depths below 0, at 0, above 6 m, exactly on the 6 * k / 255 boundaries and one float32 step either side,
and NaN and +-inf in the rendered depth.
Run:  python tests/golden/eval/make_golden_eval_frames.py   (needs the reference installed by oracle/reference.py)
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


def _load(name):
    spec = importlib.util.spec_from_file_location(name, os.path.join(HERE, name + ".py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


B = _load("make_golden_eval")
NVS = _load("make_golden_eval_nvs")

H, W = 168, 176
SIL_THRES = 0.5
DIRS = ("rendered_rgb", "rendered_depth", "rgb", "depth")
# name: (reference function, frames (for eval_nvs: the first train frame, then the test views), eval_every, seed)
CASES = {
    "eval": ("eval", 4, 2, 90),
    "eval_nvs": ("eval_nvs", 4, 2, 91),
}


def tie_values():
    """float32 x in [0, 1] whose float32 product x * 255 is exactly k + 0.5 (k = 0 .. 254): the round-half-to-even
    cases of cv2's saturate_cast."""
    out = []
    for k in range(255):
        x = np.float32((k + 0.5) / 255)
        for _ in range(8):
            p = np.float32(x * np.float32(255))
            if p == np.float32(k + 0.5):
                out.append(x)
                break
            x = np.nextafter(x, np.float32(2 if p < k + 0.5 else -1), dtype=np.float32)
    return torch.from_numpy(np.array(out, np.float32))


def depth_boundaries():
    """6 * k / 255 in float32 for k = 0 .. 255 and one float32 step below and above each."""
    b = (torch.arange(256, dtype=torch.float32) * 6) / 255
    below = torch.nextafter(b, torch.full_like(b, -1.0))
    above = torch.nextafter(b, torch.full_like(b, 10.0))
    return torch.stack([b, below, above], 1).reshape(-1)


_SPECIAL = torch.tensor([float("nan"), float("inf"), -float("inf"), -0.0, 0.0, 1.0, -1e-8, 1 + 1e-7, 1e30, -1e30])


def _rows(img, row, values):
    """Writes `values` into consecutive pixels of `img` [H, W] from the start of `row`, wrapping to the next rows."""
    img.view(-1)[row * W: row * W + values.numel()] = values


def _images(t, g):
    """(im [3,H,W], depth_sil [3,H,W], gt colour [3,H,W], gt depth [1,H,W]) of frame t."""
    yy, xx = torch.meshgrid(torch.arange(H, dtype=torch.float32), torch.arange(W, dtype=torch.float32), indexing="ij")
    ch = torch.tensor([0.0, 1.0, 2.0])[:, None, None]
    gt = 0.5 + 0.55 * torch.sin(xx / (19.0 + t) + ch + yy / 23.0)                    # -0.05 .. 1.05
    im = 0.5 + 0.7 * torch.sin(xx / (17.0 + t) + ch + yy / 21.0 + 0.1 * torch.rand(1, generator=g))   # -0.2 .. 1.2
    ties = tie_values()
    for c in range(3):
        _rows(im[c], 4, ties.roll(c))
        _rows(gt[c], 4, ties.roll(-c))
        _rows(im[c], 8, _SPECIAL.roll(c).repeat(3))
    d = 3.5 + 4.0 * torch.sin(xx / 29.0 + yy / 31.0 + 0.5 * t)                      # -0.5 .. 7.5
    gd = (3.0 + 3.5 * torch.sin(xx / 27.0 - yy / 33.0 + 0.3 * t))[None].clone()     # -0.5 .. 6.5
    gd[:, 100:130, 20:60] = 0.0                                                      # a hole
    bounds = depth_boundaries()
    _rows(d, 12, bounds)
    _rows(gd[0], 20, bounds.flip(0))
    _rows(d, 30, _SPECIAL.repeat(2))
    sil = 0.3 + 0.7 * torch.sin(xx / 15.0 + t) ** 2
    return im, torch.stack([d, sil, d * d + 0.01]), gt, gd


def frames_case(name):
    """Inputs of one case in the shape of make_golden_eval.eval_case (kind "eval") or make_golden_eval_nvs.nvs_case
    (kind "eval_nvs"): dict(kind, dataset, params, renders, sil_thres, mapping_iters, add_new_gaussians, eval_every,
    and gt_w2c [T,4,4] for eval_nvs)."""
    kind, T, eval_every, seed = CASES[name]
    g = torch.Generator().manual_seed(seed)
    K = torch.tensor([[150.0, 0, (W - 1) / 2, 0], [0, 150.0, (H - 1) / 2, 0], [0, 0, 1, 0], [0, 0, 0, 1]])
    rots = torch.zeros(1, 4, T)
    rots[0, 0] = 1.0
    trans = torch.zeros(1, 3, T)
    dataset, renders, gt_w2c = [], {}, []
    for t in range(T):
        w2c = B._quat_w2c(torch.tensor([1.0, 0.01 * t, -0.02 * t, 0.005 * t]),
                          torch.tensor([0.05 * t, -0.02 * t, 0.1 + 0.03 * t]))
        gt_w2c.append(w2c)
        trans[0, :, t] = w2c[:3, 3]
        im, depth_sil, gt, gd = _images(t, g)
        renders[t] = (im, depth_sil)
        dataset.append(((gt * 255).permute(1, 2, 0).contiguous(), gd.permute(1, 2, 0).contiguous(), K,
                        torch.linalg.inv(w2c)))
    params = dict(means3D=torch.tensor([[0.0, 0.0, 0.0], [0.3, -0.2, 2.0]]), rgb_colors=torch.tensor([[0.2, 0.4, 0.6],
                  [0.7, 0.1, 0.3]]), unnorm_rotations=torch.tensor([[1.0, 0, 0, 0], [1.0, 0, 0, 0]]),
                  logit_opacities=torch.zeros(2, 1), log_scales=torch.full((2, 1), -3.0))
    if kind == "eval":
        params.update(cam_unnorm_rots=rots, cam_trans=trans)
    return dict(kind=kind, dataset=dataset, params=params, renders=renders, gt_w2c=torch.stack(gt_w2c),
                sil_thres=SIL_THRES, mapping_iters=30, add_new_gaussians=True, eval_every=eval_every)


def render_frame_of(case, means3D):
    """The frame a render call of `case` belongs to (Gaussian 0 lands on the frame's camera translation)."""
    if case["kind"] == "eval":
        return B.frame_from_render_call(case["params"], means3D)
    return NVS.frame_from_render_call(case["gt_w2c"], means3D)


def read_frames(d):
    """(sorted relative paths of the PNGs under the four frame directories of `d`, their pixels as Pillow decodes
    them, uint8 [n, H, W, 3])."""
    from PIL import Image
    names = sorted(os.path.join(sub, f) for sub in DIRS if os.path.isdir(os.path.join(d, sub))
                   for f in os.listdir(os.path.join(d, sub)))
    pixels = []
    for n in names:
        with Image.open(os.path.join(d, n)) as im:
            pixels.append(np.array(im))
    return names, np.stack(pixels) if pixels else np.zeros((0, H, W, 3), np.uint8)


def run_reference(R, case):
    from oracle import metrics_torch
    E = R.eval_helpers

    class Renderer:
        def __init__(self, raster_settings=None):
            pass

        def __call__(self, means3D, colors_precomp, **rv):
            im, depth_sil = case["renders"][render_frame_of(case, means3D)]
            out = depth_sil if bool((colors_precomp[:, 1] == 1).all()) else im
            return out.clone(), torch.zeros(means3D.shape[0], dtype=torch.int32), None

    E.Renderer = Renderer
    E.ms_ssim = metrics_torch.ms_ssim
    E.loss_fn_alex = lambda a, b: torch.tensor(0.0)
    E.plot_rgbd_silhouette = lambda *a, **k: None
    E.plt = B._NoPlot()
    fn = getattr(E, case["kind"])
    with tempfile.TemporaryDirectory() as d, B.cpu_only(), warnings.catch_warnings(), \
            np.errstate(invalid="ignore", over="ignore"):
        warnings.simplefilter("ignore", RuntimeWarning)
        fn(case["dataset"], case["params"], len(case["dataset"]), d, case["sil_thres"], case["mapping_iters"],
           case["add_new_gaussians"], eval_every=case["eval_every"], save_frames=True)
        return read_frames(d)


def main():
    sys.path.insert(0, ROOT)
    import types
    import cv2  # noqa: F401  (the real cv2 writes the files; refsrc would stub it only if the import failed)
    import refsrc
    pkg = types.ModuleType("fake_rasterizer_pkg")
    pkg.GaussianRasterizer = object
    pkg.GaussianRasterizationSettings = B._Camera
    R = refsrc.load(pkg)
    out = {}
    for name in CASES:
        names, pixels = run_reference(R, frames_case(name))
        out[name + "_files"], out[name + "_pixels"] = np.array(names), pixels
        print(name, names)
    path = os.path.join(HERE, "ref_eval_frames.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, "%d arrays, %.1f KB" % (len(out), os.path.getsize(path) / 1024))


if __name__ == "__main__":
    main()
