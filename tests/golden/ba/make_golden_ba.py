"""Generates tests/golden/ba/ref_ba.npz: SplaTAM's mapping loop with keyframe-pose refinement as the reference's OWN
code computes it on the CPU -- the unmodified get_loss(mapping=True, do_ba=True) and initialize_optimizer(...,
tracking=False) of R/scripts/splatam.py and prune_gaussians of R/utils/slam_external.py, imported through refsrc.load,
with the float32 brute-force composite of oracle/bruteforce_torch.py as the rasterizer (the test renders with it too).

Two problems, a 160-Gaussian isotropic and a 160-Gaussian anisotropic map at 48x32, each with three keyframes rendered
from the unperturbed map at known poses; the map and all three camera columns start perturbed.  Eight mapping
iterations draw the keyframes in the fixed order ITER_IDS (keyframe 2 twice in a row) with the shipped Replica mapping
rates and non-zero camera rates; iteration PRUNE_ITER prunes, as the reference's loop does between backward and
optimizer.step(), so there the Gaussians take no Adam step and the cameras do.

Stored per problem: the inputs (map, cameras, frames, scene radius) and per iteration the drawn id, the loss, the full
gradients of cam_unnorm_rots [1,4,3] and cam_trans [1,3,3] and all seven tensors after the step.
`.cuda()` and device="cuda" are patched to stay on the CPU.  Nothing is copied into the repository: the functions run
where they lie.  Run:  python tests/golden/ba/make_golden_ba.py   (needs the reference installed by oracle/reference.py)
"""
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, ROOT)

T = 3
ITER_IDS = (1, 0, 2, 2, 1, 0, 1, 2)
PRUNE_ITER = 4
PRUNE = dict(start_after=PRUNE_ITER, remove_big_after=100, stop_after=PRUNE_ITER, prune_every=PRUNE_ITER,
             removal_opacity_threshold=0.1, final_removal_opacity_threshold=0.1, reset_opacities=False,
             reset_opacities_every=500)
CAM_LRS = dict(cam_unnorm_rots=0.0004, cam_trans=0.002)       # Replica's tracking rates
KEYS = ("means3D", "rgb_colors", "unnorm_rotations", "logit_opacities", "log_scales", "cam_unnorm_rots", "cam_trans")


def lrs(aniso):
    """Replica's mapping rates (R/configs/replica/splatam.py) and CAM_LRS.  An isotropic map's loss does not depend on
    its rotations: their gradient is rounding noise, which Adam would turn into +-lr steps, so their rate is 0 there."""
    return dict(means3D=0.0001, rgb_colors=0.0025, unnorm_rotations=0.001 if aniso else 0.0, logit_opacities=0.05,
                log_scales=0.001, **CAM_LRS)


def render(settings, means3D, means2D, opacities, colors_precomp, scales, rotations):
    """The rasterizer of both sides: oracle/bruteforce_torch.py in float32."""
    from oracle import bruteforce_torch as BF
    out = BF.render(means3D, colors_precomp, opacities, scales, rotations, width=settings.image_width,
                    height=settings.image_height, tanfovx=settings.tanfovx, tanfovy=settings.tanfovy, bg=settings.bg,
                    viewmatrix=settings.viewmatrix[0], projmatrix=settings.projmatrix[0], means2D=means2D,
                    dtype=torch.float32)
    return out["color"], out["radii"], out["depth"]


def camera(sc):
    import splatam_b200 as S
    return sc.settings(S.GaussianRasterizationSettings, "cpu")


def problem(aniso):
    """(initial map, initial cameras, frames [dict(id, im, depth)], scene radius) of one problem."""
    import scenes
    from splatam_b200 import slam
    sc = scenes.config1(seed=8, P=160, w=48, h=32)
    gt = dict(means3D=sc.means3D, rgb_colors=sc.colors, unnorm_rotations=sc.rotations,
              logit_opacities=torch.logit(sc.opacities.clamp(0.05, 0.95)),
              log_scales=torch.log(sc.scales if aniso else sc.scales[:, :1]))
    rots, trans = slam.look_trajectory(T, "cpu", step=(0.004, -0.002, 0.003), rot_step=(0.001, -0.001, 0.0005))
    cam = camera(sc)
    frames = []
    for t in range(T):
        fr = slam.render_frame(gt, rots, trans, t, cam, render=render)
        frames.append(dict(id=t, im=fr["im"], depth=fr["depth"]))
    g = torch.Generator().manual_seed(15 + int(aniso))
    init = {k: v + 0.02 * torch.randn(v.shape, generator=g) for k, v in gt.items()}
    cams = dict(cam_unnorm_rots=rots + 0.004 * torch.randn(rots.shape, generator=g),
                cam_trans=trans + 0.01 * torch.randn(trans.shape, generator=g))
    return init, cams, frames, float(frames[0]["depth"].max()) / 3.0


def cpu_patches():
    torch.Tensor.cuda = lambda self, *a, **k: self
    for name in ("zeros", "zeros_like", "ones", "eye"):
        orig = getattr(torch, name)
        setattr(torch, name, (lambda o: lambda *a, **k: o(*a, **{kk: vv for kk, vv in k.items()
                                                            if not (kk == "device" and str(vv).startswith("cuda"))}))(orig))


def run_reference(R, aniso, out):
    import scenes
    S_, E_ = R.splatam, R.slam_external
    cam = camera(scenes.config1(seed=8, P=160, w=48, h=32))
    init, cams, frames, radius = problem(aniso)
    tag = "aniso_" if aniso else "iso_"
    params = {k: torch.nn.Parameter(v.clone().float().contiguous().requires_grad_(True))
              for k, v in dict(init, **cams).items()}
    for k, v in params.items():
        out[tag + "in_" + k] = v.detach().numpy().copy()
    for t, fr in enumerate(frames):
        out[tag + "im%d" % t], out[tag + "depth%d" % t] = fr["im"].numpy(), fr["depth"].numpy()
    out[tag + "scene_radius"] = np.float64(radius)
    P = params["means3D"].shape[0]
    variables = dict(max_2D_radius=torch.zeros(P), means2D_gradient_accum=torch.zeros(P), denom=torch.zeros(P),
                     timestep=torch.zeros(P), scene_radius=torch.tensor(radius))
    optimizer = S_.initialize_optimizer(params, lrs(aniso), tracking=False)
    losses, counts = [], []
    for it, k in enumerate(ITER_IDS):
        data = dict(cam=cam, im=frames[k]["im"], depth=frames[k]["depth"], id=k, intrinsics=None, w2c=torch.eye(4),
                    iter_gt_w2c_list=None)
        loss, variables, _ = S_.get_loss(params, data, variables, k, dict(im=0.5, depth=1.0), use_sil_for_loss=False,
                                         sil_thres=0.5, use_l1=True, ignore_outlier_depth_loss=False, mapping=True,
                                         do_ba=True)
        loss.backward()
        out[tag + "grad_cam_unnorm_rots_%d" % it] = params["cam_unnorm_rots"].grad.numpy().copy()
        out[tag + "grad_cam_trans_%d" % it] = params["cam_trans"].grad.numpy().copy()
        with torch.no_grad():
            params, variables = E_.prune_gaussians(params, variables, optimizer, it, PRUNE)
            optimizer.step()
            optimizer.zero_grad(set_to_none=True)
        for key in KEYS:
            out[tag + "out_%s_%d" % (key, it)] = params[key].detach().numpy().copy()
        losses.append(float(loss.detach()))
        counts.append(params["means3D"].shape[0])
    out[tag + "loss"] = np.array(losses, np.float64)
    out[tag + "counts"] = np.array(counts, np.int64)
    return counts


def main():
    import refsrc
    cpu_patches()
    pkg = types.ModuleType("fake_rasterizer_pkg")
    pkg.GaussianRasterizer = object
    pkg.GaussianRasterizationSettings = object
    R = refsrc.load(pkg)

    class Renderer:               # stand-in for diff_gaussian_rasterization.GaussianRasterizer
        def __init__(self, raster_settings):
            self.s = raster_settings

        def __call__(self, **rv):
            return render(self.s, **rv)
    R.splatam.Renderer = Renderer
    out = dict(iter_ids=np.array(ITER_IDS, np.int64), prune_iter=np.int64(PRUNE_ITER))
    for aniso in (False, True):
        counts = run_reference(R, aniso, out)
        print("%s: Gaussians per iteration %s" % ("aniso" if aniso else "iso", counts))
    path = os.path.join(HERE, "ref_ba.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, "%d arrays, %.1f KB" % (len(out), os.path.getsize(path) / 1024))


if __name__ == "__main__":
    main()
