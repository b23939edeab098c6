"""Generates tests/golden/offline/ref_offline.npz from the reference's OWN offline-loop functions on the CPU:
get_loss_gs (R/scripts/post_splatam_opt.py, compiled from the script's AST: importing the script needs wandb, tqdm
and the dataset readers), params2rendervar / params2depthplussilhouette / get_depth_and_silhouette / l1_loss_v1
(R/utils/gs_helpers.py, compiled from its AST for the same reason), and densify / calc_ssim / get_expon_lr_func /
update_learning_rate (R/utils/gs_external.py, imported unmodified).  The rasterizer is the float32 brute-force
composite of oracle/bruteforce_torch.py, used by the test as well.

The loop is the one of post_splatam_opt.py from line 290 on: a 160-Gaussian map at 48x32, three frames (stride 1, so
the record's camera column t is frame t's pose in both readings), four iterations with seed_everything(0)'s frame
sequence, and a densify schedule that fires at iterations 3 and 6 (clones, splits, pruning, and an opacity reset at 6;
both Adam steps skipped).  Densify's split samples are the one random draw of the loop; the generator and the test
both draw them through `split_normal`, torch.normal from a generator seeded the same on every call, so every row of
the final map can be compared by value.  `.cuda()` and device="cuda" are patched to stay on the CPU.
Run:  python tests/golden/offline/make_golden_offline.py"""
import ast
import os
import random
import sys

import numpy as np
import torch
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, ROOT)
REF = "/root/reference"

T, ITERS, SEED = 3, 9, 0
SPLIT_SEED = 11
DENSIFY = dict(start_after=2, remove_big_after=0, stop_after=20, densify_every=3, grad_thresh=2e-6,
               num_to_split_into=2, removal_opacity_threshold=0.005, final_removal_opacity_threshold=0.005,
               reset_opacities=True, reset_opacities_every=6)
# the shipped rates, except unnorm_rotations: the map is isotropic, so the loss does not depend on the rotations and their
# gradient is rounding noise, which Adam turns into +-lr steps that differ between any two float orderings; the split
# samples are rotated by them, so at lr 0 every row of the map can be compared by value
LRS = dict(means3D=0.00032, rgb_colors=0.0025, unnorm_rotations=0.0, logit_opacities=0.05, log_scales=0.005,
           cam_unnorm_rots=0.0, cam_trans=0.0)
LR_FINAL = 0.0000032


def _functions(path, names, ns):
    """Compiles the top-level functions `names` of the file at `path` into namespace `ns`."""
    tree = ast.parse(open(path).read())
    body = [n for n in tree.body if isinstance(n, ast.FunctionDef) and n.name in names]
    assert sorted(n.name for n in body) == sorted(names), [n.name for n in body]
    exec(compile(ast.Module(body=body, type_ignores=[]), path, "exec"), ns)
    return ns


def split_normal(normal=torch.normal):
    """torch.normal for densify's split samples, drawn from a generator seeded with SPLIT_SEED on each call."""
    return lambda mean, std, generator=None: normal(mean=mean, std=std,
                                                     generator=torch.Generator().manual_seed(SPLIT_SEED))


def _patch_cuda():
    torch.Tensor.cuda = lambda self, *a, **k: self
    for name in ("zeros", "zeros_like", "ones", "eye"):
        orig = getattr(torch, name)
        setattr(torch, name, (lambda o: lambda *a, **k: o(*a, **{kk: vv for kk, vv in k.items()
                                                            if not (kk == "device" and str(vv).startswith("cuda"))}))(orig))


def problem():
    """The scene, the training frames (id, cam at identity, w2c, im, depth) and their poses, and the initial map --
    shared with tests/test_offline_cpu.py."""
    import scenes
    import splatam_b200 as S
    from oracle import bruteforce_torch as BF
    from splatam_b200 import mapping as M, slam

    def render(settings, means3D, means2D, opacities, colors_precomp, scales, rotations):
        out = BF.render(means3D, colors_precomp, opacities, scales, rotations, width=settings.image_width,
                        height=settings.image_height, tanfovx=settings.tanfovx, tanfovy=settings.tanfovy,
                        bg=settings.bg, viewmatrix=settings.viewmatrix[0], projmatrix=settings.projmatrix[0],
                        means2D=means2D, dtype=torch.float32)
        return out["color"], out["radii"], out["depth"]
    sc = scenes.config1(seed=8, P=160, w=48, h=32)
    cam = sc.settings(S.GaussianRasterizationSettings, "cpu")
    gt = dict(means3D=sc.means3D, rgb_colors=sc.colors, unnorm_rotations=sc.rotations,
              logit_opacities=torch.logit(sc.opacities.clamp(0.05, 0.95)), log_scales=torch.log(sc.scales[:, :1]))
    rots, trans = slam.look_trajectory(T, "cpu", step=(0.004, -0.002, 0.003), rot_step=(0.001, -0.001, 0.0005))
    frames = [slam.render_frame(gt, rots, trans, t, cam, render=render) for t in range(T)]
    g = torch.Generator().manual_seed(5)
    init = {k: v + 0.02 * torch.randn(v.shape, generator=g) for k, v in gt.items()}
    timestep = torch.randint(0, T, (sc.means3D.shape[0],), generator=g).float()
    K = torch.tensor([[sc.fx, 0.0, sc.cx], [0.0, sc.fy, sc.cy], [0.0, 0.0, 1.0]])
    return dict(sc=sc, cam=cam, frames=frames, rots=rots, trans=trans, init=init, timestep=timestep, K=K,
                render=render, w2c=[M.camera_w2c(rots[..., t], trans[..., t])[0] for t in range(T)])


def main():
    import splatam_b200 as S
    from splatam_b200 import datasets
    pr = problem()
    _patch_cuda()
    import importlib.util
    spec = importlib.util.spec_from_file_location("ref_gs_external", os.path.join(REF, "utils", "gs_external.py"))
    gx = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(gx)

    class Renderer:               # stand-in for diff_gaussian_rasterization.GaussianRasterizer
        def __init__(self, raster_settings):
            self.s = raster_settings

        def __call__(self, **rv):
            return pr["render"](self.s, **rv)
    ns = _functions(os.path.join(REF, "utils", "gs_helpers.py"),
                    ["params2rendervar", "params2depthplussilhouette", "get_depth_and_silhouette", "l1_loss_v1"],
                    dict(torch=torch, F=F))
    ns.update(Renderer=Renderer, calc_ssim=gx.calc_ssim)
    ns = _functions(os.path.join(REF, "scripts", "post_splatam_opt.py"), ["get_loss_gs", "initialize_optimizer"], ns)
    sc, frames = pr["sc"], pr["frames"]
    # initialize_first_timestep_from_ckpt: every record key but the popped ones becomes a parameter
    params = {k: v.clone().float().requires_grad_(True) for k, v in pr["init"].items()}
    params["cam_unnorm_rots"] = pr["rots"].clone().requires_grad_(True)
    params["cam_trans"] = pr["trans"].clone().requires_grad_(True)
    P = params["means3D"].shape[0]
    variables = dict(max_2D_radius=torch.zeros(P), means2D_gradient_accum=torch.zeros(P), denom=torch.zeros(P),
                     timestep=pr["timestep"].clone(), scene_radius=torch.max(frames[0]["depth"]) / 2.0)
    gs_cams = [datasets.setup_camera(sc.w, sc.h, pr["K"].numpy(), w.numpy(), "cpu") for w in pr["w2c"]]
    random.seed(SEED); np.random.seed(SEED); torch.manual_seed(SEED)         # seed_everything
    optimizer = ns["initialize_optimizer"](params, LRS)
    sched = gx.get_expon_lr_func(lr_init=LRS["means3D"], lr_final=LR_FINAL, lr_delay_mult=0.01, max_steps=ITERS)
    seq, lrs, losses, counts = [], [], [], []
    torch.normal = split_normal()
    for it in range(ITERS):
        lrs.append(gx.update_learning_rate(optimizer, sched, it + 1))
        k = random.randint(0, T - 1)
        data = {"cam": gs_cams[k], "im": frames[k]["im"], "depth": frames[k]["depth"], "id": k,
                "intrinsics": pr["K"], "w2c": pr["w2c"][k]}
        loss, variables, _ = ns["get_loss_gs"](params, data, variables, {"im": 0.5, "depth": 1.0})
        loss.backward()
        with torch.no_grad():
            params, variables = gx.densify(params, variables, optimizer, it, DENSIFY)
            optimizer.step()
            optimizer.zero_grad(set_to_none=True)
        seq.append(k); losses.append(float(loss.detach())); counts.append(params["means3D"].shape[0])
    out = dict(frame_seq=np.array(seq, np.int64), lr=np.array(lrs, np.float64), loss=np.array(losses, np.float64),
               counts=np.array(counts, np.int64), timestep=variables["timestep"].numpy(),
               scene_radius=np.float32(variables["scene_radius"]))
    for k in pr["init"]:
        out["out_" + k] = params[k].detach().numpy()
        st = optimizer.state[params[k]]
        out["out_" + k + "_exp_avg"], out["out_" + k + "_exp_avg_sq"] = st["exp_avg"].numpy(), st["exp_avg_sq"].numpy()
        out["out_" + k + "_step"] = np.float64(st["step"])
    np.savez_compressed(os.path.join(HERE, "ref_offline.npz"), **out)
    print("wrote ref_offline.npz: frames %s, counts %s" % (seq, counts))


if __name__ == "__main__":
    main()
