"""Generates tests/golden/slam_s/ref_splatam_s.npz: SplaTAM-S's densification-resolution wiring as the reference's OWN
code computes it on the CPU, over the synthetic Replica sequence stored in tests/golden/datasets/ref_datasets.npz.

* initialize_first_timestep, get_pointcloud, initialize_params, initialize_new_params and add_new_gaussians are
  compiled from R/scripts/splatam.py's AST (importing the whole script needs wandb / matplotlib); setup_camera,
  transform_to_frame, transformed_params2depthplussilhouette and build_rotation come from the reference's utils
  modules (refsrc.load);
* the datasets are the reference's unmodified ReplicaDataset (make_golden_datasets.reference_datasets), with the
  real cv2: the desired size 48x64 and the densification size 24x32 (the exact 2x case), start 1, end 11, stride 5,
  so the retained frames are files 1 and 6.

Stored:
* init_*: initialize_first_timestep(dataset, densify_dataset=..., gaussian_distribution="isotropic",
  mean_sq_dist_method="projective", scene_radius_depth_ratio=3): the initial Gaussian rows, scene_radius, both 3x3
  intrinsics, and the fields of cam and densify_cam (image size, tanfov, viewmatrix, projmatrix, campos);
* add_*: add_new_gaussians for the second retained frame with densify_curr_data built as splatam.py:783-787, the
  parameters holding a fixed camera pose at that index, and a stand-in Renderer that records the raster settings it
  receives and returns a seeded depth / silhouette [3,24,32]: the settings it saw, the preset render, the pose, and
  the new rows.

The reference hard-codes `.cuda()` / device="cuda"; for this CPU run both are patched to stay on the CPU.  Nothing
is copied into the repository: the functions run where they lie.
Run:  python tests/golden/slam_s/make_golden_splatam_s.py   (needs the reference installed by oracle/reference.py)
"""
import ast
import importlib.util
import os
import sys
import tempfile
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.dirname(HERE)
ROOT = os.path.dirname(os.path.dirname(GOLDEN))
sys.path.insert(0, ROOT)
import refsrc  # noqa: E402

DESIRED = dict(desired_height=48, desired_width=64, start=1, end=11, stride=5)
DENSIFY = dict(desired_height=24, desired_width=32, start=1, end=11, stride=5)
TIME_IDX = 1                                           # the second retained frame
SIL_THRES = 0.5
CAM_FIELDS = ("image_height", "image_width", "tanfovx", "tanfovy", "viewmatrix", "projmatrix", "campos")
# the fixed camera pose of frame TIME_IDX (unnormalised quaternion, translation)
POSE_ROT = (0.998, 0.02, -0.035, 0.015)
POSE_TRANS = (0.03, -0.02, 0.05)


def datasets_generator():
    spec = importlib.util.spec_from_file_location("make_golden_datasets",
                                                  os.path.join(GOLDEN, "datasets", "make_golden_datasets.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def cpu_patches():
    torch.Tensor.cuda = lambda self, *a, **k: self
    for name in ("zeros", "zeros_like", "ones", "eye", "tensor"):
        orig = getattr(torch, name)
        setattr(torch, name, (lambda o: lambda *a, **k: o(*a, **{kk: vv for kk, vv in k.items()
                                                            if not (kk == "device" and str(vv).startswith("cuda"))}))(orig))


class Settings:       # stands in for diff_gaussian_rasterization.GaussianRasterizationSettings: keeps its fields
    def __init__(self, **kw):
        self.__dict__.update(kw)


def functions_from_source(path, names, namespace):
    tree = ast.parse(open(path).read())
    keep = [n for n in tree.body if isinstance(n, ast.FunctionDef) and n.name in names]
    exec(compile(ast.Module(body=keep, type_ignores=[]), path, "exec"), namespace)
    return [namespace[n] for n in names]


def cam_fields(cam):
    return {k: np.asarray(getattr(cam, k).numpy() if torch.is_tensor(getattr(cam, k)) else getattr(cam, k))
            for k in CAM_FIELDS}


def preset_depth_sil(depth):
    """A seeded depth / silhouette render [3,h,w]: silhouette uniform in [0,1] (about half the pixels below the
    threshold), depth near the observed one, a few pixels far behind it (the depth branch of the non-presence
    mask)."""
    g = torch.Generator().manual_seed(77)
    _, h, w = depth.shape
    ds = torch.zeros(3, h, w)
    ds[1] = torch.rand(h, w, generator=g)
    ds[0] = depth[0] * (1.0 + 0.02 * torch.randn(h, w, generator=g))
    far = torch.rand(h, w, generator=g) < 0.05
    ds[0][far] += 5.0
    ds[2] = ds[0] ** 2
    return ds


def main():
    gen = datasets_generator()
    fx = dict(np.load(os.path.join(GOLDEN, "datasets", "ref_datasets.npz")))
    cpu_patches()
    pkg = types.ModuleType("fake_rasterizer_pkg")
    pkg.GaussianRasterizer = object
    pkg.GaussianRasterizationSettings = Settings
    R = refsrc.load(pkg)
    ns = {"torch": torch, "np": np, "setup_camera": R.recon_helpers.setup_camera,
          "transform_to_frame": R.slam_helpers.transform_to_frame,
          "transformed_params2depthplussilhouette": R.slam_helpers.transformed_params2depthplussilhouette,
          "build_rotation": R.slam_external.build_rotation}
    initialize_first_timestep, add_new_gaussians = functions_from_source(
        os.path.join(R.root, "scripts", "splatam.py"),
        ["get_pointcloud", "initialize_params", "initialize_new_params", "initialize_first_timestep",
         "add_new_gaussians"], ns)[3:]
    out = {}
    with tempfile.TemporaryDirectory() as d, gen.reference_datasets() as G:
        gen.write_sequences(d, fx)
        root = os.path.join(d, "replica")
        dataset = G.ReplicaDataset(gen.config("replica"), root, gen.SEQUENCES["replica"], device="cpu", **DESIRED)
        densify_dataset = G.ReplicaDataset(gen.config("replica"), root, gen.SEQUENCES["replica"], device="cpu",
                                           **DENSIFY)
        num_frames = len(dataset)
        params, variables, intrinsics, first_frame_w2c, cam, densify_intrinsics, densify_cam = \
            initialize_first_timestep(dataset, num_frames, 3, "projective", densify_dataset=densify_dataset,
                                      gaussian_distribution="isotropic")
        P0 = params["means3D"].shape[0]
        for k in ("means3D", "rgb_colors", "unnorm_rotations", "logit_opacities", "log_scales"):
            out["init_" + k] = params[k].detach().numpy()
        out["init_scene_radius"] = np.float32(variables["scene_radius"])
        out["init_intrinsics"] = intrinsics.numpy()
        out["init_densify_intrinsics"] = densify_intrinsics.numpy()
        out["init_first_frame_w2c"] = first_frame_w2c.numpy()
        for tag, c in (("cam", cam), ("densify_cam", densify_cam)):
            for k, v in cam_fields(c).items():
                out["init_%s_%s" % (tag, k)] = v

        # add_new_gaussians on the densification-size frame TIME_IDX
        with torch.no_grad():
            params["cam_unnorm_rots"][..., TIME_IDX] = torch.tensor(POSE_ROT)[None]
            params["cam_trans"][..., TIME_IDX] = torch.tensor(POSE_TRANS)[None]
        densify_color, densify_depth, _, _ = densify_dataset[TIME_IDX]
        densify_color = densify_color.permute(2, 0, 1) / 255
        densify_depth = densify_depth.permute(2, 0, 1)
        densify_curr_data = {"cam": densify_cam, "im": densify_color, "depth": densify_depth, "id": TIME_IDX,
                             "intrinsics": densify_intrinsics, "w2c": first_frame_w2c, "iter_gt_w2c_list": None}
        depth_sil = preset_depth_sil(densify_depth)
        seen = []

        class Renderer:
            def __init__(self, raster_settings=None):
                seen.append(raster_settings)

            def __call__(self, **rv):
                assert rv["means3D"].shape[0] == P0
                return depth_sil.clone(), torch.zeros(P0, dtype=torch.int32), None
        ns["Renderer"] = Renderer
        params, variables = add_new_gaussians(params, variables, densify_curr_data, SIL_THRES, TIME_IDX,
                                              "projective", "isotropic")
        assert len(seen) == 1 and seen[0] is densify_cam
        for k, v in cam_fields(seen[0]).items():
            out["add_settings_" + k] = v
        n = params["means3D"].shape[0] - P0
        assert 0 < n < densify_depth.numel(), n
        for k in ("means3D", "rgb_colors", "unnorm_rotations", "logit_opacities", "log_scales"):
            out["add_new_" + k] = params[k].detach()[P0:].numpy()
        out["add_new_timestep"] = variables["timestep"][P0:].numpy()
        out["add_depth_sil"] = depth_sil.numpy()
        out["add_cam_unnorm_rots"] = params["cam_unnorm_rots"].detach().numpy()
        out["add_cam_trans"] = params["cam_trans"].detach().numpy()
        out["add_time_idx"] = np.int64(TIME_IDX)
        out["add_sil_thres"] = np.float32(SIL_THRES)
    path = os.path.join(HERE, "ref_splatam_s.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, "%d arrays, %.1f KB; %d initial Gaussians, %d added, scene_radius %.6f"
          % (len(out), os.path.getsize(path) / 1024, P0, n, float(out["init_scene_radius"])))


if __name__ == "__main__":
    main()
