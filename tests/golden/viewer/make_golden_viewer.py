"""Generates tests/golden/viewer/ref_viewer.npz by running the reference's UNMODIFIED viewers -- `visualize` of
viz_scripts/final_recon.py and of viz_scripts/online_recon.py, with their load_camera, load_scene_data,
get_rendervars, render, rgbd2pcd and make_lineset -- on the CPU, from the install in oracle/_ref.

Stand-ins (the viewers' window and plotting libraries are absent here):
  * open3d: a Visualizer whose view control hands back the camera it was given, geometries that record their points,
    colours and lines, and `LineSet.create_camera_visualization` recording its arguments; Vector3dVector / Vector2iVector
    are np.asarray.  poll_events lets online_recon step through every frame once, then ends both loops.
  * matplotlib: `get_cmap(name)(x)` returns (x, x, x, 1), so the recorded "colour" of each frustum and trajectory
    segment is the colormap argument the reference computed; `Normalize` records vmax; `ScalarMappable.to_rgba` returns
    zeros, so rgbd2pcd's depth-mode colours are 1 - mask and reveal its `d < 15` mask.
  * online_recon's wall clock: time.time() steps by one frame per call (viz_fps = 1), so frame t is visited at step t.
  * the renderer: oracle/bruteforce_torch.py in float32 behind the reference's GaussianRasterizer call; Tensor.cuda is
    the identity and device="cuda" arguments are dropped (tests/golden/eval/make_golden_eval.py:cpu_only).

Records (`record_arrays`, seeded, in the reference's params.npz layout): `mono` (non-decreasing timestep, as SLAM
leaves it) and `shuffled` (the same Gaussians in a seeded order, timestep not monotone, as offline densification
leaves it).  Runs (`RUNS`): the final view with and without offset_first_viz_cam, in colour and depth mode, and the
online view in colour, depth and centres mode on both records.  Stored per run `<run>_...`: k, all_w2cs, the view w2c
of every render (`view_w2c`, [n,4,4]), the selected rendervars of every displayed frame (concatenated, with
`frame_counts`), the frustum arguments (w2c, k, w, h, size) and colormap arguments, the trajectory's points, lines
and colormap arguments, and rgbd2pcd's inputs (depth), points and depth-mode mask and vmax.
Run:  python tests/golden/viewer/make_golden_viewer.py   (needs the reference installed by oracle/reference.py)"""
import importlib.util
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(os.path.dirname(HERE)))

T, P = 4, 60
VIZ = dict(render_mode="color", offset_first_viz_cam=True, show_sil=False, visualize_cams=True, viz_w=48, viz_h=32,
           viz_near=0.01, viz_far=100.0, view_scale=2, viz_fps=1, enter_interactive_post_online=True)
# name: (script, record, viz overrides)
RUNS = {
    "final_color": ("final_recon", "mono", dict()),
    "final_depth_nooffset": ("final_recon", "mono", dict(render_mode="depth", offset_first_viz_cam=False)),
    "online_color": ("online_recon", "mono", dict()),
    "online_depth": ("online_recon", "mono", dict(render_mode="depth")),
    "online_centers_shuffled": ("online_recon", "shuffled", dict(render_mode="centers")),
    "online_color_shuffled": ("online_recon", "shuffled", dict()),
}


def record_arrays(name):
    """The params.npz arrays of record `name` (float32 Gaussians and cameras, 0-d int64 sizes)."""
    g = torch.Generator().manual_seed(11)
    means = torch.cat([(torch.rand(P, 2, generator=g) - 0.5) * 1.6, 1.0 + 2.5 * torch.rand(P, 1, generator=g)], 1)
    means[:4, 2] = 20.0                                  # far behind the rest: depth mode's d >= 15 pixels
    rec = dict(means3D=means, rgb_colors=torch.rand(P, 3, generator=g),
               unnorm_rotations=torch.randn(P, 4, generator=g),
               logit_opacities=torch.randn(P, 1, generator=g) + 1.0,
               log_scales=torch.log(0.05 + 0.1 * torch.rand(P, 1, generator=g)),
               timestep=torch.sort(torch.randint(0, T, (P,), generator=g).float()).values)
    rots = torch.zeros(1, 4, T)
    rots[0, 0] = 1.0
    rots[0, 1:] = 0.03 * torch.randn(3, T, generator=g)
    rots[0, :, 0] = torch.tensor([1.0, 0, 0, 0])
    trans = 0.05 * torch.randn(1, 3, T, generator=g)
    trans[..., 0] = 0
    out = {k: v.numpy().astype(np.float32) for k, v in rec.items()}
    out.update(cam_unnorm_rots=rots.numpy(), cam_trans=trans.numpy(),
               intrinsics=np.array([[60.0, 0, 31.5], [0, 58.0, 23.5], [0, 0, 1]], np.float32),
               w2c=np.eye(4, dtype=np.float32), org_width=np.array(64, np.int64), org_height=np.array(48, np.int64),
               gt_w2c_all_frames=np.tile(np.eye(4, dtype=np.float32), (T, 1, 1)),
               keyframe_time_indices=np.arange(T, dtype=np.int64))
    if name == "shuffled":
        perm = torch.randperm(P, generator=torch.Generator().manual_seed(12)).numpy()
        for k in ("means3D", "rgb_colors", "unnorm_rotations", "logit_opacities", "log_scales", "timestep"):
            out[k] = out[k][perm]
    return out


class _Rec:
    """What the stand-ins saw during one visualize() call."""

    def __init__(self):
        self.frustums, self.lines, self.views, self.rv_views, self.selected, self.pcd = [], [], [], [], [], []


def _open3d(rec, polls):
    o3d = types.ModuleType("open3d")
    as_array = lambda x: np.asarray(x)

    class Geometry:
        def __init__(self):
            self.points = self.colors = self.lines = None

        def paint_uniform_color(self, c):
            self.paint = np.asarray(c)

    class LineSet(Geometry):
        @staticmethod
        def create_camera_visualization(w, h, k, w2c, size):
            ls = LineSet()
            ls.args = (w, h, np.array(k), np.array(w2c), size)
            return ls

    class Intrinsic:
        intrinsic_matrix, height, width = None, None, None

    class Pinhole:
        def __init__(self):
            self.extrinsic, self.intrinsic = None, Intrinsic()

    class ViewControl:
        def convert_from_pinhole_camera_parameters(self, p, allow_arbitrary=False):
            self.ext = np.array(p.extrinsic, np.float64)          # Open3D holds the camera in double precision
            self.k = np.array(p.intrinsic.intrinsic_matrix, np.float64)

        def convert_to_pinhole_camera_parameters(self):
            p = Pinhole()
            p.extrinsic, p.intrinsic.intrinsic_matrix = self.ext.copy(), self.k.copy()
            return p

    class Visualizer:
        def __init__(self):
            self.vc, self.calls = ViewControl(), 0

        def create_window(self, **k):
            pass

        def add_geometry(self, g):
            if isinstance(g, LineSet):
                (rec.frustums if hasattr(g, "args") else rec.lines).append(g)

        remove_geometry = update_geometry = update_renderer = destroy_window = lambda self, *a: None

        def poll_events(self):
            self.calls += 1
            return self.calls < polls

        def get_view_control(self):
            return self.vc

        def get_render_option(self):
            return types.SimpleNamespace()

    o3d.geometry = types.SimpleNamespace(PointCloud=Geometry, LineSet=LineSet)
    o3d.utility = types.SimpleNamespace(Vector3dVector=as_array, Vector2iVector=as_array)
    o3d.camera = types.SimpleNamespace(PinholeCameraParameters=Pinhole)
    o3d.visualization = types.SimpleNamespace(Visualizer=Visualizer)
    return o3d


def _matplotlib(rec):
    plt = types.ModuleType("matplotlib.pyplot")

    class Normalize:
        def __init__(self, vmin=0, vmax=1):
            rec.vmax = float(vmax)

    class ScalarMappable:
        def __init__(self, norm=None, cmap=None):
            pass

        def to_rgba(self, x):
            return np.zeros((len(x), 4))

    plt.get_cmap = lambda name: (lambda x: (float(x), float(x), float(x), 1.0))
    plt.Normalize = Normalize
    plt.cm = types.SimpleNamespace(ScalarMappable=ScalarMappable)
    mpl = types.ModuleType("matplotlib")
    mpl.pyplot = plt
    return mpl, plt


def _rasterizer(rec):
    from oracle import bruteforce_torch as BF
    pkg = types.ModuleType("diff_gaussian_rasterization")

    class Camera:
        def __init__(self, **kw):
            self.__dict__.update(kw)

    class Renderer:
        def __init__(self, raster_settings=None):
            self.s = raster_settings

        def __call__(self, means3D, means2D, opacities, colors_precomp, scales, rotations):
            s = self.s
            out = BF.render(means3D, colors_precomp, opacities, scales, rotations, width=s.image_width,
                            height=s.image_height, tanfovx=s.tanfovx, tanfovy=s.tanfovy, bg=s.bg,
                            viewmatrix=s.viewmatrix[0], projmatrix=s.projmatrix[0], means2D=means2D,
                            dtype=torch.float32)
            return out["color"], out["radii"], out["depth"]

    pkg.GaussianRasterizer, pkg.GaussianRasterizationSettings = Renderer, Camera
    return pkg


def _load_script(script, rec, polls):
    """viz_scripts/<script>.py from oracle/_ref with the stand-ins in sys.modules for the import."""
    import refsrc
    root = refsrc.ref_root()
    path = None if root is None else os.path.join(root, "viz_scripts", script + ".py")
    if path is None or not os.path.isfile(path):
        raise SystemExit("the reference's viz_scripts are not installed in oracle/_ref (oracle/reference_viz.py)")
    mpl, plt = _matplotlib(rec)
    stand_ins = {"open3d": _open3d(rec, polls), "matplotlib": mpl, "matplotlib.pyplot": plt,
                 "diff_gaussian_rasterization": _rasterizer(rec)}
    owned = lambda k: k in stand_ins or k == "utils" or k.startswith("utils.")
    saved = {k: sys.modules.pop(k) for k in [k for k in sys.modules if owned(k)]}
    added = refsrc._stub_missing()
    sys.modules.update(stand_ins)
    path_before = list(sys.path)
    try:
        spec = importlib.util.spec_from_file_location("_ref_" + script, path)
        mod = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(mod)
    finally:
        sys.path[:] = path_before
        for k in [k for k in sys.modules if owned(k)]:
            del sys.modules[k]
        for k in added:
            sys.modules.pop(k, None)
        sys.modules.update(saved)
    return mod


def run(name, record_path):
    script, _, over = RUNS[name]
    cfg = dict(VIZ, **over)
    rec = _Rec()
    mod = _load_script(script, rec, polls=T if script == "online_recon" else 1)
    load_camera, render, rgbd2pcd, get_rendervars = mod.load_camera, mod.render, mod.rgbd2pcd, \
        getattr(mod, "get_rendervars", None)
    rec.k = load_camera(cfg, record_path)[1].copy()

    def load_scene_data(*a):
        out = mod_load(*a)
        rec.all_w2cs = np.stack(out[-1])
        if script == "final_recon":
            rec.selected.append({k: out[0][k].clone() for k in ("means3D", "colors_precomp", "rotations", "opacities",
                                                                  "scales")})
        return out

    def rec_render(w2c, k, data, depth_data, c):
        rec.views.append(np.array(w2c, np.float32))
        return render(w2c, k, data, depth_data, c)

    def rec_rgbd2pcd(color, depth, w2c, k, c):
        pts, cols = rgbd2pcd(color, depth, w2c, k, c)
        rec.pcd.append((depth[0].numpy().copy(), np.asarray(pts), np.asarray(cols), np.array(w2c, np.float64),
                        np.array(k, np.float64), getattr(rec, "vmax", np.nan)))
        return pts, cols

    def rec_get_rendervars(params, w2c, curr_timestep):
        rv, drv = get_rendervars(params, w2c, curr_timestep)
        rec.selected.append({k: rv[k].clone() for k in ("means3D", "colors_precomp", "rotations", "opacities",
                                                          "scales")})
        rec.rv_views.append(np.array(w2c, np.float32))
        return rv, drv

    mod_load = mod.load_scene_data
    mod.load_scene_data, mod.render, mod.rgbd2pcd = load_scene_data, rec_render, rec_rgbd2pcd
    if get_rendervars is not None:
        mod.get_rendervars = rec_get_rendervars
        clock = iter([0.0] + [t + 0.5 for t in range(T)] + [T + 0.5] * 4)
        mod.time = types.SimpleNamespace(time=lambda: next(clock))
    sys.path.insert(0, os.path.join(ROOT, "tests", "golden", "eval"))
    from make_golden_eval import cpu_only
    with cpu_only(), torch.no_grad():
        mod.visualize(record_path, cfg)
    return rec


def pack(name, rec):
    online = RUNS[name][0] == "online_recon"
    # online_recon calls get_rendervars, render and rgbd2pcd once before its loop (frame 0 at the first-frame camera),
    # once per frame, and render / rgbd2pcd once more in its interactive loop; final_recon renders once before its
    # loop (at the first-frame camera, before the offset) and once in it
    frames = slice(1, T + 1) if online else slice(-1, None)
    views = rec.rv_views if online else rec.views
    out = {"k": rec.k, "all_w2cs": rec.all_w2cs, "view_w2c": np.stack(views[frames])}
    sel = rec.selected[frames] if online else rec.selected
    out["frame_counts"] = np.array([s["means3D"].shape[0] for s in sel], np.int64)
    for k in sel[0]:
        out["sel_" + k] = torch.cat([s[k] for s in sel]).numpy()
    if rec.frustums:
        out["frustum_w2c"] = np.stack([f.args[3] for f in rec.frustums])
        out["frustum_k"] = np.stack([f.args[2] for f in rec.frustums])
        out["frustum_whs"] = np.array([[f.args[0], f.args[1], f.args[4]] for f in rec.frustums], np.float64)
        out["frustum_cmap_x"] = np.array([f.paint[0] for f in rec.frustums])
    if rec.lines:
        last = rec.lines[-1]
        out["traj_points"] = np.asarray(last.points)
        out["traj_lines"] = np.asarray(last.lines)
        out["traj_cmap_x"] = np.asarray(last.colors)[:, 0]
        out["traj_cmap_x_per_frame"] = np.concatenate([np.asarray(l.colors)[:, 0] for l in rec.lines])
        out["traj_counts_per_frame"] = np.array([len(l.lines) for l in rec.lines], np.int64)
    pcd = rec.pcd[frames] if rec.pcd else []
    if pcd:
        out["pcd_depth"] = np.stack([p[0] for p in pcd])
        out["pcd_points"] = np.stack([p[1] for p in pcd])
        out["pcd_cols"] = np.stack([p[2] for p in pcd])
        out["pcd_w2c"] = np.stack([p[3] for p in pcd])
        out["pcd_k"] = np.stack([p[4] for p in pcd])
        out["pcd_vmax"] = np.array([p[5] for p in pcd])
    return {name + "_" + k: v for k, v in out.items()}


def main():
    import tempfile
    sys.path.insert(0, ROOT)
    out = {}
    with tempfile.TemporaryDirectory() as d:
        for r in ("mono", "shuffled"):
            arrays = record_arrays(r)
            np.savez(os.path.join(d, r + ".npz"), **arrays)
            out.update({"record_%s_%s" % (r, k): v for k, v in arrays.items()})
        for name, (_, r, _) in RUNS.items():
            rec = run(name, os.path.join(d, r + ".npz"))
            packed = pack(name, rec)
            out.update(packed)
            print(name, {k[len(name) + 1:]: v.shape for k, v in packed.items()})
    path = os.path.join(HERE, "ref_viewer.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, "%d arrays, %.1f KB" % (len(out), os.path.getsize(path) / 1024))


if __name__ == "__main__":
    main()
