"""Generates tests/golden/capture/ref_capture.npz by running the reference's UNMODIFIED capture code on the CPU over
seeded small packets, with stand-ins bound only while it runs:

* `cyclonedds`: a module tree whose DataReader serves the prepared packets (its read_next returns None once, as a
  reader with nothing waiting does); colour is 7.5x the depth's size in each axis, as on the phone (60x45 from 8x6),
  depth holds NaN, +-inf, negative and over-range values, and packet 2 has no depth.
* R/scripts/nerfcapture2dataset.py's dataset_capture_loop writes a capture; its files and transforms.json bytes are
  stored.
* R/scripts/iphone_demo.py's dataset_capture_loop, with `Tensor.cuda` the identity and the SLAM functions it imports
  replaced by recorders (tracking runs one recorded iteration, mapping none): each frame's tracking-size and
  densification-size colour and depth, both intrinsics, gt_w2c per frame, the params.npz fields it saves, and the
  capture it writes.
* R/datasets/gradslam_datasets/nerfcapture.py's NeRFCaptureDataset over the capture the demo wrote (through the
  stand-ins of make_golden_datasets.py): frames, poses and intrinsics at 22x30 (desired = half size, not an exact 2x).
* For full-size packets (1920x1440 colour, 256x192 depth) only a seed and SHA-256 digests of cv2's outputs are stored:
  INTER_LINEAR colour at 720x960 and 360x480, INTER_NEAREST float depth at both sizes, and the saved uint16 depth.

Run:  python tests/golden/capture/make_golden_capture.py   (needs cv2 and the reference installed by oracle/reference.py)
"""
import contextlib
import hashlib
import importlib.util
import io
import os
import sys
import tempfile
import types
from pathlib import Path

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(os.path.dirname(HERE)))
SRC = os.path.join(ROOT, "oracle", "_ref", "SplaTAM")

N_PACKETS = 7                 # packet 2 has no depth, so 6 frames
NO_DEPTH = 2
SIZE = dict(width=60, height=45, depth_width=8, depth_height=6)
DEMO = dict(downscale_factor=2.0, densify_downscale_factor=4.0)
FULL_SEED = 2031
FULL_SIZES = ((720, 960), (360, 480))


def _datasets_generator():
    spec = importlib.util.spec_from_file_location(
        "make_golden_datasets", os.path.join(ROOT, "tests", "golden", "datasets", "make_golden_datasets.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def special_depth(g, h, w):
    """float32 metres with the values the cast rules care about."""
    d = g.uniform(0.2, 6.0, (h, w)).astype(np.float32)
    flat = d.reshape(-1)
    flat[:8] = [np.nan, np.inf, -np.inf, -0.5, 10.5, 0.0, 3.3e5, 1e9]
    g.shuffle(flat)
    return d


def c2w(g, t):
    from scipy.spatial.transform import Rotation
    m = np.eye(4)
    m[:3, :3] = Rotation.from_rotvec(g.normal(0, 0.2, 3) + [0.0, 0.05 * t, 0.0]).as_matrix()
    m[:3, 3] = g.normal(0, 0.5, 3) + [0.02 * t, 0.0, -0.01 * t]
    return m


class Sample:
    pass


def make_packets(seed=2030):
    """The packets as attribute objects with the DDS message's fields (float32 values stored as Python floats)."""
    g = np.random.default_rng(seed)
    out = []
    f32 = lambda v: float(np.float32(v))
    for t in range(N_PACKETS):
        s = Sample()
        s.id, s.timestamp = t, 0.125 * t
        s.fl_x, s.fl_y, s.cx, s.cy = f32(45.3), f32(44.9), f32(29.7), f32(22.1)
        s.transform_matrix = [f32(v) for v in c2w(g, t).T.reshape(-1)]
        s.width, s.height = SIZE["width"], SIZE["height"]
        s.image = g.integers(0, 256, (s.height, s.width, 3), dtype=np.uint8).reshape(-1).tolist()
        s.has_depth = t != NO_DEPTH
        s.depth_width, s.depth_height, s.depth_scale = SIZE["depth_width"], SIZE["depth_height"], f32(1.0)
        d = special_depth(g, s.depth_height, s.depth_width)
        s.depth_image = d.view(np.uint8).reshape(-1).tolist() if s.has_depth else []
        out.append(s)
    return out


@contextlib.contextmanager
def cyclonedds_stub(packets):
    """A cyclonedds module tree whose DataReader serves `packets` (None once before each)."""
    names = ["cyclonedds", "cyclonedds.idl", "cyclonedds.idl.annotations", "cyclonedds.idl.types",
             "cyclonedds.domain", "cyclonedds.core", "cyclonedds.sub", "cyclonedds.topic", "cyclonedds.util"]
    mods = {n: types.ModuleType(n) for n in names}

    class IdlStruct:
        def __init_subclass__(cls, **kw):
            pass
    mods["cyclonedds.idl"].IdlStruct = IdlStruct
    ann = mods["cyclonedds.idl.annotations"]
    ann.final = lambda c: c
    ann.autoid = lambda *a: (lambda c: c)
    ann.key = lambda *a: None
    tp = mods["cyclonedds.idl.types"]
    for n in ("uint8", "uint32", "float32", "float64"):
        setattr(tp, n, int)
    tp.array = tp.sequence = types.SimpleNamespace(__getitem__=None)

    class _Generic:
        def __class_getitem__(cls, item):
            return list
    tp.array = tp.sequence = _Generic

    class Reader:
        def __init__(self, *a, **k):
            self.queue = []
            for p in packets:
                self.queue += [None, p]

        def read_next(self):
            if not self.queue:
                raise RuntimeError("the stand-in reader ran out of packets")
            return self.queue.pop(0)
    mods["cyclonedds.sub"].DataReader = Reader
    for n, attrs in (("cyclonedds.domain", ("DomainParticipant", "Domain")), ("cyclonedds.core", ("Qos", "Policy")),
                     ("cyclonedds.topic", ("Topic",)), ("cyclonedds.util", ("duration",))):
        for a in attrs:
            setattr(mods[n], a, lambda *x, **k: None)
    saved = {k: sys.modules.get(k) for k in mods}
    sys.modules.update(mods)
    try:
        yield Reader
    finally:
        for k, v in saved.items():
            if v is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = v


def _load(name, path):
    spec = importlib.util.spec_from_file_location(name, path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def read_tree(root):
    out = {}
    for dirpath, _, files in os.walk(root):
        for f in files:
            p = os.path.join(dirpath, f)
            with open(p, "rb") as fh:
                out[os.path.relpath(p, root)] = fh.read()
    return out


def run_capture_script(packets, dst):
    with cyclonedds_stub(packets) as Reader:
        mod = _load("ref_nerfcapture2dataset", os.path.join(SRC, "scripts", "nerfcapture2dataset.py"))
        try:
            mod.dataset_capture_loop(Reader(), Path(dst), False, N_PACKETS, 10.0)
        except SystemExit as e:
            assert e.code == 0, e.code
    return read_tree(dst)


@contextlib.contextmanager
def demo_stand_ins(rec):
    """The modules iphone_demo.py imports besides cv2, numpy, torch and the reference's geometryutils."""
    names = ["matplotlib", "matplotlib.pyplot", "tqdm", "utils", "utils.common_utils", "utils.eval_helpers",
             "utils.keyframe_selection", "utils.recon_helpers", "utils.slam_external", "utils.slam_helpers",
             "scripts", "scripts.splatam", "diff_gaussian_rasterization"]
    mods = {n: types.ModuleType(n) for n in names}

    class Bar:
        def __init__(self, *a, **k):
            pass
        update = close = lambda self, *a: None
    mods["tqdm"].tqdm = Bar

    def frame(kind, data):
        rec.setdefault(kind, {})[int(data["id"])] = {k: (v.clone() if torch.is_tensor(v) else v)
                                                     for k, v in data.items() if k != "cam"}

    def report_progress(params, data, *a, **k):
        frame("tracking", data)

    def get_loss(params, data, variables, *a, **k):
        frame("tracking", data)
        return torch.zeros((), requires_grad=True), variables, {"depth": 0.0}

    def get_pointcloud(color, depth, intrinsics, w2c, **k):
        rec["densify0"] = dict(im=color.clone(), depth=depth.clone(), intrinsics=intrinsics.clone())
        return None, None

    def initialize_params(pt, num_frames, *a):
        rots = torch.zeros(1, 4, num_frames); rots[:, 0] = 1
        return dict(cam_unnorm_rots=rots, cam_trans=torch.zeros(1, 3, num_frames)), dict(timestep=torch.zeros(3))

    def add_new_gaussians(params, variables, data, *a):
        frame("densify", data)
        return params, variables

    def save_params(params, out):
        rec["params"] = {k: (v.clone() if torch.is_tensor(v) else v) for k, v in params.items()}

    opt = types.SimpleNamespace(step=lambda: None, zero_grad=lambda **k: None)
    m = mods
    m["utils.common_utils"].seed_everything = lambda **k: None
    m["utils.common_utils"].save_params_ckpt = lambda *a: None
    m["utils.common_utils"].save_params = save_params
    m["utils.eval_helpers"].report_progress = report_progress
    m["utils.keyframe_selection"].keyframe_selection_overlap = lambda *a: []
    m["utils.recon_helpers"].setup_camera = lambda w, h, k, w2c: dict(w=w, h=h)
    m["utils.slam_external"].build_rotation = lambda q: torch.eye(3)[None]
    m["utils.slam_external"].prune_gaussians = m["utils.slam_external"].densify = None
    m["utils.slam_helpers"].matrix_to_quaternion = None
    sp = m["scripts.splatam"]
    sp.get_loss, sp.initialize_params, sp.get_pointcloud, sp.add_new_gaussians = (get_loss, initialize_params,
                                                                                 get_pointcloud, add_new_gaussians)
    sp.initialize_optimizer = lambda *a, **k: opt
    sp.initialize_camera_pose = lambda params, t, **k: params
    m["diff_gaussian_rasterization"].GaussianRasterizer = None
    saved = {k: sys.modules.get(k) for k in mods}
    sys.modules.update(mods)
    cuda = torch.Tensor.cuda
    torch.Tensor.cuda = lambda self, *a, **k: self
    try:
        yield
    finally:
        torch.Tensor.cuda = cuda
        for k, v in saved.items():
            if v is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = v


def demo_config(workdir):
    h, w = SIZE["height"], SIZE["width"]
    f, fd = DEMO["downscale_factor"], DEMO["densify_downscale_factor"]
    return dict(workdir=workdir, run_name="SplaTAM_iPhone", overwrite=False, depth_scale=10.0, num_frames=N_PACKETS - 1,
                seed=0, map_every=1, keyframe_every=1, mapping_window_size=32, report_global_progress_every=100,
                scene_radius_depth_ratio=3, mean_sq_dist_method="projective", gaussian_distribution="isotropic",
                report_iter_progress=False, save_checkpoints=False, checkpoint_interval=5,
                data=dict(downscale_factor=f, densify_downscale_factor=fd, desired_image_height=int(h // f),
                          desired_image_width=int(w // f), densification_image_height=int(h // fd),
                          densification_image_width=int(w // fd)),
                tracking=dict(use_gt_poses=False, forward_prop=True, visualize_tracking_loss=False, num_iters=1,
                              use_sil_for_loss=True, sil_thres=0.99, use_l1=True, use_depth_loss_thres=False,
                              depth_loss_thres=20000, ignore_outlier_depth_loss=False, loss_weights={}, lrs={}),
                mapping=dict(num_iters=0, add_new_gaussians=True, sil_thres=0.5, use_l1=True,
                             ignore_outlier_depth_loss=False, use_sil_for_loss=False, loss_weights={}, lrs={},
                             prune_gaussians=True, pruning_dict={}, use_gaussian_splatting_densification=False,
                             densify_dict={}))


def run_demo(packets, dst):
    """iphone_demo.dataset_capture_loop over the packets (the reference's DataReader loop, all its conversions)."""
    rec = {}
    D = _datasets_generator()
    with D.reference_datasets(), cyclonedds_stub(packets) as Reader, demo_stand_ins(rec), \
            contextlib.redirect_stdout(io.StringIO()):
        mod = _load("ref_iphone_demo", os.path.join(SRC, "scripts", "iphone_demo.py"))
        cfg = demo_config(dst)
        mod.dataset_capture_loop(Reader(), Path(dst), False, cfg["num_frames"], cfg["depth_scale"], cfg)
    return rec


def full_size_digests():
    import cv2
    g = np.random.default_rng(FULL_SEED)
    rgb, depth = full_size_inputs(g)
    out = {}
    sha = lambda a: hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()
    for H, W in FULL_SIZES:
        out["color_%dx%d" % (H, W)] = sha(cv2.resize(rgb, (W, H), interpolation=cv2.INTER_LINEAR))
        out["depth_%dx%d" % (H, W)] = sha(cv2.resize(depth, (W, H), interpolation=cv2.INTER_NEAREST))
    with np.errstate(invalid="ignore"):
        q = (depth * 65535 / float(10.0)).astype(np.uint16)
    out["depth_u16"] = sha(cv2.resize(q, (1920, 1440), interpolation=cv2.INTER_NEAREST))
    return out


def full_size_inputs(g):
    """The full-size packet of FULL_SEED: uint8 [1440, 1920, 3] colour and float32 [192, 256] depth."""
    rgb = g.integers(0, 256, (1440, 1920, 3), dtype=np.uint8)
    depth = special_depth(g, 192, 256)
    depth.reshape(-1)[:4000] = g.uniform(-2.0, 12.0, 4000).astype(np.float32)    # negative and over-range depth
    return rgb, depth


def main():
    import torch  # noqa: F401
    packets = make_packets()
    out = {}
    with tempfile.TemporaryDirectory() as d:
        files = run_capture_script(packets, os.path.join(d, "script"))
        for k, v in sorted(files.items()):
            out["script/" + k] = np.frombuffer(v, np.uint8)
        demo_dir = os.path.join(d, "demo")
        rec = run_demo(packets, demo_dir)
        files = read_tree(demo_dir)
        for k, v in sorted(files.items()):
            out["demo/" + k] = np.frombuffer(v, np.uint8)
        T = N_PACKETS - 1
        for kind, key in (("tracking", "im"), ("tracking", "depth"), ("densify", "im"), ("densify", "depth")):
            frames = dict(rec[kind])
            if kind == "densify":
                frames[0] = rec["densify0"]
            out["demo_%s_%s" % (kind, key)] = np.stack([frames[t][key].numpy() for t in range(T)])
        out["demo_intrinsics"] = rec["tracking"][0]["intrinsics"].numpy()
        out["demo_densify_intrinsics"] = rec["densify0"]["intrinsics"].numpy()
        out["demo_gt_w2c"] = np.stack([m.numpy() for m in rec["tracking"][T - 1]["iter_gt_w2c_list"]])
        for k in ("intrinsics", "w2c", "org_width", "org_height", "gt_w2c_all_frames"):
            out["demo_params_" + k] = np.asarray(rec["params"][k])
        # the reader over the demo's capture
        D = _datasets_generator()
        with D.reference_datasets() as G:
            ds = G.NeRFCaptureDataset(d, "demo", desired_height=22, desired_width=30, device="cpu")
            cs, ds_, ps = [], [], []
            for t in range(len(ds)):
                color, depth, K, pose = ds[t]
                cs.append((color.permute(2, 0, 1) / 255).numpy())
                ds_.append(depth.permute(2, 0, 1).numpy())
                ps.append(pose.numpy())
            out["reader_color"], out["reader_depth"], out["reader_poses"] = np.stack(cs), np.stack(ds_), np.stack(ps)
            out["reader_intrinsics"] = K.numpy()
            out["reader_color_names"] = np.array([os.path.relpath(p, demo_dir) for p in ds.color_paths])
            out["reader_depth_names"] = np.array([os.path.relpath(p, demo_dir) for p in ds.depth_paths])
    for k, v in full_size_digests().items():
        out["digest_" + k] = np.array(v)
    out["full_seed"] = np.array(FULL_SEED)
    path = os.path.join(HERE, "ref_capture.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, "%d arrays, %.1f KB" % (len(out), os.path.getsize(path) / 1024))


if __name__ == "__main__":
    main()
