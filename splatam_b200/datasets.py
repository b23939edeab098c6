"""Readers for the datasets of SplaTAM's tables -- Replica, TUM-RGBD, ScanNet, ScanNet++ and ReplicaV2 -- that turn a
sequence on disk into the frame dicts `slam.run_slam`, `evaluate.evaluate` and `evaluate.evaluate_nvs` consume.

They follow the reference's loaders (R/datasets/gradslam_datasets/basedataset.py, replica.py, tum.py, scannet.py,
scannetpp.py):
the same files in the same (natural) order, the same `start / end / stride` subsampling, TUM's timestamp association,
poses relative to the first retained frame, intrinsics scaled to the desired size, and pixels decoded with Pillow
(imageio's backend for these formats).  What differs is where the per-frame work runs: the reference converts every
frame to float64 on the host, resizes it with cv2, divides the depth and uploads the float64 arrays (32 B per pixel)
from pageable memory, synchronously.  Here the raw uint8 colour and uint16 depth (5 B per pixel) are uploaded from pinned memory and one
CUDA kernel (csrc/ingest.cu, `ingest_rgbd`) resizes, scales and lays them out exactly as the reference's float path
does.  With `prefetch` > 0 a host thread decodes the next frames while the GPU works on the current one, and the
upload and the kernel run on a side stream that the consumer's stream waits on.  With a separate densification size
(SplaTAM-S) a second launch of the same kernel turns the already uploaded pixels into the frame at that size.

Dataset configs have the reference's YAML shape (``camera_params``: image_height / image_width, fx / fy / cx / cy,
png_depth_scale; crop_edge and distortion are accepted and unused, as in the reference); `default_config` holds the
values of R/configs/data/{replica,TUM/*,scannet,replica_v2}.yaml.  ScanNet++ has no YAML: its camera is read from the
sequence's dslr/nerfstudio/transforms_undistorted.json.

ScanNet++ and ReplicaV2 also have a held-out test split (``split="test"``) for novel-view evaluation: its frames
follow the first train frame, which becomes frame 0, so every test pose is relative to it.  CUDA only for the
pixels: there is no CPU fallback."""
import collections
import concurrent.futures
import glob
import json
import numbers
import os
import re
import time
import warnings

import numpy as np
import torch

from . import _lib
from .rasterizer import GaussianRasterizationSettings

DATASETS = ("replica", "tum", "scannet", "scannetpp", "replicav2")
SPLITS = ("train", "test")
_SPLIT_DATASETS = ("scannetpp", "replicav2")         # the datasets that have a held-out test split


def _camera_params(h, w, fx, fy, cx, cy, png_depth_scale, **extra):
    return dict(image_height=h, image_width=w, fx=fx, fy=fy, cx=cx, cy=cy, png_depth_scale=png_depth_scale, **extra)


# R/configs/data/replica.yaml, scannet.yaml, replica_v2.yaml and TUM/*.yaml (the TUM cameras differ per Freiburg
# sensor); ReplicaV2's depth PNGs are in millimetres, Replica's in 1/6553.5 m
_CONFIGS = {
    "replica": _camera_params(680, 1200, 600.0, 600.0, 599.5, 339.5, 6553.5, crop_edge=0),
    "replicav2": _camera_params(680, 1200, 600.0, 600.0, 599.5, 339.5, 1000.0, crop_edge=0),
    "scannet": _camera_params(968, 1296, 1169.621094, 1167.105103, 646.295044, 489.927032, 1000.0),
    "freiburg1": _camera_params(480, 640, 517.3, 516.5, 318.6, 255.3, 5000.0, crop_edge=8),
    "freiburg2": _camera_params(480, 640, 520.9, 521.0, 325.1, 249.7, 5000.0, crop_edge=8),
    "freiburg3": _camera_params(480, 640, 535.4, 539.2, 320.1, 247.6, 5000.0, crop_edge=8),
}


def default_config(dataset, sequence=""):
    """The reference's shipped data config for `dataset` ("replica", "tum", "scannet", "replicav2"); for TUM the
    camera of the Freiburg sensor named in `sequence` (freiburg1 when none is named).  ScanNet++ has none: its camera
    comes with each sequence (`scannetpp_config`)."""
    if dataset not in DATASETS:
        raise ValueError("unknown dataset %r (expected one of %s)" % (dataset, ", ".join(DATASETS)))
    if dataset == "scannetpp":
        raise ValueError("scannetpp has no shipped data config: its camera is read from each sequence "
                         "(scannetpp_config)")
    key = dataset
    if dataset == "tum":
        m = re.search(r"freiburg([123])", sequence)
        key = "freiburg" + (m.group(1) if m else "1")
    return dict(dataset_name=dataset, camera_params=dict(_CONFIGS[key]))


def load_config(path):
    """A dataset config from a YAML file of the reference's shape."""
    import yaml
    with open(path) as f:
        cfg = yaml.safe_load(f)
    missing = [k for k in ("image_height", "image_width", "fx", "fy", "cx", "cy", "png_depth_scale")
               if k not in cfg.get("camera_params", {})]
    if missing:
        raise ValueError("%s: camera_params lacks %s" % (path, ", ".join(missing)))
    return cfg


def natural_key(s):
    """Sort key that orders digit runs by value ("frame2" before "frame10"), as natsort.natsorted does."""
    return [int(t) if t.isdigit() else t for t in re.split(r"(\d+)", s)]


def natsorted(paths):
    return sorted(paths, key=natural_key)


# ---- file discovery and poses (host only) -------------------------------------------------------------------------

def _pose_lines(path, n):
    """The first `n` c2w rows of a file with one row-major 4x4 matrix per line, as float32 [4,4] tensors."""
    with open(path) as f:
        lines = f.readlines()
    if len(lines) < n:
        raise ValueError("%s: %d poses for %d images" % (path, len(lines), n))
    return [torch.from_numpy(np.array([float(v) for v in lines[i].split()]).reshape(4, 4)).float() for i in range(n)]


def _replica_files(root):
    colors = natsorted(glob.glob(os.path.join(root, "results", "frame*.jpg")))
    depths = natsorted(glob.glob(os.path.join(root, "results", "depth*.png")))
    return colors, depths, _pose_lines(os.path.join(root, "traj.txt"), len(colors))


def _read_list(path, skiprows=0):
    with warnings.catch_warnings():               # numpy notes that '#' comment lines are not counted as rows
        warnings.simplefilter("ignore", UserWarning)
        return np.loadtxt(path, delimiter=" ", dtype=str, skiprows=skiprows, ndmin=2)


def tum_associate(t_image, t_depth, t_pose, max_dt=0.08, frame_rate=32):
    """TUM frame selection (R/datasets/gradslam_datasets/tum.py:50-106): each colour timestamp is paired with the
    nearest depth and pose timestamps and kept when both lie within `max_dt`; of those pairs a frame is kept only when
    it is more than 1 / frame_rate seconds after the previously kept one.  Returns the kept (image, depth, pose) rows."""
    pairs = []
    for i, t in enumerate(t_image):
        j = int(np.argmin(np.abs(t_depth - t)))
        k = int(np.argmin(np.abs(t_pose - t)))
        if abs(t_depth[j] - t) < max_dt and abs(t_pose[k] - t) < max_dt:
            pairs.append((i, j, k))
    kept = [0]
    for n in range(1, len(pairs)):
        if t_image[pairs[n][0]] - t_image[pairs[kept[-1]][0]] > 1.0 / frame_rate:
            kept.append(n)
    return [pairs[n] for n in kept] if pairs else []


def _tum_files(root):
    from scipy.spatial.transform import Rotation
    pose_file = os.path.join(root, "groundtruth.txt")
    if not os.path.isfile(pose_file):
        pose_file = os.path.join(root, "pose.txt")
    images, depths = _read_list(os.path.join(root, "rgb.txt")), _read_list(os.path.join(root, "depth.txt"))
    pose_rows = _read_list(pose_file, skiprows=1)     # the reference skips the first line of the pose file
    vecs = pose_rows[:, 1:].astype(np.float64)
    rows = tum_associate(images[:, 0].astype(np.float64), depths[:, 0].astype(np.float64),
                         pose_rows[:, 0].astype(np.float64))
    colors, depth_paths, poses = [], [], []
    for i, j, k in rows:
        colors.append(os.path.join(root, images[i, 1]))
        depth_paths.append(os.path.join(root, depths[j, 1]))
        c2w = np.eye(4)                               # tx ty tz qx qy qz qw -> c2w
        c2w[:3, :3] = Rotation.from_quat(vecs[k][3:]).as_matrix()
        c2w[:3, 3] = vecs[k][:3]
        poses.append(torch.from_numpy(c2w).float())
    return colors, depth_paths, poses


def _scannet_files(root):
    colors = natsorted(glob.glob(os.path.join(root, "color", "*.jpg")))
    depths = natsorted(glob.glob(os.path.join(root, "depth", "*.png")))
    # float64 as np.loadtxt reads them; -inf poses (ScanNet's invalid frames) are kept, as the reference keeps them
    poses = [torch.from_numpy(np.loadtxt(p)) for p in natsorted(glob.glob(os.path.join(root, "pose", "*.txt")))]
    return colors, depths, poses


def _read_json(path):
    if not os.path.isfile(path):
        raise FileNotFoundError("%s: no such file" % path)
    with open(path) as f:
        return json.load(f)


def _scannetpp_meta(root):
    return _read_json(os.path.join(root, "dslr", "nerfstudio", "transforms_undistorted.json"))


def scannetpp_config(root):
    """The config of the ScanNet++ sequence at `root`, as ScannetPPDataset builds it: the undistorted DSLR camera of
    dslr/nerfstudio/transforms_undistorted.json (fl_x, fl_y, cx, cy, w, h) and depth PNGs in millimetres."""
    meta = _scannetpp_meta(root)
    return dict(dataset_name="scannetpp", camera_params=_camera_params(
        meta["h"], meta["w"], meta["fl_x"], meta["fl_y"], meta["cx"], meta["cy"], 1000.0))


def _scannetpp_files(root, split, ignore_bad):
    """R/datasets/gradslam_datasets/scannetpp.py: the split's image names in the order of dslr/train_test_lists.json,
    looked up by file_path in `frames` (train) or `test_frames` (test); the test split starts with the first train
    frame; with `ignore_bad`, the split's own frames whose metadata has is_bad set are dropped.  Poses are
    P @ c2w @ P^T with P = diag(1, -1, -1, 1) (OpenGL -> OpenCV camera axes), in float32."""
    lists = _read_json(os.path.join(root, "dslr", "train_test_lists.json"))
    meta = _scannetpp_meta(root)
    P = torch.tensor([[1, 0, 0, 0], [0, -1, 0, 0], [0, 0, -1, 0], [0, 0, 0, 1]]).float()

    def lookup(frames, key, name):
        index = {fr["file_path"]: i for i, fr in enumerate(frames)}
        if name not in index:
            raise ValueError("%s: image %r of the %s list is not in transforms_undistorted.json's %r"
                             % (root, name, "train" if key == "frames" else "test", key))
        return frames[index[name]]

    def entry(name, fr):
        c2w = torch.from_numpy(np.array(fr["transform_matrix"])).float()
        return (os.path.join(root, "dslr", "undistorted_images", name),
                os.path.join(root, "dslr", "undistorted_depths", name.replace(".JPG", ".png")), P @ c2w @ P.T)

    key = "frames" if split == "train" else "test_frames"
    rows = []
    if split == "test":                               # never dropped, even when it is bad
        first = lists["train"][0]
        rows.append(entry(first, lookup(meta["frames"], "frames", first)))
    for name in lists[split]:
        fr = lookup(meta[key], key, name)
        if ignore_bad and fr["is_bad"]:
            continue
        rows.append(entry(name, fr))
    return [r[0] for r in rows], [r[1] for r in rows], [r[2] for r in rows]


def _replicav2_files(root, split):
    """R/datasets/gradslam_datasets/replica.py (ReplicaV2Dataset): train = imap/00, test = imap/01 after imap/00's
    first frame; rgb/rgb_*.png and depth/depth_*.png in natural order, poses from traj_w_c.txt, one per image."""
    train = os.path.join(root, "imap", "00")
    folder = train if split == "train" else os.path.join(root, "imap", "01")
    colors = natsorted(glob.glob(os.path.join(folder, "rgb", "rgb_*.png")))
    depths = natsorted(glob.glob(os.path.join(folder, "depth", "depth_*.png")))
    poses = _pose_lines(os.path.join(folder, "traj_w_c.txt"), len(colors))
    if split == "test":
        colors = [os.path.join(train, "rgb", "rgb_0.png")] + colors
        depths = [os.path.join(train, "depth", "depth_0.png")] + depths
        poses = _pose_lines(os.path.join(train, "traj_w_c.txt"), 1) + poses
    return colors, depths, poses


_FILES = {"replica": _replica_files, "tum": _tum_files, "scannet": _scannet_files}


def relative_poses(poses):
    """Every pose relative to the first: inv(P0) @ P_t with a general inverse (the reference's relative_transformation
    with orthogonal_rotations=False), composed as [R0' R_t | R0' t_t + t0'] in the poses' own dtype."""
    inv0 = torch.inverse(poses[0].unsqueeze(0).repeat(poses.shape[0], 1, 1))
    out = torch.zeros_like(inv0)
    out[..., :3, 0:3] += torch.matmul(inv0[..., :3, :3], poses[..., :3, :3])
    out[..., :3, -1:] += torch.matmul(inv0[..., :3, :3], poses[..., :3, -1:]) + inv0[..., :3, -1:]
    out[..., -1, -1:] += 1.0
    return out


def scaled_intrinsics(cam, height, width):
    """4x4 float32 intrinsics of the native camera scaled by desired / native per axis (datautils.scale_intrinsics)."""
    K = torch.from_numpy(np.array([[cam["fx"], 0.0, cam["cx"]], [0.0, cam["fy"], cam["cy"]], [0.0, 0.0, 1.0]]))
    K = K.to(torch.float).clone()
    h_ratio, w_ratio = float(height) / cam["image_height"], float(width) / cam["image_width"]
    K[0, 0] *= w_ratio
    K[1, 1] *= h_ratio
    K[0, 2] *= w_ratio
    K[1, 2] *= h_ratio
    out = torch.eye(4).to(K)
    out[:3, :3] = K
    return out


class SequenceFiles:
    """What a sequence is before any pixel is read: colour and depth paths, relative float32 c2w poses [N,4,4], the
    retained indices into the discovered (for TUM: associated) frames, the native camera (`camera_params`) and the
    scaled 4x4 intrinsics.

    start / end / stride select frames as the reference does: end = -1 means all, otherwise end > start.  `split`:
    "train", or for ScanNet++ and ReplicaV2 "test" (the first train frame, then the held-out views; start / end /
    stride apply to that combined list).  `ignore_bad` (ScanNet++ only) drops the frames its metadata marks is_bad."""

    def __init__(self, dataset, basedir, sequence, config=None, start=0, end=-1, stride=1, desired_height=None,
                 desired_width=None, split="train", ignore_bad=False):
        if dataset not in DATASETS:
            raise ValueError("unknown dataset %r (expected one of %s)" % (dataset, ", ".join(DATASETS)))
        if split not in SPLITS:
            raise ValueError("split must be one of %s, got %r" % (", ".join(SPLITS), split))
        if split != "train" and dataset not in _SPLIT_DATASETS:
            raise ValueError("%s has no %r split (only %s have a test split)" % (dataset, split,
                                                                                 " and ".join(_SPLIT_DATASETS)))
        if ignore_bad and dataset != "scannetpp":
            raise ValueError("ignore_bad applies to scannetpp only")
        self.root = os.path.join(basedir, sequence)
        if not os.path.isdir(self.root):
            raise FileNotFoundError("%s: no such sequence directory" % self.root)
        if config is None:
            config = scannetpp_config(self.root) if dataset == "scannetpp" else default_config(dataset, sequence)
        cam = config["camera_params"]
        if start < 0:
            raise ValueError("start must be >= 0, got %d" % start)
        if not (end == -1 or end > start):
            raise ValueError("end (%d) must be -1 (all frames) or greater than start (%d)" % (end, start))
        if stride < 1:
            raise ValueError("stride must be >= 1, got %d" % stride)
        self.dataset, self.split = dataset, split
        self.camera_params = dict(cam)
        self.height = int(cam["image_height"] if desired_height is None else desired_height)
        self.width = int(cam["image_width"] if desired_width is None else desired_width)
        self.png_depth_scale = float(cam["png_depth_scale"])
        if dataset == "scannetpp":
            colors, depths, poses = _scannetpp_files(self.root, split, ignore_bad)
        elif dataset == "replicav2":
            colors, depths, poses = _replicav2_files(self.root, split)
        else:
            colors, depths, poses = _FILES[dataset](self.root)
        if len(colors) != len(depths):
            raise ValueError("%s: %d colour and %d depth images" % (self.root, len(colors), len(depths)))
        if not colors:
            raise ValueError("%s: no frames found" % self.root)
        n = len(colors)
        end = n if end == -1 else end
        self.color_paths, self.depth_paths = colors[start:end:stride], depths[start:end:stride]
        self.retained_inds = torch.arange(n)[start:end:stride]
        raw = torch.stack(poses[start:end:stride])
        self.poses = relative_poses(raw).float()
        self.intrinsics = scaled_intrinsics(cam, self.height, self.width)

    def __len__(self):
        return len(self.color_paths)


# ---- decoding and the ingest kernel --------------------------------------------------------------------------------

def decode_color(path):
    """uint8 [h, w, 3] RGB as Pillow decodes it."""
    from PIL import Image
    with Image.open(path) as im:
        a = np.array(im)                              # writable: torch.from_numpy shares it without a warning
    if a.dtype != np.uint8 or a.ndim != 3 or a.shape[2] != 3:
        raise ValueError("%s: expected 8-bit 3-channel RGB colour, got %s %s" % (path, a.dtype, a.shape))
    return a


def decode_depth(path):
    """uint16 [h, w] raw depth as Pillow decodes a 16-bit PNG."""
    from PIL import Image
    with Image.open(path) as im:
        a = np.array(im)
    if a.ndim != 2 or a.dtype.kind not in "ui" or (a.size and (a.min() < 0 or a.max() > 65535)):
        raise ValueError("%s: expected single-channel 16-bit depth, got %s %s" % (path, a.dtype, a.shape))
    return a.astype(np.uint16, copy=False)


def ingest_rgbd(rgb, depth, height, width, png_depth_scale, color_out=None, depth_out=None):
    """One `sb_ingest_rgbd` launch on the current stream: rgb uint8 [h, w, 3] and depth uint16 [hd, wd] CUDA tensors
    -> (colour float32 [3, height, width] in [0, 1], depth float32 [1, height, width] in metres), exactly as the
    reference's loader and splatam.py compute them in float64 (see csrc/ingest.cu)."""
    _lib.need_cuda("ingest_rgbd", rgb, depth)
    if rgb.dtype != torch.uint8 or rgb.dim() != 3 or rgb.shape[2] != 3 or not rgb.is_contiguous():
        raise _lib.SplatamB200Error("ingest_rgbd expects contiguous uint8 [h, w, 3] colour, got %s %s"
                                    % (rgb.dtype, tuple(rgb.shape)))
    if depth.dtype != torch.uint16 or depth.dim() != 2 or not depth.is_contiguous():
        raise _lib.SplatamB200Error("ingest_rgbd expects contiguous uint16 [h, w] depth, got %s %s"
                                    % (depth.dtype, tuple(depth.shape)))
    dev = rgb.device
    if color_out is None:
        color_out = torch.empty(3, height, width, dtype=torch.float32, device=dev)
    if depth_out is None:
        depth_out = torch.empty(1, height, width, dtype=torch.float32, device=dev)
    _lib.call("sb_ingest_rgbd", rgb, rgb.shape[0], rgb.shape[1], depth, depth.shape[0], depth.shape[1], height, width,
              float(png_depth_scale), color_out, depth_out, device=dev)
    return color_out, depth_out


def setup_camera(w, h, K, w2c, device, near=0.01, far=100.0):
    """Raster settings of one view as R/utils/recon_helpers.py:setup_camera builds them (float32, w2c transposed,
    full projection = w2c^T @ opengl_proj^T)."""
    fx, fy, cx, cy = K[0][0], K[1][1], K[0][2], K[1][2]
    w2c = torch.tensor(w2c).to(device).float()
    cam_center = torch.inverse(w2c)[:3, 3]
    w2c = w2c.unsqueeze(0).transpose(1, 2)
    proj = torch.tensor([[2 * fx / w, 0.0, -(w - 2 * cx) / w, 0.0],
                         [0.0, 2 * fy / h, -(h - 2 * cy) / h, 0.0],
                         [0.0, 0.0, far / (far - near), -(far * near) / (far - near)],
                         [0.0, 0.0, 1.0, 0.0]]).to(device).float().unsqueeze(0).transpose(1, 2)
    return GaussianRasterizationSettings(image_height=h, image_width=w, tanfovx=w / (2 * fx), tanfovy=h / (2 * fy),
                                         bg=torch.tensor([0, 0, 0], dtype=torch.float32, device=device),
                                         scale_modifier=1.0, viewmatrix=w2c, projmatrix=w2c.bmm(proj), sh_degree=0,
                                         campos=cam_center, prefiltered=False)


class _Slot:
    """One pinned staging pair and the event recorded after its last host-to-device copy."""

    def __init__(self):
        self.rgb = self.depth = None
        self.copied = None

    def arrays(self, rgb_shape, depth_shape):
        if self.copied is not None:
            self.copied.synchronize()                 # refilled only once its previous upload has completed
        if self.rgb is None or tuple(self.rgb.shape) != rgb_shape:
            self.rgb = torch.empty(rgb_shape, dtype=torch.uint8, pin_memory=True)
        if self.depth is None or tuple(self.depth.shape) != depth_shape:
            self.depth = torch.empty(depth_shape, dtype=torch.uint16, pin_memory=True)
        return self.rgb, self.depth


class RGBDSequence:
    """A sequence on disk as a list of frame dicts: ``len(seq)``, ``seq[t]`` and slices (which return lists).

    ``seq[t]`` is dict(id=t, cam, w2c, im [3,H,W], depth [1,H,W], intrinsics [3,3], gt_w2c [4,4]) on `device`:
    `cam` and `w2c` belong to the first frame (w2c = inv(pose_0), as SplaTAM's initialize_first_timestep computes it),
    `gt_w2c` = inv(pose_t) of the relative pose (SplaTAM's gt_w2c; on a test split, the held-out view's pose),
    `intrinsics` the scaled 3x3 camera matrix.
    Colour and depth are fresh tensors per frame (keyframes keep them); the last `cache` frames are remembered, so
    repeated `seq[t]` returns the same tensors.

    densify_height / densify_width (both or neither): the densification resolution of SplaTAM-S
    (R/scripts/splatam.py:498-507,781-794).  When it differs from the desired size, every frame dict also carries
    ``densify`` = dict(id, cam, w2c, im [3,h,w], depth [1,h,w], intrinsics [3,3]) at that size: `intrinsics` scaled
    to it (`densify_intrinsics`), `cam` = `densify_cam` (that size, the first frame's w2c), and the pixels from a
    second ingest launch on the same uploaded frame, so each file is decoded and uploaded once.  `run_slam` grows the
    map from it.  At the desired size, or when not given, there is no ``densify`` entry and both attributes are None.

    prefetch = k > 0: while frame t is consumed, a host thread decodes frames t+1 .. t+k into a ring of k pinned
    staging slots and enqueues their upload and the ingest kernel(s) on a side stream; `seq[t]` makes the caller's
    current stream wait on frame t's event and blocks the host only while frame t is still being decoded.
    prefetch = 0 reads synchronously on the current stream.  `load_wait_s` accumulates the host time spent in
    `seq[t]` for frames that were not cached (the load time the caller sees)."""

    def __init__(self, dataset, basedir, sequence, config=None, start=0, end=-1, stride=1, desired_height=None,
                 desired_width=None, device="cuda", prefetch=2, cache=4, split="train", ignore_bad=False,
                 densify_height=None, densify_width=None):
        if (densify_height is None) != (densify_width is None):
            raise ValueError("give both densify_height and densify_width or neither, got %r and %r"
                             % (densify_height, densify_width))
        for name, v in (("densify_height", densify_height), ("densify_width", densify_width)):
            if v is not None and (isinstance(v, bool) or not isinstance(v, numbers.Integral) or v <= 0):
                raise ValueError("%s must be a positive integer, got %r" % (name, v))
        self.files = SequenceFiles(dataset, basedir, sequence, config, start, end, stride, desired_height,
                                   desired_width, split=split, ignore_bad=ignore_bad)
        self.device = torch.device(device)
        if self.device.type == "cuda" and self.device.index is None:
            self.device = torch.device("cuda", torch.cuda.current_device())
        self.height, self.width = self.files.height, self.files.width
        self.intrinsics = self.files.intrinsics[:3, :3].to(self.device)
        self.w2c = torch.linalg.inv(self.files.poses[0].to(self.device))
        self.cam = setup_camera(self.width, self.height, self.intrinsics.cpu().numpy(), self.w2c.cpu().numpy(),
                                self.device)
        self.densify_height = self.densify_width = self.densify_intrinsics = self.densify_cam = None
        if densify_height is not None and (int(densify_height), int(densify_width)) != (self.height, self.width):
            self.densify_height, self.densify_width = int(densify_height), int(densify_width)
            K_d = scaled_intrinsics(self.files.camera_params, self.densify_height, self.densify_width)
            self.densify_intrinsics = K_d[:3, :3].to(self.device)
            self.densify_cam = setup_camera(self.densify_width, self.densify_height,
                                            self.densify_intrinsics.cpu().numpy(), self.w2c.cpu().numpy(), self.device)
        self.prefetch = int(prefetch)
        self._cache = collections.OrderedDict()
        self._cache_size = max(int(cache), 1)
        self._pending = {}
        self.load_wait_s = 0.0
        self._pool = None
        if self.prefetch > 0:
            self._pool = concurrent.futures.ThreadPoolExecutor(max_workers=1, thread_name_prefix="rgbd-prefetch")
            self._side = torch.cuda.Stream(self.device)
            self._slots = [_Slot() for _ in range(self.prefetch)]
            self._submitted = 0

    def __len__(self):
        return len(self.files)

    def _gt_w2c(self, t):
        """inv(pose_t) on the device; all NaN where the pose is not finite (ScanNet's invalid -inf poses), which the
        evaluation's ATE skips as the reference's does."""
        pose = self.files.poses[t]
        if not bool(torch.isfinite(pose).all()):
            return torch.full((4, 4), float("nan"), device=self.device)
        return torch.linalg.inv(pose.to(self.device))

    @property
    def gt_w2c(self):
        """SplaTAM's gt_w2c_all_frames: `_gt_w2c` of every frame."""
        return [self._gt_w2c(t) for t in range(len(self))]

    def _decode(self, t):
        return decode_color(self.files.color_paths[t]), decode_depth(self.files.depth_paths[t])

    def _ingest(self, rgb, depth):
        """The ingest launch(es) on the current stream for one uploaded frame: (colour, depth) at the desired size and
        the (colour, depth) pair at the densification size, or None when there is none."""
        scale = self.files.png_depth_scale
        color, depth_out = ingest_rgbd(rgb, depth, self.height, self.width, scale)
        dens = None
        if self.densify_height is not None:
            dens = ingest_rgbd(rgb, depth, self.densify_height, self.densify_width, scale)
        return color, depth_out, dens

    def _load_sync(self, t):
        rgb, depth = self._decode(t)
        return self._ingest(torch.from_numpy(rgb).to(self.device), torch.from_numpy(depth).to(self.device)) + (None,)

    def _load_async(self, t, slot):
        """Worker thread: decode into the slot's pinned arrays, then enqueue upload + ingest on the side stream."""
        rgb, depth = self._decode(t)
        pr, pd = slot.arrays(rgb.shape, depth.shape)
        pr.numpy()[...] = rgb
        pd.numpy()[...] = depth
        with torch.cuda.device(self.device), torch.cuda.stream(self._side):
            dr = pr.to(self.device, non_blocking=True)
            dd = pd.to(self.device, non_blocking=True)
            slot.copied = torch.cuda.Event()
            slot.copied.record(self._side)
            out = self._ingest(dr, dd)
            ready = torch.cuda.Event()
            ready.record(self._side)
        return out + (ready,)

    def _submit(self, t):
        if t in self._pending or t in self._cache or not 0 <= t < len(self):
            return
        slot = self._slots[self._submitted % len(self._slots)]
        self._submitted += 1
        self._pending[t] = self._pool.submit(self._load_async, t, slot)

    def _frame(self, t):
        t0 = time.perf_counter()
        if self._pool is None:
            color, depth, dens, _ = self._load_sync(t)
        else:
            self._submit(t)
            for j in range(t + 1, t + 1 + self.prefetch):
                self._submit(j)
            fut = self._pending.pop(t)
            for j in [j for j in self._pending if j < t or j > t + self.prefetch]:
                self._pending.pop(j)                  # stale look-ahead after a jump: its results are dropped
            color, depth, dens, ready = fut.result()
            consumer = torch.cuda.current_stream(self.device)
            consumer.wait_event(ready)
            for x in (color, depth) + (dens or ()):
                x.record_stream(consumer)             # allocated on the side stream, used and freed on the consumer's
        self.load_wait_s += time.perf_counter() - t0
        fr = dict(id=t, cam=self.cam, w2c=self.w2c, im=color, depth=depth, intrinsics=self.intrinsics,
                  gt_w2c=self._gt_w2c(t))
        if dens is not None:
            fr["densify"] = dict(id=t, cam=self.densify_cam, w2c=self.w2c, im=dens[0], depth=dens[1],
                                 intrinsics=self.densify_intrinsics)
        return fr

    def __getitem__(self, t):
        if isinstance(t, slice):
            return [self[i] for i in range(*t.indices(len(self)))]
        t = int(t)
        if t < 0:
            t += len(self)
        if not 0 <= t < len(self):
            raise IndexError("frame %d out of range for a sequence of %d" % (t, len(self)))
        if t in self._cache:
            self._cache.move_to_end(t)
            return self._cache[t]
        fr = self._frame(t)
        self._cache[t] = fr
        while len(self._cache) > self._cache_size:
            self._cache.popitem(last=False)
        return fr

    def close(self):
        """Waits for the look-ahead in flight and stops the prefetch thread."""
        if self._pool is not None:
            self._pool.shutdown(wait=True)
            self._pool = None
            self._pending.clear()

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
