"""Generates tests/golden/datasets/ref_datasets.npz by reading tiny synthetic sequences with the reference's UNMODIFIED
dataset classes (R/datasets/gradslam_datasets: ReplicaDataset, TUMDataset, ScannetDataset, imported from the install
that oracle/reference.py writes, as refsrc.py imports the reference) on the CPU, then applying splatam.py's
``permute(2, 0, 1) / 255`` to the colour.

Stand-ins for what this image lacks, bound only while the reference is imported and run:
* imageio.imread is Pillow, ``np.asarray(Image.open(path))`` (Pillow is imageio's backend for JPEG and PNG);
* natsort.natsorted is a natural sort (digit runs compared by value);
* kornia.geometry.linalg.compose_transformations is kornia's composition restated ([R1 R2 | R1 t2 + t1] added into a
  zero matrix whose corner is 1); inverse_transformation is never called (orthogonal_rotations=False);
* np.unicode_, which NumPy 2 removed and tum.py's parse_list names, is np.str_.
cv2 is the real OpenCV.

`write_sequences(dst, npz)` writes the stored files back; the tests call it.  Every input file is stored as its exact
bytes, so the tests never depend on a JPEG or PNG encoder.  The sequences come from one seeded generator:
* replica  (64x48, 12 frames named frame0 .. frame11, so lexical and natural order differ), read at native size and
  at 40x30, 100x70 and the exact-2x 32x24, with start 1, end 11, stride 5 (the full read keeps only file names and
  poses);
* tum      (32x24 PNG colour, timestamps where some colour frames find no depth or pose within 0.08 s and some follow
  the previous kept frame by less than 1/32 s), read at 40x30 with start 1, stride 2;
* scannet  (130x97 colour, 64x48 depth, one pose of -inf), read at 64x48 with start 2, stride 3.
Stored per read: colour [N,3,H,W] and depth [N,1,H,W] float32, the 4x4 intrinsics, the relative poses [N,4,4]
float32, the retained indices and the colour / depth file names.
Run:  python tests/golden/datasets/make_golden_datasets.py   (needs the reference installed by oracle/reference.py)
"""
import contextlib
import io
import os
import re
import sys
import tempfile
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(os.path.dirname(HERE)))

# name: (dataset, config camera_params, sequence, reader kwargs)
CONFIGS = {
    "replica": dict(image_height=48, image_width=64, fx=50.0, fy=52.0, cx=31.5, cy=23.5, png_depth_scale=6553.5,
                    crop_edge=0),
    "tum": dict(image_height=24, image_width=32, fx=25.85, fy=25.83, cx=15.93, cy=12.77, png_depth_scale=5000.0,
                crop_edge=8),
    "scannet": dict(image_height=97, image_width=130, fx=116.96, fy=116.71, cx=64.63, cy=48.99, png_depth_scale=1000.0),
}
SEQUENCES = {"replica": "room0", "tum": "rgbd_dataset_freiburg1_desk", "scannet": "scene0000_00"}
READS = {
    "replica_all": ("replica", dict(desired_height=48, desired_width=64)),
    "replica_native": ("replica", dict(desired_height=48, desired_width=64, start=1, end=11, stride=5)),
    "replica_down": ("replica", dict(desired_height=30, desired_width=40, start=1, end=11, stride=5)),
    "replica_up": ("replica", dict(desired_height=70, desired_width=100, start=1, end=11, stride=5)),
    "replica_half": ("replica", dict(desired_height=24, desired_width=32, start=1, end=11, stride=5)),
    "tum_up": ("tum", dict(desired_height=30, desired_width=40, start=1, stride=2)),
    "scannet_mixed": ("scannet", dict(desired_height=48, desired_width=64, start=2, stride=3)),
}


def config(dataset):
    return dict(dataset_name=dataset, camera_params=dict(CONFIGS[dataset]))


def _png16(a):
    from PIL import Image
    buf = io.BytesIO()
    Image.fromarray(a.astype(np.uint16)).save(buf, format="PNG")
    return buf.getvalue()


def _image(a, fmt):
    from PIL import Image
    buf = io.BytesIO()
    Image.fromarray(a).save(buf, format=fmt, **({"quality": 90} if fmt == "JPEG" else {}))
    return buf.getvalue()


def _rgb(g, h, w, t):
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float64)
    base = 127.5 + 100 * np.sin(xx[..., None] / (5.0 + t) + yy[..., None] / 7.0 + np.array([0.0, 2.0, 4.0]))
    return np.clip(base + g.normal(0, 3, (h, w, 3)), 0, 255).astype(np.uint8)


def _depth(g, h, w, scale):
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float64)
    d = (1.5 + 0.5 * np.sin(xx / 9.0 + g.random()) * np.cos(yy / 7.0)) * scale
    d[g.random((h, w)) < 0.03] = 0                    # holes
    return np.minimum(d, 65535).astype(np.uint16)


def _c2w(g, t):
    q = g.normal(0, 1, 4) * 0.1 + np.array([0.0, 0.0, 0.0, 1.0])
    x, y, z, w = q / np.linalg.norm(q)
    m = np.eye(4)
    m[:3, :3] = [[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
                 [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
                 [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]]
    m[:3, 3] = g.normal(0, 0.5, 3) + 0.05 * t
    return m


def make_files(seed=2026):
    """{relative path: bytes} of the three synthetic sequences."""
    g = np.random.default_rng(seed)
    files = {}
    # Replica: results/frame<i>.jpg, results/depth<i>.png, traj.txt (one c2w per line, row-major)
    root = "replica/" + SEQUENCES["replica"] + "/"
    traj = []
    for t in range(12):
        files[root + "results/frame%d.jpg" % t] = _image(_rgb(g, 48, 64, t), "JPEG")
        files[root + "results/depth%d.png" % t] = _png16(_depth(g, 48, 64, 6553.5))
        traj.append(" ".join("%.17g" % v for v in _c2w(g, t).reshape(-1)))
    files[root + "traj.txt"] = ("\n".join(traj) + "\n").encode()
    # TUM: rgb.txt / depth.txt / groundtruth.txt with '#' headers; colour frames at ~30 Hz, some too close together,
    # depth missing around frames 4 and 9, poses at 100 Hz with a gap around frame 13
    root = "tum/" + SEQUENCES["tum"] + "/"
    t_img = 1305031102.0 + np.cumsum([0.0] + [0.02 if k in (3, 7, 8) else 0.0333 for k in range(17)])
    t_img += g.uniform(-0.002, 0.002, t_img.size)
    rgb_lines = ["# color images", "# file: 'rgbd_dataset_freiburg1_desk.bag'", "# timestamp filename"]
    depth_lines = ["# depth maps", "# file: 'rgbd_dataset_freiburg1_desk.bag'", "# timestamp filename"]
    for i, ts in enumerate(t_img):
        name = "rgb/%.6f.png" % ts
        files[root + name] = _image(_rgb(g, 24, 32, i), "PNG")
        rgb_lines.append("%.6f %s" % (ts, name))
        if i in (4, 9):
            continue
        td = ts + g.uniform(-0.015, 0.015)
        dname = "depth/%.6f.png" % td
        files[root + dname] = _png16(_depth(g, 24, 32, 5000.0))
        depth_lines.append("%.6f %s" % (td, dname))
    gt_lines = ["# ground truth trajectory", "# file: 'rgbd_dataset_freiburg1_desk.bag'", "# timestamp tx ty tz qx qy qz qw"]
    for tp in np.arange(t_img[0] - 0.05, t_img[-1] + 0.05, 0.01):
        if abs(tp - t_img[13]) < 0.1:
            continue
        q = g.normal(0, 1, 4) * 0.2 + np.array([0.0, 0.0, 0.0, 1.0])
        q = q / np.linalg.norm(q) * 1.0001                  # not exactly unit: the reader normalises
        tr = g.normal(0, 0.5, 3)
        gt_lines.append("%.4f %.4f %.4f %.4f %.4f %.4f %.4f %.4f" % ((tp,) + tuple(tr) + tuple(q)))
    files[root + "rgb.txt"] = ("\n".join(rgb_lines) + "\n").encode()
    files[root + "depth.txt"] = ("\n".join(depth_lines) + "\n").encode()
    files[root + "groundtruth.txt"] = ("\n".join(gt_lines) + "\n").encode()
    # ScanNet: color/<i>.jpg (130x97), depth/<i>.png (64x48), pose/<i>.txt; frame 5's pose is -inf
    root = "scannet/" + SEQUENCES["scannet"] + "/"
    for t in range(11):
        files[root + "color/%d.jpg" % t] = _image(_rgb(g, 97, 130, t), "JPEG")
        files[root + "depth/%d.png" % t] = _png16(_depth(g, 48, 64, 1000.0))
        pose = np.full((4, 4), -np.inf) if t == 5 else _c2w(g, t)
        files[root + "pose/%d.txt" % t] = ("\n".join(" ".join("%.9f" % v for v in row) for row in pose) + "\n").encode()
    return files


def write_sequences(dst, npz):
    """Writes the sequences stored in `npz` (the fixture) under dst/<dataset>/<sequence>."""
    for name, blob in zip(npz["file_names"], npz["file_blobs_offsets"].reshape(-1, 2)):
        path = os.path.join(dst, str(name))
        os.makedirs(os.path.dirname(path), exist_ok=True)
        with open(path, "wb") as f:
            f.write(npz["file_blobs"][blob[0]:blob[1]].tobytes())


def _natural_key(s):
    return [int(t) if t.isdigit() else t for t in re.split(r"(\d+)", s)]


def _compose_transformations(trans_01, trans_12):
    import torch
    out = torch.zeros_like(trans_01)
    out[..., :3, 0:3] += torch.matmul(trans_01[..., :3, :3], trans_12[..., :3, :3])
    out[..., :3, -1:] += torch.matmul(trans_01[..., :3, :3], trans_12[..., :3, -1:]) + trans_01[..., :3, -1:]
    out[..., -1, -1:] += 1.0
    return out


@contextlib.contextmanager
def reference_datasets():
    """The reference's gradslam_datasets package with the stand-ins above."""
    from PIL import Image
    src = os.path.join(ROOT, "oracle", "_ref", "SplaTAM")
    if not os.path.isdir(os.path.join(src, "datasets", "gradslam_datasets")):
        raise RuntimeError("the reference is not installed under oracle/_ref (run oracle/reference.py)")
    imread = lambda p, *a, **k: np.asarray(Image.open(p))
    mods = {"imageio": types.ModuleType("imageio"), "imageio.v2": types.ModuleType("imageio.v2"),
            "natsort": types.ModuleType("natsort"), "kornia": types.ModuleType("kornia"),
            "kornia.geometry": types.ModuleType("kornia.geometry"),
            "kornia.geometry.linalg": types.ModuleType("kornia.geometry.linalg")}
    mods["imageio"].imread = mods["imageio.v2"].imread = imread
    mods["imageio"].v2 = mods["imageio.v2"]
    mods["natsort"].natsorted = lambda seq: sorted(seq, key=_natural_key)
    mods["kornia.geometry.linalg"].compose_transformations = _compose_transformations
    mods["kornia.geometry.linalg"].inverse_transformation = None
    pkg = types.ModuleType("datasets")
    pkg.__path__ = [os.path.join(src, "datasets")]
    mods["datasets"] = pkg
    saved = {k: sys.modules.get(k) for k in list(mods) + ["datasets.gradslam_datasets"]}
    sys.modules.update(mods)
    np.unicode_ = np.str_
    try:
        import importlib
        yield importlib.import_module("datasets.gradslam_datasets")
    finally:
        del np.unicode_
        for k in [k for k in sys.modules if k == "datasets" or k.startswith("datasets.")] + list(mods):
            sys.modules.pop(k, None)
        for k, v in saved.items():
            if v is not None:
                sys.modules[k] = v


def run_reference(G, root, read):
    import torch
    dataset, kw = READS[read]
    cls = {"replica": G.ReplicaDataset, "tum": G.TUMDataset, "scannet": G.ScannetDataset}[dataset]
    ds = cls(config(dataset), os.path.join(root, dataset), SEQUENCES[dataset], device="cpu", **kw)
    colors, depths, poses, K = [], [], [], None
    for t in range(len(ds)):
        color, depth, intrinsics, pose = ds[t]
        colors.append((color.permute(2, 0, 1) / 255).numpy())          # splatam.py:649-650
        depths.append(depth.permute(2, 0, 1).numpy())
        poses.append(pose.numpy())
        K = intrinsics.numpy()
    assert colors[0].dtype == np.float32 and depths[0].dtype == np.float32
    return {"color": np.stack(colors), "depth": np.stack(depths), "intrinsics": K, "poses": np.stack(poses),
            "retained": ds.retained_inds.numpy().astype(np.int64),
            "color_names": np.array([os.path.relpath(p, os.path.join(root, dataset, SEQUENCES[dataset]))
                                     for p in ds.color_paths]),
            "depth_names": np.array([os.path.relpath(p, os.path.join(root, dataset, SEQUENCES[dataset]))
                                     for p in ds.depth_paths])}


def main():
    files = make_files()
    names = sorted(files)
    blobs = [np.frombuffer(files[n], np.uint8) for n in names]
    ends = np.cumsum([b.size for b in blobs])
    out = {"file_names": np.array(names), "file_blobs": np.concatenate(blobs),
           "file_blobs_offsets": np.stack([ends - [b.size for b in blobs], ends], 1).astype(np.int64)}
    with tempfile.TemporaryDirectory() as d, reference_datasets() as G:
        write_sequences(d, out)
        for read in READS:
            for k, v in run_reference(G, d, read).items():
                if read != "replica_all" or k not in ("color", "depth"):
                    out[read + "_" + k] = v
    path = os.path.join(HERE, "ref_datasets.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, "%d arrays, %.1f KB" % (len(out), os.path.getsize(path) / 1024))
    for read in READS:
        print(read, out[read + "_poses"].shape, "retained", out[read + "_retained"].tolist())


if __name__ == "__main__":
    main()
