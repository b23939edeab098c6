"""Generates tests/golden/datasets/ref_nvs_datasets.npz by reading tiny synthetic ScanNet++ and ReplicaV2 sequences with
the reference's UNMODIFIED dataset classes (R/datasets/gradslam_datasets: ScannetPPDataset, ReplicaV2Dataset), with the
stand-ins and file helpers of make_golden_datasets.py, and applying splatam.py's ``permute(2, 0, 1) / 255`` to the
colour.

Every input file is stored as its exact bytes (`write_sequences` of make_golden_datasets.py writes them back).  The
sequences come from one seeded generator:
* scannetpp (dslr/undistorted_images/*.JPG colour and dslr/undistorted_depths/*.png depth at 64x48;
  dslr/nerfstudio/transforms_undistorted.json with `frames` and `test_frames` listed in an order that differs from
  dslr/train_test_lists.json; one is_bad frame in each split, the train one being the first train frame, which the
  test split prepends and never drops), read for both splits with ignore_bad off and on, at the exact-2x 32x24 and at
  40x30;
* replicav2 (imap/00 with 12 train frames, imap/01 with 11 test frames, so natural and lexical order differ;
  rgb/rgb_<i>.png, depth/depth_<i>.png and a traj_w_c.txt with more lines than images), read for the train split,
  the whole test split and the test split with start 1, end 10, stride 2 at 40x30.
Stored per read: colour [N,3,H,W] and depth [N,1,H,W] float32, the 4x4 intrinsics, the relative poses [N,4,4]
float32, the retained indices and the colour / depth file names relative to the sequence directory.
Run:  python tests/golden/datasets/make_golden_nvs_datasets.py   (needs the reference installed by oracle/reference.py)
"""
import importlib.util
import json
import os
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))


def _base():
    spec = importlib.util.spec_from_file_location("make_golden_datasets", os.path.join(HERE, "make_golden_datasets.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


B = _base()
write_sequences = B.write_sequences

SEQUENCES = {"scannetpp": "8b5caf3398", "replicav2": "room_0"}
REPLICAV2_CONFIG = dict(dataset_name="replicav2", camera_params=dict(
    image_height=48, image_width=64, fx=50.0, fy=52.0, cx=31.5, cy=23.5, png_depth_scale=1000.0, crop_edge=0))
# name: (dataset, split, reader kwargs)
READS = {
    "scannetpp_train": ("scannetpp", "train", dict(desired_height=24, desired_width=32)),
    "scannetpp_train_bad": ("scannetpp", "train", dict(desired_height=30, desired_width=40, ignore_bad=True)),
    "scannetpp_test": ("scannetpp", "test", dict(desired_height=24, desired_width=32)),
    "scannetpp_test_bad": ("scannetpp", "test", dict(desired_height=30, desired_width=40, ignore_bad=True)),
    "replicav2_train": ("replicav2", "train", dict(desired_height=48, desired_width=64)),
    "replicav2_test": ("replicav2", "test", dict(desired_height=48, desired_width=64)),
    "replicav2_test_sel": ("replicav2", "test", dict(desired_height=30, desired_width=40, start=1, end=10, stride=2)),
}
SCANNETPP_TRAIN = ["DSC%05d.JPG" % i for i in (4, 1, 7, 2, 9, 5)]
SCANNETPP_TEST = ["DSC%05d.JPG" % i for i in (8, 3, 6)]
SCANNETPP_BAD = {"DSC00004.JPG", "DSC00006.JPG"}           # the first train frame and one test frame


def make_files(seed=2027):
    """{relative path: bytes} of the two synthetic sequences."""
    g = np.random.default_rng(seed)
    files = {}
    root = "scannetpp/" + SEQUENCES["scannetpp"] + "/dslr/"
    frames = {}
    for t, name in enumerate(sorted(SCANNETPP_TRAIN + SCANNETPP_TEST)):
        files[root + "undistorted_images/" + name] = B._image(B._rgb(g, 48, 64, t), "JPEG")
        files[root + "undistorted_depths/" + name.replace(".JPG", ".png")] = B._png16(B._depth(g, 48, 64, 1000.0))
        frames[name] = dict(file_path=name, transform_matrix=B._c2w(g, t).tolist(), is_bad=name in SCANNETPP_BAD)
    meta = dict(fl_x=50.25, fl_y=51.5, cx=31.75, cy=23.25, w=64, h=48, camera_model="PINHOLE",
                frames=[frames[n] for n in sorted(SCANNETPP_TRAIN, reverse=True)],
                test_frames=[frames[n] for n in sorted(SCANNETPP_TEST)])
    files[root + "nerfstudio/transforms_undistorted.json"] = json.dumps(meta, indent=1).encode()
    files[root + "train_test_lists.json"] = json.dumps(dict(train=SCANNETPP_TRAIN, test=SCANNETPP_TEST)).encode()
    root = "replicav2/" + SEQUENCES["replicav2"] + "/imap/"
    for split, n in (("00", 12), ("01", 11)):
        traj = []
        for t in range(n):
            files[root + split + "/rgb/rgb_%d.png" % t] = B._image(B._rgb(g, 48, 64, t), "PNG")
            files[root + split + "/depth/depth_%d.png" % t] = B._png16(B._depth(g, 48, 64, 1000.0))
        for t in range(n + 2):                         # two poses more than images
            traj.append(" ".join("%.17g" % v for v in B._c2w(g, t).reshape(-1)))
        files[root + split + "/traj_w_c.txt"] = ("\n".join(traj) + "\n").encode()
    return files


def run_reference(G, root, read):
    dataset, split, kw = READS[read]
    kw = dict(kw, use_train_split=split == "train", device="cpu")
    base = os.path.join(root, dataset)
    if dataset == "scannetpp":
        ds = G.ScannetPPDataset(base, SEQUENCES[dataset], **kw)
    else:
        ds = G.ReplicaV2Dataset(REPLICAV2_CONFIG, base, SEQUENCES[dataset], **kw)
    colors, depths, poses, K = [], [], [], None
    for t in range(len(ds)):
        color, depth, intrinsics, pose = ds[t]
        colors.append((color.permute(2, 0, 1) / 255).numpy())          # splatam.py:649-650
        depths.append(depth.permute(2, 0, 1).numpy())
        poses.append(pose.numpy())
        K = intrinsics.numpy()
    assert colors[0].dtype == np.float32 and depths[0].dtype == np.float32
    seq = os.path.join(base, SEQUENCES[dataset])
    return {"color": np.stack(colors), "depth": np.stack(depths), "intrinsics": K, "poses": np.stack(poses),
            "retained": ds.retained_inds.numpy().astype(np.int64),
            "color_names": np.array([os.path.relpath(p, seq) for p in ds.color_paths]),
            "depth_names": np.array([os.path.relpath(p, seq) for p in ds.depth_paths])}


def main():
    files = make_files()
    names = sorted(files)
    blobs = [np.frombuffer(files[n], np.uint8) for n in names]
    ends = np.cumsum([b.size for b in blobs])
    out = {"file_names": np.array(names), "file_blobs": np.concatenate(blobs),
           "file_blobs_offsets": np.stack([ends - [b.size for b in blobs], ends], 1).astype(np.int64)}
    with tempfile.TemporaryDirectory() as d, B.reference_datasets() as G:
        write_sequences(d, out)
        for read in READS:
            for k, v in run_reference(G, d, read).items():
                out[read + "_" + k] = v
    path = os.path.join(HERE, "ref_nvs_datasets.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, "%d arrays, %.1f KB" % (len(out), os.path.getsize(path) / 1024))
    for read in READS:
        print(read, out[read + "_poses"].shape, "retained", out[read + "_retained"].tolist(),
              out[read + "_color_names"].tolist())


if __name__ == "__main__":
    main()
