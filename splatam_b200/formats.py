"""Data formats either side of the hot path (SURVEY.md section 8(f) row N4): SplaTAM's `params.npz` checkpoints
and the 3DGS-viewer PLY export, byte-compatible with what the reference writes.

* ``save_params`` / ``save_params_ckpt`` / ``load_params``   R/utils/common_utils.py:25-52 (np.savez of every entry of
  the params dict, tensors as contiguous CPU numpy arrays, non-tensors stored as they are)
* ``save_checkpoint`` / ``load_checkpoint``                  R/scripts/splatam.py:604-643,927-931 (`params{t}.npz` and
  `keyframe_time_indices{t}.npy`, plus a `run_state{t}.npz` sidecar that only this project reads)
* ``save_run_record``                                        R/scripts/splatam.py:973-986 (the final `params.npz` with
  the reference's 14 keys)
* ``read_record`` / ``check_camera_columns`` / ``record_tensors``   the one checked reader of a run record (this
  project's or the reference's `params.npz`, the 13-key offline record, a checkpoint's `params{t}.npz`)
* ``save_ply`` / ``load_ply`` / ``export_ply``               R/scripts/export_ply.py:20-77 (binary little-endian PLY,
  one `vertex` element of 17 float32 properties; the reference writes it through the `plyfile` package, which is
  not a dependency here: the header and the packed records are produced directly)
* ``save_mesh_ply`` / ``load_mesh_ply``                      a coloured triangle mesh (splatam_b200/mesh.py) as a
  binary little-endian PLY that MeshLab and Blender open; ``load_mesh_ply`` also reads the ground-truth meshes of the
  datasets (ASCII or binary, extra properties, same-count polygons)
* ``save_nav_map`` / ``load_nav_map``                        a navigation map (splatam_b200/navmap.py): labels, ESDF
  and grid in one npz, read back through a checked reader
"""
import os

import numpy as np

GAUSSIAN_KEYS = ("means3D", "rgb_colors", "unnorm_rotations", "logit_opacities", "log_scales")
CHECKPOINT_KEYS = GAUSSIAN_KEYS + ("cam_unnorm_rots", "cam_trans")
# the keys save_params writes at the end of the reference's run, in its order (splatam.py:973-983)
RECORD_KEYS = CHECKPOINT_KEYS + ("timestep", "intrinsics", "w2c", "org_width", "org_height", "gt_w2c_all_frames",
                                 "keyframe_time_indices")
# the record keys the reference's loaders leave out of the Gaussian parameters; a checkpoint holds none of them
CAMERA_KEYS = ("intrinsics", "w2c", "org_width", "org_height")

C0 = 0.28209479177387814            # SH band-0 constant (export_ply.py:9)

PLY_ATTRS = ("x", "y", "z", "nx", "ny", "nz", "f_dc_0", "f_dc_1", "f_dc_2", "opacity",
             "scale_0", "scale_1", "scale_2", "rot_0", "rot_1", "rot_2", "rot_3")


def params2cpu(params):
    out = {}
    for k, v in params.items():
        if hasattr(v, "detach"):                                  # torch.Tensor / Parameter
            out[k] = np.ascontiguousarray(v.detach().cpu().numpy())
        else:
            out[k] = v
    return out


def save_params(output_params, output_dir, name="params.npz"):
    """np.savez(<output_dir>/params.npz, **params) -- the file R/scripts/export_ply.py, the viewers and
    post_splatam_opt.py load."""
    os.makedirs(output_dir, exist_ok=True)
    path = os.path.join(output_dir, name)
    np.savez(path, **params2cpu(output_params))
    return path


def save_params_ckpt(output_params, output_dir, time_idx):
    return save_params(output_params, output_dir, name="params" + str(time_idx) + ".npz")


def load_params(path, device=None):
    """dict of numpy arrays (device=None) or torch tensors on `device`; scalar / object entries (e.g. the stored
    intrinsics, `org_width`) are returned as numpy, like dict(np.load(path, allow_pickle=True))."""
    raw = dict(np.load(path, allow_pickle=True))
    if device is None:
        return raw
    floats = [k for k, v in raw.items() if isinstance(v, np.ndarray) and v.dtype.kind == "f"]
    return dict(raw, **record_tensors(raw, floats, device))


def record_tensors(rec, keys, device):
    """{k: rec[k] as a contiguous float32 tensor on `device`} for each of `keys`."""
    import torch
    return {k: torch.from_numpy(np.ascontiguousarray(rec[k], dtype=np.float32)).to(device) for k in keys}


def read_record(path, need, camera=None):
    """The entries of a run record on the host, as dict(np.load(path, allow_pickle=True)) gives them, with `camera`
    (dict(intrinsics=, w2c=, org_width=, org_height=), any subset) applied over them.  ValueError when a key of `need`
    is missing; when `need` holds cam_unnorm_rots and cam_trans, unless they are [1,4,T] and [1,3,T] with one T >= 1;
    and when a Gaussian tensor or `timestep` has another row count than means3D."""
    with np.load(path, allow_pickle=True) as z:
        rec = dict(z)
    rec.update(camera or {})
    missing = [k for k in need if k not in rec]
    if missing:
        hint = " (a checkpoint holds no camera: pass camera=dict(intrinsics=, w2c=, org_width=, org_height=))" \
            if set(missing) <= set(CAMERA_KEYS) else ""
        raise ValueError("%s lacks %s%s" % (path, ", ".join(missing), hint))
    if {"cam_unnorm_rots", "cam_trans"} <= set(need):
        rots, trans = np.shape(rec["cam_unnorm_rots"]), np.shape(rec["cam_trans"])
        if len(rots) != 3 or rots[:2] != (1, 4) or len(trans) != 3 or trans[:2] != (1, 3) or rots[-1] != trans[-1] \
                or rots[-1] < 1:
            raise ValueError("camera count mismatch: cam_unnorm_rots %s and cam_trans %s must be [1,4,T] and [1,3,T] "
                             "with one T >= 1" % (rots, trans))
    if "means3D" in rec:
        P = np.shape(rec["means3D"])[0]
        for k in GAUSSIAN_KEYS + ("timestep",):
            if k in rec and np.shape(rec[k])[0] != P:
                raise ValueError("%s has %d rows for %d Gaussians" % (k, np.shape(rec[k])[0], P))
    return rec


def check_camera_columns(path, rec, indices):
    """ValueError naming the first of the frame `indices` outside [0, T), T the camera count of the record `rec`."""
    T = np.shape(rec["cam_unnorm_rots"])[-1]
    bad = [k for k in indices if not 0 <= k < T]
    if bad:
        raise ValueError("%s has %d camera columns; frame index %d has none" % (path, T, bad[0]))


def _ckpt_paths(directory, time_idx):
    t = str(int(time_idx))
    return (os.path.join(directory, "params" + t + ".npz"), os.path.join(directory, "keyframe_time_indices" + t + ".npy"),
            os.path.join(directory, "run_state" + t + ".npz"))


def save_checkpoint(directory, time_idx, params, keyframe_time_indices, run_state=None):
    """The reference's checkpoint of frame `time_idx` (splatam.py:927-931): `params{t}.npz` with exactly the seven
    CHECKPOINT_KEYS -- the reference turns every key of that file into an optimised parameter (splatam.py:609-610), so
    nothing else may go in it -- and `keyframe_time_indices{t}.npy` (int64, as np.array of a list of ints gives it).
    `run_state`: dict of numpy arrays written to `run_state{t}.npz`, the sidecar an exact continuation needs
    (see slam.run_slam).  Returns the paths written."""
    os.makedirs(directory, exist_ok=True)
    p_path, k_path, s_path = _ckpt_paths(directory, time_idx)
    np.savez(p_path, **params2cpu({k: params[k] for k in CHECKPOINT_KEYS}))
    np.save(k_path, np.array([int(i) for i in keyframe_time_indices], dtype=np.int64))
    written = [p_path, k_path]
    if run_state is not None:
        np.savez(s_path, **run_state)
        written.append(s_path)
    return written


def load_checkpoint(directory, time_idx, device):
    """Reads the checkpoint of frame `time_idx` -> dict(time_idx, gauss = the five Gaussian tensors, cam_unnorm_rots,
    cam_trans (float32 tensors on `device`), keyframe_time_indices (list of int), state = the `run_state{t}.npz`
    sidecar as a dict of numpy arrays, or None when there is none, e.g. for a checkpoint the reference wrote).  A
    missing `params{t}.npz` or `keyframe_time_indices{t}.npy` raises FileNotFoundError naming the path."""
    p_path, k_path, s_path = _ckpt_paths(directory, time_idx)
    for path in (p_path, k_path):
        if not os.path.isfile(path):
            raise FileNotFoundError("checkpoint file not found: %s" % path)
    with np.load(p_path) as z:
        missing = [k for k in CHECKPOINT_KEYS if k not in z.files]
        if missing:
            raise ValueError("%s lacks %s" % (p_path, ", ".join(missing)))
        t = record_tensors(z, CHECKPOINT_KEYS, device)
    state = None
    if os.path.isfile(s_path):
        with np.load(s_path) as z:
            state = {k: z[k] for k in z.files}
    return dict(time_idx=int(time_idx), gauss={k: t[k] for k in GAUSSIAN_KEYS},
                cam_unnorm_rots=t["cam_unnorm_rots"], cam_trans=t["cam_trans"],
                keyframe_time_indices=[int(i) for i in np.load(k_path).reshape(-1).tolist()], state=state)


def save_run_record(out_dir, gauss, rots, trans, timestep, intrinsics, first_w2c, width, height, gt_w2c,
                    keyframe_time_indices):
    """`<out_dir>/params.npz` as the reference writes it after a run (splatam.py:973-986), with its 14 RECORD_KEYS:
    the five Gaussian tensors, cam_unnorm_rots / cam_trans, `timestep` [P], `intrinsics` [3,3], `w2c` (the first
    frame's) [4,4], all float32; `org_width` / `org_height` as 0-d int64; `gt_w2c_all_frames` [T,4,4] float32 (NaN where
    the pose is invalid); `keyframe_time_indices` int64.  `gt_w2c`: a [T,4,4] tensor / array or a list of [4,4].
    keyframe_time_indices=None writes the 13 keys without it, as the offline drivers save their record
    (R/scripts/post_splatam_opt.py:372-383).  Returns the path."""
    f32 = lambda a: np.ascontiguousarray(np.asarray(a.detach().cpu().numpy() if hasattr(a, "detach") else a,
                                                    dtype=np.float32))
    rec = {k: f32(gauss[k]) for k in GAUSSIAN_KEYS}
    rec.update(cam_unnorm_rots=f32(rots), cam_trans=f32(trans), timestep=f32(timestep).reshape(-1),
               intrinsics=f32(intrinsics)[:3, :3], w2c=f32(first_w2c).reshape(4, 4),
               org_width=np.array(int(width), dtype=np.int64), org_height=np.array(int(height), dtype=np.int64),
               gt_w2c_all_frames=(np.stack([f32(m).reshape(4, 4) for m in gt_w2c]) if len(gt_w2c)
                                  else np.zeros((0, 4, 4), np.float32)))
    if keyframe_time_indices is not None:
        rec["keyframe_time_indices"] = np.array([int(i) for i in keyframe_time_indices], dtype=np.int64)
    if rec["timestep"].shape[0] != rec["means3D"].shape[0]:
        raise ValueError("timestep has %d entries for %d Gaussians" % (rec["timestep"].shape[0],
                                                                     rec["means3D"].shape[0]))
    os.makedirs(out_dir, exist_ok=True)
    path = os.path.join(out_dir, "params.npz")
    np.savez(path, **{k: rec[k] for k in RECORD_KEYS if k in rec})
    return path


def save_exposure(out_dir, cam_exposure):
    """`<out_dir>/exposure.npz` with one key, `cam_exposure` float32 [1,6,T]: a run's per-frame colour corrections
    (slam.run_slam's `exposure`).  Kept out of params.npz, whose readers take every key they do not know for a
    per-Gaussian tensor or an optimised parameter.  Returns the path."""
    a = np.ascontiguousarray(np.asarray(_host(cam_exposure), dtype=np.float32))
    if a.ndim != 3 or a.shape[:2] != (1, 6):
        raise ValueError("cam_exposure must be [1,6,T], got %s" % (a.shape,))
    os.makedirs(out_dir, exist_ok=True)
    path = os.path.join(out_dir, "exposure.npz")
    np.savez(path, cam_exposure=a)
    return path


def save_dynamic(out_dir, stats, keyframe_ids, keyframe_masks):
    """`<out_dir>/dynamic.npz` of a run with motion masks (slam.run_slam's `dynamic`): per tracked frame `frame`
    (int64), `scale`, `dynamic_frac` and `inconsistent_frac` (float32), from the result's `dynamic` list; the
    keyframes' ids `keyframe_ids` (int64 [K]) and their masks as `keyframe_masks` (np.packbits of the bool [K,H,W]
    stack) with `keyframe_masks_shape`.  Kept out of params.npz, as exposure.npz is.  Returns the path."""
    m = np.stack([np.asarray(_host(x), dtype=bool) for x in keyframe_masks])
    if m.ndim != 3 or m.shape[0] != len(keyframe_ids):
        raise ValueError("%d keyframe ids for keyframe masks of shape %s" % (len(keyframe_ids), m.shape))
    os.makedirs(out_dir, exist_ok=True)
    path = os.path.join(out_dir, "dynamic.npz")
    np.savez(path, frame=np.array([r["frame"] for r in stats], dtype=np.int64),
             scale=np.array([r["scale"] for r in stats], dtype=np.float32),
             dynamic_frac=np.array([r["dynamic_frac"] for r in stats], dtype=np.float32),
             inconsistent_frac=np.array([r["inconsistent_frac"] for r in stats], dtype=np.float32),
             keyframe_ids=np.asarray(keyframe_ids, dtype=np.int64), keyframe_masks=np.packbits(m.reshape(-1)),
             keyframe_masks_shape=np.array(m.shape, dtype=np.int64))
    return path


def load_dynamic(path):
    """The record of `save_dynamic`: dict(frame, scale, dynamic_frac, inconsistent_frac, keyframe_ids, keyframe_masks
    bool [K,H,W]) of numpy arrays.  ValueError when a key is missing or the shapes disagree."""
    keys = ("frame", "scale", "dynamic_frac", "inconsistent_frac", "keyframe_ids", "keyframe_masks",
            "keyframe_masks_shape")
    with np.load(path) as z:
        missing = [k for k in keys if k not in z.files]
        if missing:
            raise ValueError("%s lacks %s" % (path, missing))
        d = {k: np.asarray(z[k]) for k in keys}
    shape = tuple(int(x) for x in d.pop("keyframe_masks_shape").reshape(-1))
    n = int(np.prod(shape)) if len(shape) == 3 else -1
    if n < 0 or shape[0] != d["keyframe_ids"].shape[0] or d["keyframe_masks"].size * 8 < n:
        raise ValueError("%s: keyframe masks of shape %s for %d keyframes" % (path, shape, d["keyframe_ids"].shape[0]))
    if not d["frame"].shape == d["scale"].shape == d["dynamic_frac"].shape == d["inconsistent_frac"].shape:
        raise ValueError("%s: per-frame arrays of different lengths" % path)
    d["keyframe_masks"] = np.unpackbits(d["keyframe_masks"].astype(np.uint8))[:n].reshape(shape).astype(bool)
    return d


def load_exposure(path, num_frames=None, device=None):
    """The `cam_exposure` [1,6,T] of an exposure.npz (`save_exposure`): numpy, or a float32 tensor on `device`.
    ValueError when the key is missing, the shape is not [1,6,T] or T differs from `num_frames`."""
    with np.load(path) as z:
        if "cam_exposure" not in z.files:
            raise ValueError("%s lacks cam_exposure" % path)
        a = np.asarray(z["cam_exposure"], dtype=np.float32)
    if a.ndim != 3 or a.shape[:2] != (1, 6) or (num_frames is not None and a.shape[2] != num_frames):
        raise ValueError("%s: cam_exposure has shape %s, expected (1, 6, %s)"
                         % (path, a.shape, "T" if num_frames is None else num_frames))
    if device is None:
        return a
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).to(device)


NAV_MAP_KEYS = ("labels", "esdf", "origin", "voxel_size", "trunc", "min_weight", "occ_dist", "unknown_is_obstacle")


def save_nav_map(path, labels, esdf, origin, voxel_size, trunc, min_weight, occ_dist, unknown_is_obstacle):
    """A navigation map (splatam_b200/navmap.py) as one npz: `labels` uint8 and `esdf` float32, both [nz,ny,nx];
    `origin` float32 [3]; `voxel_size`, `trunc`, `min_weight` and `occ_dist` as 0-d float32; `unknown_is_obstacle`
    as 0-d bool.  Returns the path."""
    lab = np.ascontiguousarray(np.asarray(_host(labels), dtype=np.uint8))
    e = np.ascontiguousarray(np.asarray(_host(esdf), dtype=np.float32))
    d = os.path.dirname(os.path.abspath(path))
    os.makedirs(d, exist_ok=True)
    f32 = lambda x: np.array(x, dtype=np.float32)
    with open(path, "wb") as f:
        np.savez(f, labels=lab, esdf=e, origin=f32(origin).reshape(3), voxel_size=f32(voxel_size), trunc=f32(trunc),
                 min_weight=f32(min_weight), occ_dist=f32(occ_dist),
                 unknown_is_obstacle=np.array(bool(unknown_is_obstacle)))
    return path


def load_nav_map(path):
    """The record of `save_nav_map` as a dict of numpy arrays (the scalars as 0-d arrays).  ValueError naming the key
    when a key is missing, has another dtype or shape, a label is above 2, the origin is not finite, the voxel size
    or trunc is not finite and positive, or min_weight or occ_dist is not finite."""
    want = dict(labels=np.uint8, esdf=np.float32, origin=np.float32, voxel_size=np.float32, trunc=np.float32,
                min_weight=np.float32, occ_dist=np.float32, unknown_is_obstacle=np.bool_)
    with np.load(path) as z:
        missing = [k for k in NAV_MAP_KEYS if k not in z.files]
        if missing:
            raise ValueError("%s lacks %s" % (path, ", ".join(missing)))
        d = {k: np.asarray(z[k]) for k in NAV_MAP_KEYS}
    for k, t in want.items():
        if d[k].dtype != t:
            raise ValueError("%s: %s has dtype %s, expected %s" % (path, k, d[k].dtype, np.dtype(t)))
    if d["labels"].ndim != 3 or min(d["labels"].shape) < 1:
        raise ValueError("%s: labels has shape %s, expected [nz,ny,nx]" % (path, d["labels"].shape))
    if d["esdf"].shape != d["labels"].shape:
        raise ValueError("%s: esdf has shape %s, labels %s" % (path, d["esdf"].shape, d["labels"].shape))
    if d["origin"].shape != (3,):
        raise ValueError("%s: origin has shape %s, expected (3,)" % (path, d["origin"].shape))
    for k in ("voxel_size", "trunc", "min_weight", "occ_dist", "unknown_is_obstacle"):
        if d[k].shape != ():
            raise ValueError("%s: %s has shape %s, expected a scalar" % (path, k, d[k].shape))
    if d["labels"].size and int(d["labels"].max()) > 2:
        raise ValueError("%s: labels holds %d, above 2 (occupied)" % (path, int(d["labels"].max())))
    if not np.all(np.isfinite(d["origin"])):
        raise ValueError("%s: origin %s is not finite" % (path, d["origin"]))
    for k in ("voxel_size", "trunc"):
        if not (np.isfinite(d[k]) and d[k] > 0):
            raise ValueError("%s: %s %r must be finite and positive" % (path, k, float(d[k])))
    for k in ("min_weight", "occ_dist"):
        if not np.isfinite(d[k]):
            raise ValueError("%s: %s %r must be finite" % (path, k, float(d[k])))
    return d


def rgb_to_spherical_harmonic(rgb):
    return (rgb - 0.5) / C0


def spherical_harmonic_to_rgb(sh):
    return sh * C0 + 0.5


def _ply_header(n):
    lines = ["ply", "format binary_little_endian 1.0", f"element vertex {n}"]
    lines += [f"property float {a}" for a in PLY_ATTRS]
    lines += ["end_header", ""]
    return "\n".join(lines).encode("ascii")


def save_ply(path, means, scales, rotations, rgbs, opacities, normals=None):
    """Arguments as R/scripts/export_ply.py:20 -- the RAW stored parameters: `scales` are log-scales [N,1] or [N,3],
    `rotations` the unnormalised quaternions, `opacities` the logits [N,1]; colours are converted to SH band 0."""
    means = np.asarray(means, dtype=np.float32)
    n = means.shape[0]
    normals = np.zeros_like(means) if normals is None else np.asarray(normals, dtype=np.float32)
    colors = rgb_to_spherical_harmonic(np.asarray(rgbs, dtype=np.float32))
    scales = np.asarray(scales, dtype=np.float32)
    if scales.shape[1] == 1:
        scales = np.tile(scales, (1, 3))
    table = np.concatenate((means, normals, colors, np.asarray(opacities, dtype=np.float32).reshape(n, 1), scales,
                            np.asarray(rotations, dtype=np.float32)), axis=1).astype("<f4")
    assert table.shape == (n, len(PLY_ATTRS))
    with open(path, "wb") as f:
        f.write(_ply_header(n))
        f.write(np.ascontiguousarray(table).tobytes())
    return path


def load_ply(path):
    """Inverse of save_ply for files with exactly the 17 float properties (any order of header whitespace)."""
    with open(path, "rb") as f:
        blob = f.read()
    end = blob.index(b"end_header\n") + len(b"end_header\n")
    header = blob[:end].decode("ascii").split("\n")
    assert header[0] == "ply" and header[1].startswith("format binary_little_endian")
    n = int([h for h in header if h.startswith("element vertex")][0].split()[-1])
    props = [h.split()[-1] for h in header if h.startswith("property")]
    assert all(h.split()[1] == "float" for h in header if h.startswith("property"))
    table = np.frombuffer(blob, dtype="<f4", count=n * len(props), offset=end).reshape(n, len(props))
    col = {p: table[:, i] for i, p in enumerate(props)}
    pick = lambda names: np.stack([col[a] for a in names], axis=1)
    return dict(means3D=pick(("x", "y", "z")), normals=pick(("nx", "ny", "nz")),
                rgb_colors=spherical_harmonic_to_rgb(pick(("f_dc_0", "f_dc_1", "f_dc_2"))),
                logit_opacities=pick(("opacity",)), log_scales=pick(("scale_0", "scale_1", "scale_2")),
                unnorm_rotations=pick(("rot_0", "rot_1", "rot_2", "rot_3")))


def export_ply(params_path, ply_path=None):
    """params.npz -> splat.ply beside it (the __main__ of R/scripts/export_ply.py:55-77)."""
    p = dict(np.load(params_path, allow_pickle=True))
    ply_path = ply_path or os.path.join(os.path.dirname(params_path), "splat.ply")
    return save_ply(ply_path, p["means3D"], p["log_scales"], p["unnorm_rotations"], p["rgb_colors"], p["logit_opacities"])


MESH_VERTEX_DTYPE = np.dtype([("x", "<f4"), ("y", "<f4"), ("z", "<f4"), ("red", "u1"), ("green", "u1"),
                              ("blue", "u1")])
MESH_FACE_DTYPE = np.dtype([("n", "u1"), ("v", "<i4", (3,))])


def _mesh_ply_header(nv, nf):
    lines = ["ply", "format binary_little_endian 1.0", f"element vertex {nv}", "property float x", "property float y",
             "property float z", "property uchar red", "property uchar green", "property uchar blue",
             f"element face {nf}", "property list uchar int vertex_indices", "end_header", ""]
    return "\n".join(lines).encode("ascii")


def _host(a):
    return a.detach().cpu().numpy() if hasattr(a, "detach") else np.asarray(a)


def save_mesh_ply(path, vertices, colors, faces):
    """Writes vertices [V,3] (float32), colors [V,3] in [0, 1] and faces [F,3] (vertex indices) as a binary
    little-endian PLY: `element vertex V` with float x, y, z and uchar red, green, blue, `element face F` with
    `property list uchar int vertex_indices`.  Colours become rint(clip(c, 0, 1) * 255), NaN -> 0.  Accepts numpy
    arrays or tensors on any device.  Returns the path."""
    v = np.asarray(_host(vertices), np.float32).reshape(-1, 3)
    c = np.nan_to_num(np.asarray(_host(colors), np.float64).reshape(-1, 3), nan=0.0)
    f = np.asarray(_host(faces)).reshape(-1, 3)
    if c.shape[0] != v.shape[0]:
        raise ValueError("%d colours for %d vertices" % (c.shape[0], v.shape[0]))
    if f.size and (f.min() < 0 or f.max() >= v.shape[0]):
        raise ValueError("face indices must lie in [0, %d)" % v.shape[0])
    vert = np.empty(v.shape[0], MESH_VERTEX_DTYPE)
    vert["x"], vert["y"], vert["z"] = v[:, 0], v[:, 1], v[:, 2]
    u8 = np.rint(np.clip(c, 0.0, 1.0) * 255).astype(np.uint8)
    vert["red"], vert["green"], vert["blue"] = u8[:, 0], u8[:, 1], u8[:, 2]
    face = np.empty(f.shape[0], MESH_FACE_DTYPE)
    face["n"] = 3
    face["v"] = f.astype(np.int32)
    with open(path, "wb") as out:
        out.write(_mesh_ply_header(v.shape[0], f.shape[0]))
        out.write(vert.tobytes())
        out.write(face.tobytes())
    return path


_PLY_TYPES = {"char": "i1", "int8": "i1", "uchar": "u1", "uint8": "u1", "short": "i2", "int16": "i2",
              "ushort": "u2", "uint16": "u2", "int": "i4", "int32": "i4", "uint": "u4", "uint32": "u4",
              "float": "f4", "float32": "f4", "double": "f8", "float64": "f8"}


def _parse_ply_header(path, blob):
    """(format, [(element name, count, [(property, dtype) or (property, count dtype, index dtype)])], data offset)."""
    end = blob.find(b"end_header")
    nl = blob.find(b"\n", end)
    if not blob.startswith(b"ply") or end < 0 or nl < 0:
        raise ValueError("%s is not a PLY file" % path)
    fmt, elements = None, []
    for line in blob[:end].decode("ascii", "replace").splitlines()[1:]:
        t = line.split()
        if not t or t[0] in ("comment", "obj_info"):
            continue
        if t[0] == "format":
            fmt = t[1] if len(t) > 1 else None
        elif t[0] == "element" and len(t) == 3:
            elements.append((t[1], int(t[2]), []))
        elif t[0] == "property" and elements and len(t) == 3 and t[1] in _PLY_TYPES:
            elements[-1][2].append((t[2], _PLY_TYPES[t[1]]))
        elif (t[0] == "property" and elements and len(t) == 5 and t[1] == "list" and t[2] in _PLY_TYPES
              and t[3] in _PLY_TYPES):
            elements[-1][2].append((t[4], _PLY_TYPES[t[2]], _PLY_TYPES[t[3]]))
        else:
            raise ValueError("%s: unsupported PLY header line %r" % (path, line))
    if fmt == "binary_big_endian":
        raise ValueError("%s is a big-endian PLY, which is not supported" % path)
    if fmt not in ("binary_little_endian", "ascii"):
        raise ValueError("%s: unsupported PLY format %r" % (path, fmt))
    return fmt, elements, nl + 1


def _face_layout(path, props):
    """(index of the vertex list among the face properties, count dtype, index dtype)."""
    lists = [k for k, p in enumerate(props) if len(p) == 3]
    if len(lists) != 1 or props[lists[0]][0] not in ("vertex_indices", "vertex_index"):
        raise ValueError("%s: the face element needs one list property vertex_indices or vertex_index" % path)
    k = lists[0]
    if np.dtype(props[k][1]).kind not in "ui" or np.dtype(props[k][2]).kind not in "ui":
        raise ValueError("%s: the face list must have integer counts and indices" % path)
    return k, props[k][1], props[k][2]


def _read_binary(path, blob, offset, elements):
    """{element name: structured array}; faces are read with one dtype for the count of their first face."""
    out = {}
    for name, count, props in elements:
        if any(len(p) == 3 for p in props):
            if name != "face":
                raise ValueError("%s: list properties are supported on the face element only" % path)
            k, ct, it = _face_layout(path, props)
            n = 0
            if count:
                head = np.dtype([(p[0], "<" + p[1]) for p in props[:k]])
                n = int(np.frombuffer(blob, "<" + ct, count=1, offset=offset + head.itemsize)[0])
            fields = [(p[0], "<" + p[1]) if len(p) == 2 else ("n", "<" + ct) for p in props]
            fields[k] = ("n", "<" + ct)
            fields.insert(k + 1, ("v", "<" + it, (n,)))
            dt = np.dtype(fields)
        else:
            dt = np.dtype([(p[0], "<" + p[1]) for p in props])
        if offset + count * dt.itemsize > len(blob):
            raise ValueError("%s is truncated in its %s element%s" % (
                path, name, " or mixes polygons of different vertex counts" if name == "face" else ""))
        out[name] = np.frombuffer(blob, dt, count=count, offset=offset)
        if name == "face" and count and not np.all(out[name]["n"] == n):
            raise ValueError("%s mixes polygons of different vertex counts" % path)
        offset += count * dt.itemsize
    return out


def _read_ascii(path, blob, offset, elements):
    lines = blob[offset:].decode("ascii", "replace").split("\n")
    out, row = {}, 0
    for name, count, props in elements:
        block = [ln.split() for ln in lines[row:row + count]]
        row += count
        if len(block) != count:
            raise ValueError("%s is truncated in its %s element" % (path, name))
        widths = {len(b) for b in block}
        if len(widths) > 1:
            raise ValueError("%s mixes polygons of different vertex counts" % path if name == "face" else
                             "%s: rows of its %s element differ in length" % (path, name))
        vals = np.array(block, dtype=np.float64).reshape(count, -1) if count else np.zeros((0, 0))
        if any(len(p) == 3 for p in props):
            if name != "face":
                raise ValueError("%s: list properties are supported on the face element only" % path)
            k, _, it = _face_layout(path, props)
            n = int(vals[0, k]) if count else 0
            if count and (vals.shape[1] != len(props) + n or not np.all(vals[:, k] == n)):
                raise ValueError("%s mixes polygons of different vertex counts" % path)
            out[name] = dict(n=np.full(count, n), v=vals[:, k + 1:k + 1 + n].astype(np.int64))
        else:
            if count and vals.shape[1] != len(props):
                raise ValueError("%s: its %s rows do not have %d values" % (path, name, len(props)))
            out[name] = {p[0]: vals[:, j].astype(p[1]) for j, p in enumerate(props)}
    return out


def load_mesh_ply(path):
    """A triangle mesh from a PLY: (vertices [V,3] float32, colors [V,3] uint8, faces [F,3] int32).  Reads binary
    little-endian and ASCII files with a `vertex` element holding x, y, z and any other scalar properties (skipped;
    red, green, blue are the colours when present, clipped into uint8, zeros otherwise) and a `face` element whose
    list property vertex_indices or vertex_index has an integer count and index type.  Every face must have the
    same vertex count n >= 3; n-gons are fanned into n - 2 triangles (v0, vk, vk+1).  ValueError, naming the path,
    for big-endian files, mixed polygon counts, indices outside [0, V) and non-finite vertices that a face uses.
    Reads what save_mesh_ply writes exactly as written."""
    with open(path, "rb") as f:
        blob = f.read()
    fmt, elements, offset = _parse_ply_header(path, blob)
    names = [e[0] for e in elements]
    if "vertex" not in names:
        raise ValueError("%s has no vertex element" % path)
    data = (_read_binary if fmt == "binary_little_endian" else _read_ascii)(path, blob, offset, elements)
    vert = data["vertex"]
    vprops = [p[0] for p in elements[names.index("vertex")][2]]
    if not {"x", "y", "z"} <= set(vprops):
        raise ValueError("%s: the vertex element lacks x, y or z" % path)
    verts = np.stack([np.asarray(vert[k]) for k in ("x", "y", "z")], 1).astype(np.float32)
    if {"red", "green", "blue"} <= set(vprops):
        cols = np.stack([np.clip(np.asarray(vert[k]), 0, 255) for k in ("red", "green", "blue")], 1).astype(np.uint8)
    else:
        cols = np.zeros((len(verts), 3), np.uint8)
    if "face" not in data or len(data["face"]["n"]) == 0:
        return verts, cols, np.zeros((0, 3), np.int32)
    poly = np.asarray(data["face"]["v"]).astype(np.int64)
    n = poly.shape[1]
    if n < 3:
        raise ValueError("%s has faces of %d vertices" % (path, n))
    if poly.min() < 0 or poly.max() >= len(verts):
        raise ValueError("%s has face indices outside [0, %d)" % (path, len(verts)))
    used = np.zeros(len(verts), bool)
    used[poly.reshape(-1)] = True
    if not np.all(np.isfinite(verts[used])):
        raise ValueError("%s has non-finite vertices that faces use" % path)
    if n == 3:
        return verts, cols, np.ascontiguousarray(poly).astype(np.int32)
    k = np.arange(1, n - 1)
    tris = np.stack([np.broadcast_to(poly[:, :1], (len(poly), n - 2)), poly[:, k], poly[:, k + 1]], -1)
    return verts, cols, tris.reshape(-1, 3).astype(np.int32)
