"""Data formats either side of the hot path (SURVEY.md section 8(f) row N4): SplaTAM's `params.npz` checkpoints
and the 3DGS-viewer PLY export, byte-compatible with what the reference writes.

* ``save_params`` / ``save_params_ckpt`` / ``load_params``   R/utils/common_utils.py:25-52 (np.savez of every entry of
  the params dict, tensors as contiguous CPU numpy arrays, non-tensors stored as they are)
* ``save_checkpoint`` / ``load_checkpoint``                  R/scripts/splatam.py:604-643,927-931 (`params{t}.npz` and
  `keyframe_time_indices{t}.npy`, plus a `run_state{t}.npz` sidecar that only this project reads)
* ``save_run_record``                                        R/scripts/splatam.py:973-986 (the final `params.npz` with
  the reference's 14 keys)
* ``save_ply`` / ``load_ply`` / ``export_ply``               R/scripts/export_ply.py:20-77 (binary little-endian PLY,
  one `vertex` element of 17 float32 properties; the reference writes it through the `plyfile` package, which is
  not a dependency here: the header and the packed records are produced directly)
"""
import os

import numpy as np

GAUSSIAN_KEYS = ("means3D", "rgb_colors", "unnorm_rotations", "logit_opacities", "log_scales")
CHECKPOINT_KEYS = GAUSSIAN_KEYS + ("cam_unnorm_rots", "cam_trans")
# the keys save_params writes at the end of the reference's run, in its order (splatam.py:973-983)
RECORD_KEYS = CHECKPOINT_KEYS + ("timestep", "intrinsics", "w2c", "org_width", "org_height", "gt_w2c_all_frames",
                                 "keyframe_time_indices")

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
    import torch
    out = {}
    for k, v in raw.items():
        if isinstance(v, np.ndarray) and v.dtype.kind == "f":
            out[k] = torch.from_numpy(np.ascontiguousarray(v)).to(device).float()
        else:
            out[k] = v
    return out


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
    import torch
    p_path, k_path, s_path = _ckpt_paths(directory, time_idx)
    for path in (p_path, k_path):
        if not os.path.isfile(path):
            raise FileNotFoundError("checkpoint file not found: %s" % path)
    with np.load(p_path) as z:
        missing = [k for k in CHECKPOINT_KEYS if k not in z.files]
        if missing:
            raise ValueError("%s lacks %s" % (p_path, ", ".join(missing)))
        raw = {k: z[k] for k in CHECKPOINT_KEYS}
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(device).float()
    state = None
    if os.path.isfile(s_path):
        with np.load(s_path) as z:
            state = {k: z[k] for k in z.files}
    return dict(time_idx=int(time_idx), gauss={k: t(raw[k]) for k in GAUSSIAN_KEYS},
                cam_unnorm_rots=t(raw["cam_unnorm_rots"]), cam_trans=t(raw["cam_trans"]),
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
