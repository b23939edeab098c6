"""Which Gaussians of a map do its views use?  Per-Gaussian blend statistics on the GPU (csrc/blend_forward.cu's stats
walk, sb_blend_stats) and the compaction of a run record that they make lossless.

* ``BlendStats``     accumulates, over any number of finished renders of one map, per Gaussian: `blended` (pixels it
                     was composited into), `ended` (pixels whose walk it stopped: test_T < 1e-4, nothing blended) and
                     `max_weight` (its largest blend weight alpha T)
* ``blend_stats``    those statistics over views of a record, each rendered exactly as `evaluate` renders it
                     (mapping._render_pair on the fused path, camera_grad=False, at the record's camera column)
* ``keep_mask``      the keep rule: blended > 0 or ended > 0 (lossless), or max_weight >= min_weight (lossy)
* ``compact_record`` a run record without the Gaussians the rule drops, every other entry copied as it is

Lossless: removing, in index order, Gaussians that blended and ended nothing at the views V leaves every survivor's
projection, its place in each tile list and every pixel's walk unchanged, so colour, depth/silhouette and final_T at
every view of V are bit-identical (DESIGN.md section 7, "Map compaction").  Other views get no guarantee."""
import ctypes
import os
import time

import numpy as np
import torch

from . import _lib
from . import formats
from . import mapping as M
from .rasterizer import forward_states

COUNTER_MAX = 2 ** 32 - 1          # the counters are uint32: at most this many (view, pixel) pairs per accumulation
# the record entries compact_record needs: the Gaussians, the cameras and their settings
RECORD_NEED = formats.CHECKPOINT_KEYS + ("timestep",) + formats.CAMERA_KEYS
PER_GAUSSIAN_KEYS = formats.GAUSSIAN_KEYS + ("timestep",)


class BlendStats:
    """Statistics of P Gaussians summed over the renders `add` is given.  Device arrays, integer and max atomics only:
    the same renders give the same bits."""

    def __init__(self, P, device):
        self.P, self.device = int(P), torch.device(device)
        if self.P < 0:
            raise ValueError("BlendStats needs P >= 0, got %d" % self.P)
        z = lambda: torch.zeros(max(self.P, 1), dtype=torch.int32, device=self.device)
        self._blended, self._ended, self._wbits = z(), z(), z()
        self.pixels = 0                       # (view, pixel) pairs accumulated so far
        self.views = 0

    def reserve(self, views, height, width):
        """ValueError unless `views` more H x W renders keep every counter below 2^32."""
        more = int(views) * int(height) * int(width)
        if self.pixels + more > COUNTER_MAX:
            raise ValueError("%d views of %dx%d on top of %d accumulated pixels could overflow the uint32 counters "
                             "(at most %d pixels per accumulation)" % (views, width, height, self.pixels, COUNTER_MAX))

    def add(self, state):
        """Adds the statistics of the finished render whose workspaces `state` holds (rasterizer.forward_states)."""
        if state.P != self.P:
            raise ValueError("a render of %d Gaussians added to statistics of %d" % (state.P, self.P))
        c = state.settings.c
        self.reserve(1, c.image_height, c.image_width)
        b = state.binning
        _lib.call("sb_blend_stats", ctypes.byref(state.settings.c), self.P, int(state.num_rendered), int(state.sync_free),
                  state.geom, state.geom.numel(), b, b.numel(), state.image, state.image.numel(), self._blended,
                  self._ended, self._wbits, device=self.device)
        self.pixels += int(c.image_height) * int(c.image_width)
        self.views += 1

    def result(self):
        """dict(blended int64 [P], ended int64 [P], max_weight float32 [P]) on the device."""
        u = lambda t: t[:self.P].to(torch.int64) & 0xFFFFFFFF
        return dict(blended=u(self._blended), ended=u(self._ended), max_weight=self._wbits[:self.P].view(torch.float32))


def _frame(t, cam, first_w2c):
    return dict(id=int(t), cam=cam, w2c=first_w2c)


def blend_stats(params, cam, view_ids, first_w2c, max_rendered=None):
    """BlendStats.result() of the Gaussians in `params` (the five Gaussian tensors plus cam_unnorm_rots / cam_trans
    [.., T], on one CUDA device) over the views `view_ids` (camera columns), each rendered as `evaluate` renders it:
    mapping._render_pair on the fused path, camera_grad=False, raster settings `cam`, first-frame w2c `first_w2c`.
    max_rendered: render sync-free with that instance capacity (an overflowed view adds nothing).  ValueError, before
    any render, when the views could overflow the counters."""
    _lib.need_cuda("blend_stats", params["means3D"])
    dev = params["means3D"].device
    acc = BlendStats(params["means3D"].shape[0], dev)
    acc.reserve(len(view_ids), cam.image_height, cam.image_width)
    first_w2c = torch.as_tensor(first_w2c).to(dev).float()
    with torch.no_grad(), torch.cuda.device(dev):
        for t in view_ids:
            with forward_states() as states:
                M._render_pair(params, _frame(t, cam, first_w2c), M.default_render, True, camera_grad=False,
                               max_rendered=max_rendered)
            acc.add(states[-1])
    return acc.result()


def keep_mask(stats, min_weight=0.0):
    """bool [P] of the Gaussians to keep.  min_weight == 0 (lossless): blended > 0 or ended > 0 -- a Gaussian that
    only ends walks blends nothing, but dropping it would let those pixels go on to blend the next Gaussian.
    min_weight > 0 (lossy): max_weight >= min_weight, so no pixel of the views received min_weight or more from a
    dropped Gaussian."""
    min_weight = float(min_weight)
    if not min_weight >= 0.0:
        raise ValueError("min_weight must be >= 0, got %r" % min_weight)
    if min_weight == 0.0:
        return (stats["blended"] > 0) | (stats["ended"] > 0)
    return stats["max_weight"] >= min_weight


def compact_arrays(rec, keep):
    """The record `rec` (dict of host arrays) without the Gaussians `keep` (bool [P], any device) drops: the
    per-Gaussian arrays (formats.GAUSSIAN_KEYS and timestep, float32) through map_ops.compact_plan / compact_flat,
    which keep index order; every other entry is the same object.  Runs on keep's device."""
    from . import map_ops
    P = int(np.shape(rec["means3D"])[0])
    keys = [k for k in PER_GAUSSIAN_KEYS if k in rec]
    for k in keys:
        if np.asarray(rec[k]).dtype != np.float32:
            raise ValueError("%s is %s; compaction keeps float32 Gaussian arrays" % (k, np.asarray(rec[k]).dtype))
    keep = torch.as_tensor(keep)
    if keep.dtype != torch.bool or keep.numel() != P:
        raise ValueError("keep must be a bool mask of %d Gaussians" % P)
    dev = keep.device
    widths = [int(np.prod(np.shape(rec[k])[1:], dtype=np.int64)) for k in keys]
    flat = torch.cat([torch.from_numpy(np.ascontiguousarray(rec[k]).reshape(-1)) for k in keys]).to(dev)
    m8, dst, P_new = map_ops.compact_plan(keep)
    out_flat = map_ops.compact_flat(flat, P, widths, m8, dst, P_new).cpu().numpy()
    out, off = dict(rec), 0
    for k, w in zip(keys, widths):
        out[k] = out_flat[off:off + w * P_new].reshape((P_new,) + tuple(np.shape(rec[k])[1:]))
        off += w * P_new
    return out


def record_view(rec, device):
    """(params, cam, first_w2c) of a record: the Gaussians and cameras as float32 tensors on `device`, the raster
    settings from datasets.setup_camera(org_width, org_height, intrinsics, w2c)."""
    from .datasets import setup_camera
    params = formats.record_tensors(rec, formats.CHECKPOINT_KEYS, device)
    cam = setup_camera(int(rec["org_width"]), int(rec["org_height"]), np.asarray(rec["intrinsics"], np.float32),
                       np.asarray(rec["w2c"], np.float32), device)
    first_w2c = torch.from_numpy(np.asarray(rec["w2c"], np.float32).reshape(4, 4)).to(device)
    return params, cam, first_w2c


def _render_diff(params_a, params_b, cam, first_w2c, view_ids):
    """Mean over views of (PSNR, depth L1) of b's renders against a's, from sb_frame_metrics (no masks but a's depth
    > 0)."""
    from .evaluate import _PSNR, _L1
    H, W = int(cam.image_height), int(cam.image_width)
    dev = params_a["means3D"].device
    rows = torch.zeros(len(view_ids), 7, dtype=torch.float64, device=dev)
    w_im, w_gt = (torch.empty(3, H, W, dtype=torch.float32, device=dev) for _ in range(2))
    ws = torch.empty(_lib.nbytes("sb_frame_metrics_workspace_bytes", H, W), dtype=torch.uint8, device=dev)
    with torch.no_grad(), torch.cuda.device(dev):
        for k, t in enumerate(view_ids):
            fr = _frame(t, cam, first_w2c)
            ref_im, ref_ds, _, _ = M._render_pair(params_a, fr, M.default_render, True, camera_grad=False)
            im, ds, _, _ = M._render_pair(params_b, fr, M.default_render, True, camera_grad=False)
            _lib.call("sb_frame_metrics", im.contiguous(), ds.contiguous(), ref_im.contiguous(),
                      ref_ds[0:1].contiguous(), H, W, 0.0, 0, w_im, w_gt, ws, ws.numel(), rows[k], device=dev)
    m = rows.cpu().numpy()
    return float(m[:, _PSNR].mean()), float(m[:, _L1].mean())


def compact_record(src, dst, every=1, min_weight=0.0, device=None, compare=None):
    """Writes to `dst` the run record `src` (this project's or the reference's 14-key params.npz, or the 13-key
    offline record) without the Gaussians `keep_mask(blend_stats(...), min_weight)` drops, the statistics taken over
    the frames evaluate.select_frames(T, every) picks (T = the record's camera count).  The per-Gaussian arrays keep
    their index order; every other entry is copied with its dtype.  `src` is only read; ValueError when `dst` is `src`,
    for a record without cameras (a checkpoint) and for views that could overflow the counters.
    compare (default: min_weight > 0): also renders both maps at the views and reports the compacted map's PSNR and
    depth L1 against the original's.  Returns a dict: gaussians_before / _after, views, width, height, stats_s,
    compact_s, path, and psnr_db / depth_l1_m with `compare`."""
    from .evaluate import select_frames
    if os.path.abspath(src) == os.path.abspath(dst) or \
            (os.path.exists(dst) and os.path.exists(src) and os.path.samefile(src, dst)):
        raise ValueError("--out must differ from --record: the input record is never written")
    if int(every) < 1:
        raise ValueError("every must be >= 1, got %r" % every)
    rec = formats.read_record(src, RECORD_NEED)
    dev = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
    T = int(np.shape(rec["cam_unnorm_rots"])[-1])
    ids = select_frames(T, int(every))
    params, cam, first_w2c = record_view(rec, dev)
    torch.cuda.synchronize(dev)
    t0 = time.perf_counter()
    stats = blend_stats(params, cam, ids, first_w2c)
    keep = keep_mask(stats, min_weight)
    torch.cuda.synchronize(dev)
    t1 = time.perf_counter()
    out = compact_arrays(rec, keep)
    t2 = time.perf_counter()
    with open(dst, "wb") as f:            # a file object: np.savez would append .npz to a name without it
        np.savez(f, **out)
    res = dict(path=dst, gaussians_before=int(np.shape(rec["means3D"])[0]),
               gaussians_after=int(np.shape(out["means3D"])[0]), views=len(ids), width=int(cam.image_width),
               height=int(cam.image_height), stats_s=t1 - t0, compact_s=t2 - t1)
    if compare is None:
        compare = float(min_weight) > 0.0
    if compare:
        small = formats.record_tensors(out, formats.CHECKPOINT_KEYS, dev)
        res["psnr_db"], res["depth_l1_m"] = _render_diff(params, small, cam, first_w2c, ids)
    return res
