"""Relocalisation for SplaTAM runs and localisation in a saved map: thumbnail retrieval and ICP verification on the GPU
(csrc/reloc.cu; the rules are stated in include/splatam_b200.h).

Tracking fits each frame to the map from a guess near the previous pose; after a jump (dropped frames, a resumed
capture, a fast turn) it converges to a wrong pose.  `health` tells, from the map's depth/silhouette render at the
tracked pose, whether the frame's depth agrees with the map.  `relocalise` finds where a frame is when its pose is
unknown: its small grey/depth descriptor (`thumbnails`) is scored against a `Database` of descriptors at known camera
columns, and each of the k best candidates is verified by ICP (icp.align) against the map rendered at the candidate's
pose; the best verified pose is refined by tracking and kept only if it passes the health check.

* ``DEFAULTS``           every key of run_slam's `relocalise` dict and its default; ``config`` checks a dict
* ``thumbnails``         sb_reloc_thumbnails: [B,2,h,w] descriptors of B RGB-D images
* ``score`` / ``topk``   sb_reloc_score and sb_reloc_topk
* ``Database``           descriptors with their camera columns; poses are read from camera columns at query time
* ``health``             sb_track_health (with cfg["photometric"], sb_track_health_rgb, which adds the colour NCC of the
                         map's RGB render against the frame's) on the render at column t; ``read_health`` is its host
                         view
* ``relocalise``         retrieval, ICP verification, tracking and the health check; writes column t only on success
* ``localise_sequence``  tracks a new sequence in a saved map that stays frozen, relocalising lost frames

CUDA only; CPU tensors raise."""
import ctypes
import math
import numbers

import numpy as np
import torch
import torch.nn.functional as F

from . import _lib, icp
from . import mapping as M
from .loop import _rigid_inv

DEFAULTS = dict(
    k=5,                            # candidates verified by ICP
    tau_abs=0.05,                   # health: a covered pixel is an inlier within max(tau_abs [m], ...
    tau_rel=0.02,                   # ... tau_rel * frame depth)
    min_coverage=0.05,              # health: covered / valid-depth pixels
    min_inliers=0.5,                # health: inliers / covered pixels
    min_inlier_frac=0.6,            # ICP acceptance of a candidate, on top of sb_icp_align's own
    max_rms=0.02,                   # [m]
    photometric=False,              # health: sb_track_health_rgb; candidates verified by icp.align_rgbd
    min_ncc=0.7,                    # photometric health: colour NCC of the map render against the frame (inliers)
)
MAX_K = 8
HEALTH_STATS = 5
HEALTH_RGB_STATS = 7
HEALTH_BLOCKS = 128
HEALTH_RGB_SCRATCH = 22 * HEALTH_BLOCKS     # two passes of 11 partial sums per block


def config(relocalise):
    """DEFAULTS updated by `relocalise` (a dict); unknown keys and out-of-range values raise ValueError."""
    if not isinstance(relocalise, dict):
        raise ValueError("relocalise must be None or a dict, got %r" % (relocalise,))
    bad = sorted(set(relocalise) - set(DEFAULTS))
    if bad:
        raise ValueError("unknown relocalise keys %s (known: %s)" % (bad, sorted(DEFAULTS)))
    cfg = dict(DEFAULTS, **relocalise)

    def num(k, lo, hi=math.inf, lo_open=False):
        v = cfg[k]
        if not (isinstance(v, numbers.Real) and not isinstance(v, bool) and math.isfinite(v) and v <= hi
                and (v > lo if lo_open else v >= lo)):
            raise ValueError("relocalise[%r] = %r is out of range" % (k, v))
        return float(v)

    k = cfg["k"]
    if isinstance(k, bool) or not isinstance(k, numbers.Integral) or not 1 <= k <= MAX_K:
        raise ValueError("relocalise['k'] = %r must be an integer in [1, %d]" % (k, MAX_K))
    cfg["k"] = int(k)
    cfg["tau_abs"] = num("tau_abs", 0.0, lo_open=True)
    cfg["tau_rel"] = num("tau_rel", 0.0)
    for key in ("min_coverage", "min_inliers", "min_inlier_frac"):
        cfg[key] = num(key, 0.0, 1.0)
    cfg["max_rms"] = num("max_rms", 0.0, lo_open=True)
    if not isinstance(cfg["photometric"], bool):
        raise ValueError("relocalise['photometric'] = %r must be True or False" % (cfg["photometric"],))
    cfg["min_ncc"] = num("min_ncc", -1.0, 1.0)
    return cfg


def thumbnail_size(H, W):
    h, w = ctypes.c_int(0), ctypes.c_int(0)
    _lib.call("sb_reloc_thumbnail_size", int(H), int(W), ctypes.byref(h), ctypes.byref(w))
    return h.value, w.value


def thumbnails(im, depth, sil=None):
    """Descriptors float32 [B,2,h,w] of im [B,3,H,W] (or [3,H,W]), depth [B,H,W] (or [H,W], [1,H,W]) and, for a map
    render (depth then being its depth_acc), its silhouette in depth's shape; a sensor frame passes sil=None."""
    _lib.need_cuda("reloc.thumbnails", im, depth, *([] if sil is None else [sil]))
    im = im.reshape(-1, *im.shape[-3:]).float().contiguous()
    B, _, H, W = im.shape
    depth = depth.reshape(B, H, W).float().contiguous()
    sil = None if sil is None else sil.reshape(B, H, W).float().contiguous()
    h, w = thumbnail_size(H, W)
    scratch = torch.empty(B, 2, h, w, device=im.device)
    out = torch.empty(B, 2, h, w, device=im.device)
    _lib.call("sb_reloc_thumbnails", B, H, W, im, depth, sil, scratch, out, device=im.device)
    return out


def score(query, database):
    """Scores float64 [N] of query [2,h,w] against database [N,2,h,w] (sb_reloc_score)."""
    _lib.need_cuda("reloc.score", query, database)
    N = database.shape[0]
    if query.numel() != database[0].numel() or query.numel() % 2:
        raise ValueError("query %s does not match the database's %s" % (tuple(query.shape), tuple(database.shape)))
    out = torch.empty(N, dtype=torch.float64, device=database.device)
    _lib.call("sb_reloc_score", N, query.numel() // 2, query.float().contiguous(), database.float().contiguous(), out,
              device=database.device)
    return out


def topk(scores, k):
    """(indices int32 [k'], scores float64 [k']) of the k' = min(k, N) best scores, on the device (sb_reloc_topk)."""
    _lib.need_cuda("reloc.topk", scores)
    k = min(int(k), scores.numel())
    idx = torch.empty(k, dtype=torch.int32, device=scores.device)
    top = torch.empty(k, dtype=torch.float64, device=scores.device)
    _lib.call("sb_reloc_topk", scores.numel(), k, scores.double().contiguous(), idx, top, device=scores.device)
    return idx, top


class Database:
    """Descriptors [N,2,h,w] and the camera column each was taken at.  `cameras` = (cam_unnorm_rots, cam_trans) of the
    map the columns belong to (a saved record), or None: the camera tensors of the run that queries it.  Poses are read
    from those columns when a query runs, so keyframe-pose refinement and loop closure, which move the columns, move
    the database too."""

    def __init__(self, cameras=None):
        self.cameras = cameras
        self.columns = []
        self._parts = []
        self._desc = None

    def __len__(self):
        return len(self.columns)

    def add(self, frame, column):
        """Adds the descriptor of `frame` (dict with im [3,H,W], depth and, for a map render, sil) at `column`.  A
        frame that carries a silhouette (slam.render_frame's synthetic frames) is described as a render, here and in
        `relocalise`'s query."""
        self.extend(thumbnails(frame["im"], frame["depth"], frame.get("sil")), [column])

    def extend(self, desc, columns):
        self._parts.append(desc)
        self._desc = None
        self.columns += [int(c) for c in columns]

    @property
    def descriptors(self):
        if self._desc is None:
            self._desc = torch.cat(self._parts) if len(self._parts) > 1 else self._parts[0]
            self._parts = [self._desc]
        return self._desc

    def w2c(self, rots, trans, i):
        """(w2c [4,4], normalised quaternion [1,4]) of entry i from `cameras`, else from rots / trans."""
        r, t = self.cameras if self.cameras is not None else (rots, trans)
        c = self.columns[i]
        return M.camera_w2c(r[..., c], t[..., c])

    @classmethod
    def from_record(cls, params, columns, cam, w2c0=None, render=None, fused=None, batch=32):
        """A database of renders of a saved map (`params`: Gaussian and camera tensors on the device) at camera
        `columns`, through mapping._render_pair; the thumbnails of each batch of renders are made in one call."""
        db = cls((params["cam_unnorm_rots"], params["cam_trans"]))
        dev = params["means3D"].device
        w2c0 = torch.eye(4, device=dev) if w2c0 is None else w2c0.to(dev).float()
        render = M.default_render if render is None else render
        fused = (params["means3D"].is_cuda and render is M.default_render) if fused is None else fused
        columns = [int(c) for c in columns]
        for s in range(0, len(columns), batch):
            ims, ds = [], []
            with torch.no_grad():
                for c in columns[s:s + batch]:
                    im, d, _, _ = M._render_pair(params, dict(id=c, cam=cam, w2c=w2c0), render, fused,
                                                 camera_grad=False)
                    ims.append(im)
                    ds.append(d)
                d = torch.stack(ds)
                db.extend(thumbnails(torch.stack(ims), d[:, 0], d[:, 1]), columns[s:s + batch])
        return db


def _health_of(ds, depth, cfg):
    _lib.need_cuda("reloc.health", ds, depth)
    H, W = ds.shape[-2:]
    scratch = torch.empty(4 * HEALTH_BLOCKS, dtype=torch.float64, device=ds.device)
    stats = torch.empty(HEALTH_STATS, dtype=torch.float64, device=ds.device)
    _lib.call("sb_track_health", H, W, ds[:2].float().contiguous(), depth.reshape(H, W).float().contiguous(),
              cfg["tau_abs"], cfg["tau_rel"], cfg["min_coverage"], cfg["min_inliers"], scratch, stats, device=ds.device)
    return stats


def _health_rgb_of(ds, im, depth, rgb, cfg):
    _lib.need_cuda("reloc.health", ds, im, depth, rgb)
    H, W = ds.shape[-2:]
    scratch = torch.empty(HEALTH_RGB_SCRATCH, dtype=torch.float64, device=ds.device)
    stats = torch.empty(HEALTH_RGB_STATS, dtype=torch.float64, device=ds.device)
    _lib.call("sb_track_health_rgb", H, W, ds[:2].float().contiguous(), depth.reshape(H, W).float().contiguous(),
              im.reshape(3, H, W).float().contiguous(), rgb.reshape(3, H, W).float().contiguous(), cfg["tau_abs"],
              cfg["tau_rel"], cfg["min_coverage"], cfg["min_inliers"], cfg["min_ncc"], scratch, stats,
              device=ds.device)
    return stats


def health(params, frame, t, cfg=None, render=None, fused=None):
    """The health record (device float64 [5]: valid, covered, inliers, rms, healthy) of frame t: its depth against
    the map's depth/silhouette render at column t of params (sb_track_health).  With cfg["photometric"], [7]: also
    the NCC pairs and the colour NCC of the map's RGB render against the frame's, which `healthy` then includes
    (sb_track_health_rgb)."""
    cfg = config({}) if cfg is None else cfg
    if cfg["photometric"]:
        im, ds = icp.model_render(params, t, frame, render, fused)
        return _health_rgb_of(ds, im, frame["depth"], frame["im"], cfg)
    return _health_of(icp.model_depth_sil(params, t, frame, render, fused), frame["depth"], cfg)


def read_health(stats):
    """Host dict of a health record (one device read): ok, valid, covered, inliers, coverage, inlier_frac, rms; for
    a photometric record also ncc_pairs and ncc."""
    s = stats.detach().cpu().numpy()
    d = dict(ok=bool(s[4]), valid=int(s[0]), covered=int(s[1]), inliers=int(s[2]),
             coverage=float(s[1] / s[0]) if s[0] > 0 else 0.0, inlier_frac=float(s[2] / s[1]) if s[1] > 0 else 0.0,
             rms=float(s[3]))
    if len(s) >= HEALTH_RGB_STATS:
        d.update(ncc_pairs=int(s[5]), ncc=float(s[6]))
    return d


def _render_at(params, frame, pose, render, fused, rgb=False):
    render = M.default_render if render is None else render
    fused = (params["means3D"].is_cuda and render is M.default_render) if fused is None else fused
    with torch.no_grad():
        im, ds, _, _ = M._render_pair(params, dict(id=frame["id"], cam=frame["cam"], w2c=frame["w2c"], pose=pose),
                                      render, fused, camera_grad=False)
    return (im, ds) if rgb else ds


def _column_of(w2c, w2c0):
    """(normalised quaternion [4], translation [3]) of camera column values giving `w2c` under first-frame w2c0;
    the quaternion with w >= 0."""
    rel = _rigid_inv(w2c0) @ w2c
    q = F.normalize(M.matrix_to_quaternion(rel[:3, :3]), dim=0)
    return torch.where(q[0] < 0, -q, q), rel[:3, 3]


def relocalise(params, frame, t, db, intrinsics, cfg=None, tracking=None, render=None, fused=None):
    """Finds frame t in the map when its pose is unknown and writes column t of params' camera tensors on success.

    1. The frame's descriptor is scored against `db` and the k best entries (scores above -2) are the candidates.
    2. Each candidate's pose (db.w2c) renders the map's depth/silhouette; icp.align aligns the frame's depth with it,
       the candidate pose being both w2c_prev and w2c_init (with cfg["photometric"], icp.align_rgbd against the
       candidate render's RGB too).  A candidate is accepted if the alignment accepts it and its inlier fraction >=
       min_inlier_frac and RMS <= max_rms.
    3. The first accepted candidate in score order wins (the higher score, then the lower index); its ICP pose goes
       into column t and mapping.track_frame refines it (`tracking`: its keyword arguments; the map is detached).
    4. The health check at column t decides: healthy keeps the column, otherwise column t is restored bit for bit.
    Returns dict(accepted, candidates [db indices], columns, scores, icp [per candidate dict(accepted, inlier_frac, rms,
    inliers)], chosen (db index or None), health (read_health of the final check, None if no candidate was
    accepted)).  Host reads: one for the candidates, one for all their ICP records, those of track_frame (one per
    iteration when eager) and one for the health record."""
    cfg = config({}) if cfg is None else cfg
    tracking = {} if tracking is None else tracking
    rots, trans = params["cam_unnorm_rots"], params["cam_trans"]
    _lib.need_cuda("reloc.relocalise", rots, frame["depth"], params["means3D"])
    rec = dict(frame=int(t), accepted=False, candidates=[], columns=[], scores=[], icp=[], chosen=None, health=None)
    if len(db) == 0:
        return rec
    q = thumbnails(frame["im"], frame["depth"], frame.get("sil"))[0]
    idx, top = topk(score(q, db.descriptors), cfg["k"])
    idx, top = idx.tolist(), top.tolist()                                 # host read 1
    cands = [(i, s) for i, s in zip(idx, top) if s > -2.0]
    rec["candidates"] = [i for i, _ in cands]
    rec["columns"] = [db.columns[i] for i in rec["candidates"]]
    rec["scores"] = [s for _, s in cands]
    if not cands:
        return rec
    w2c0 = frame["w2c"].float()
    outs, stats = [], []
    for i, _ in cands:
        w2c_c, q_c = db.w2c(rots, trans, i)
        pose = w2c0 @ w2c_c
        if cfg["photometric"]:
            im, ds = _render_at(params, frame, (w2c_c, q_c), render, fused, rgb=True)
            out, st = icp.align_rgbd(ds, im, frame["depth"], frame["im"], intrinsics, pose, pose)
        else:
            ds = _render_at(params, frame, (w2c_c, q_c), render, fused)
            out, st = icp.align(ds, frame["depth"], intrinsics, pose, pose)
        outs.append(out)
        stats.append(st)
    host = torch.stack(stats).cpu().numpy()                               # host read 2
    best = None
    for n, ((i, s), st) in enumerate(zip(cands, host)):
        ok = bool(st[0]) and st[1] >= cfg["min_inlier_frac"] and st[2] <= cfg["max_rms"]
        rec["icp"].append(dict(accepted=ok, inlier_frac=float(st[1]), rms=float(st[2]), inliers=int(st[3])))
        if ok and best is None:
            best = n
    if best is None:
        return rec
    rec["chosen"] = cands[best][0]
    with torch.no_grad():
        old_r, old_t = rots[..., t].detach().clone(), trans[..., t].detach().clone()
        qv, tv = _column_of(outs[best], w2c0)
        rots[0, :, t] = qv
        trans[0, :, t] = tv
    M.track_frame(params, frame, render=render, fused=fused, **tracking)
    rots, trans = params["cam_unnorm_rots"], params["cam_trans"]
    h = read_health(health(params, frame, t, cfg, render, fused))         # host read 3
    rec["health"] = h
    rec["accepted"] = h["ok"]
    if not h["ok"]:
        with torch.no_grad():
            rots[..., t] = old_r
            trans[..., t] = old_t
    return rec


def localise_sequence(params, frames, intrinsics, db, cfg=None, pose_init="constant_velocity", tracking=None,
                      render=None, fused=None):
    """Localises `frames` (dicts with id = 0..T-1, cam, w2c, im, depth) in a saved map that stays frozen: frame 0 is
    relocalised (it has no prior); every later frame starts from the constant-velocity guess (with pose_init="icp",
    refined by icp.init_pose), is tracked, health-checked and relocalised when lost.  A frame that stays lost takes
    the previous frame's column; the frame after a relocalised or lost one starts with zero velocity.  The map's
    Gaussians in `params` are used detached; `db` holds the record's cameras.  Returns dict(rots [1,4,T], trans
    [1,3,T] in the map's frame, lost, relocalised (bool lists), health [T, 5] (host; [T, 7] with cfg["photometric"]:
    also the NCC pairs and the NCC), reloc (relocalise records))."""
    if pose_init not in ("constant_velocity", "icp", "rgbd_icp"):
        raise ValueError("pose_init must be 'constant_velocity', 'icp' or 'rgbd_icp', got %r" % (pose_init,))
    cfg = config({}) if cfg is None else cfg
    tracking = {} if tracking is None else tracking
    dev = params["means3D"].device
    _lib.need_cuda("reloc.localise_sequence", params["means3D"])
    T = len(frames)
    rots = torch.zeros(1, 4, T, device=dev)
    rots[:, 0] = 1.0
    trans = torch.zeros(1, 3, T, device=dev)
    gauss = {k: v.detach() for k, v in params.items() if k not in M.CAM_KEYS}
    lost, relocd, healths, recs = [False] * T, [False] * T, [], []
    for t in range(T):
        with torch.no_grad():
            if t > 1 and not (lost[t - 1] or relocd[t - 1]):
                r1, r2 = F.normalize(rots[0, :, t - 1], dim=0), F.normalize(rots[0, :, t - 2], dim=0)
                rots[0, :, t] = F.normalize(r1 + (r1 - r2), dim=0)
                trans[0, :, t] = trans[0, :, t - 1] + (trans[0, :, t - 1] - trans[0, :, t - 2])
            elif t > 0:
                rots[0, :, t] = rots[0, :, t - 1]
                trans[0, :, t] = trans[0, :, t - 1]
        p = dict(gauss, cam_unnorm_rots=rots, cam_trans=trans)
        h = None
        if t > 0:
            if pose_init != "constant_velocity":
                icp.init_pose(p, frames[t], t, intrinsics, render=render, fused=fused,
                              photometric=pose_init == "rgbd_icp")
            M.track_frame(p, frames[t], render=render, fused=fused, **tracking)
            rots, trans = p["cam_unnorm_rots"].detach(), p["cam_trans"].detach()
            p = dict(gauss, cam_unnorm_rots=rots, cam_trans=trans)
            h = read_health(health(p, frames[t], t, cfg, render, fused))
        if h is None or not h["ok"]:
            r = relocalise(p, frames[t], t, db, intrinsics, cfg, tracking, render, fused)
            rots, trans = p["cam_unnorm_rots"].detach(), p["cam_trans"].detach()
            recs.append(r)
            if r["accepted"]:
                relocd[t], h = True, r["health"]
            else:
                lost[t] = True
                if t > 0:
                    with torch.no_grad():
                        rots[..., t] = rots[..., t - 1]
                        trans[..., t] = trans[..., t - 1]
                if h is None:
                    h = read_health(health(p, frames[t], t, cfg, render, fused))
        healths.append([h["valid"], h["covered"], h["inliers"], h["rms"], float(h["ok"])] +
                       ([h["ncc_pairs"], h["ncc"]] if cfg["photometric"] else []))
    return dict(rots=rots, trans=trans, lost=lost, relocalised=relocd, health=np.array(healths, dtype=np.float64),
                reloc=recs)
