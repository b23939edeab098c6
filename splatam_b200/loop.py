"""Loop closure for SplaTAM runs: ICP loop constraints against old keyframes, a keyframe pose graph, and map
deformation on the GPU (csrc/loop.cu; the rules are stated in include/splatam_b200.h).

At a keyframe frame t, `close_loop` looks for old keyframes whose view frame t shares (`candidates`), measures the
relative pose to the first one that aligns well (`measure`, over icp.align with the keyframe's own sensor depth as the
model), adds that loop edge to the keyframe pose graph (`PoseGraph`) and solves it.  If every edge then fits, the
error is spread over the trajectory: every camera column, every stored keyframe pose and every Gaussian moves with the
correction of the graph node it belongs to (a Gaussian by its creation frame, `ShardedMapper.timestep`).

* ``DEFAULTS``           every key of run_slam's `loop_closure` dict and its default; ``config`` checks a dict
* ``candidates``         old keyframes near frame t's camera that overlap its view, best first
* ``measure``            the ICP loop measurement against one keyframe and its acceptance
* ``PoseGraph``          odometry and loop edges, the Gauss-Newton solve and the per-frame correction table
* ``deform_gaussians``   the map deformation kernel
* ``close_loop``         run_slam's step

CUDA only; CPU tensors raise."""
import math
import numbers

import numpy as np
import torch
import torch.nn.functional as F

from . import _lib, icp
from . import keyframes as KF
from . import mapping as M

DEFAULTS = dict(
    min_gap=60,                     # frames between an old keyframe and frame t
    max_dist=0.5,                   # camera centres within this distance [m] ...
    max_angle=30.0,                 # ... and optical axes within this angle [deg]
    points=1600,                    # depth samples of frame t for the overlap score
    min_overlap=0.3,                # keyframes.overlap_fractions of a candidate
    max_candidates=3,
    min_inlier_frac=0.6,            # loop ICP acceptance, on top of sb_icp_align's own
    max_rms=0.02,                   # [m]
    max_correction=(0.3, 15.0),     # the correction the loop implies at frame t [m, deg]
    odometry_weights=(1.0, 1.0),    # (w_rot, w_trans) of odometry edges
    loop_weights=(1.0, 1.0),        # (w_rot, w_trans) of loop edges
    iters=10,                       # Gauss-Newton iterations
    max_residual=(0.05, 3.0),       # every edge after the solve [m, deg]
)
ODOMETRY, LOOP = 0, 1
STEP_TOL = 1e-10                    # a Gauss-Newton step below this norm is not applied and ends the solve


def config(loop_closure):
    """DEFAULTS updated by `loop_closure` (a dict); unknown keys and out-of-range values raise ValueError."""
    if not isinstance(loop_closure, dict):
        raise ValueError("loop_closure must be None or a dict, got %r" % (loop_closure,))
    bad = sorted(set(loop_closure) - set(DEFAULTS))
    if bad:
        raise ValueError("unknown loop_closure keys %s (known: %s)" % (bad, sorted(DEFAULTS)))
    cfg = dict(DEFAULTS, **loop_closure)

    def num(k, lo, hi=math.inf, integer=False, lo_open=False):
        v = cfg[k]
        ok = isinstance(v, numbers.Real) and not isinstance(v, bool) and math.isfinite(v) and v <= hi and (
            v > lo if lo_open else v >= lo)
        if not ok or (integer and int(v) != v):
            raise ValueError("loop_closure[%r] = %r is out of range" % (k, v))
        return int(v) if integer else float(v)

    for k in ("min_gap", "points", "max_candidates", "iters"):
        cfg[k] = num(k, 1, integer=True)
    cfg["max_dist"] = num("max_dist", 0.0, lo_open=True)
    cfg["max_angle"] = num("max_angle", 0.0, 180.0, lo_open=True)
    for k in ("min_overlap", "min_inlier_frac"):
        cfg[k] = num(k, 0.0, 1.0)
    cfg["max_rms"] = num("max_rms", 0.0, lo_open=True)
    for k in ("max_correction", "odometry_weights", "loop_weights", "max_residual"):
        v = cfg[k]
        if not (isinstance(v, (tuple, list)) and len(v) == 2 and all(
                isinstance(x, numbers.Real) and not isinstance(x, bool) and math.isfinite(x) and x > 0 for x in v)):
            raise ValueError("loop_closure[%r] = %r must be two positive numbers" % (k, v))
        cfg[k] = (float(v[0]), float(v[1]))
    return cfg


def w2c_columns(rots, trans, ids):
    """[n,4,4] float32 w2c of camera columns `ids` (camera_w2c, batched)."""
    idx = torch.as_tensor(list(ids), dtype=torch.long, device=rots.device)
    q = F.normalize(rots[0].index_select(1, idx).T, dim=1)
    out = torch.zeros(len(ids), 4, 4, device=rots.device, dtype=torch.float32)
    out[:, :3, :3] = M.build_rotation(q)
    out[:, :3, 3] = trans[0].index_select(1, idx).T
    out[:, 3, 3] = 1.0
    return out


def _rigid_inv(m):
    """Inverse of rigid [...,4,4] transforms."""
    o = torch.zeros_like(m)
    Rt = m[..., :3, :3].transpose(-1, -2)
    o[..., :3, :3] = Rt
    o[..., :3, 3] = -(Rt @ m[..., :3, 3:4])[..., 0]
    o[..., 3, 3] = 1.0
    return o


def _centres(w2c):
    return -(w2c[..., :3, :3].transpose(-1, -2) @ w2c[..., :3, 3:4])[..., 0]


def _generator(seed, t):
    """The generator of frame t's overlap samples: its own, so the global RNGs draw what they draw without loop
    closure."""
    return torch.Generator().manual_seed((int(seed) * 1_000_003 + int(t)) % (2 ** 63 - 1))


def _need_cuda(what, *tensors):
    _lib.need_cuda(what, *tensors)


def candidates(frame, t, keyframes, rots, trans, intrinsics, cfg, seed=0):
    """Indices into `keyframes` of at most max_candidates keyframes j with t - id_j >= min_gap, camera centre within
    max_dist and optical axis within max_angle of frame t's (camera columns of record), and an overlap of at least
    min_overlap, highest first (ties: the older keyframe first), with their overlaps.  The overlap is
    keyframes.overlap_fractions of `points` samples of frame t's depth, drawn from the (seed, t) generator, over the
    samples with a valid depth.  One host read, none when no keyframe is old enough."""
    _need_cuda("loop.candidates", rots, trans, frame["depth"])
    ids = [i for i, kf in enumerate(keyframes) if t - int(kf["id"]) >= cfg["min_gap"]]
    if not ids:
        return [], []
    dev = rots.device
    w2c = w2c_columns(rots, trans, [int(keyframes[i]["id"]) for i in ids] + [t])
    kw, cur = w2c[:-1], w2c[-1]
    near = (_centres(kw) - _centres(cur)).norm(dim=-1) <= cfg["max_dist"]
    cos = (kw[:, 2, :3] * cur[2, :3]).sum(-1).clamp(-1.0, 1.0)
    aligned = cos >= math.cos(math.radians(cfg["max_angle"]))
    depth = frame["depth"].reshape(-1)
    H, W = frame["depth"].shape[-2:]
    K = torch.as_tensor(intrinsics, dtype=torch.float32).to(dev)
    idx = torch.randint(H * W, (cfg["points"],), generator=_generator(seed, t)).to(dev)
    z = depth.index_select(0, idx).float()
    valid = torch.isfinite(z) & (z > 0)
    u, v = (idx % W).float(), (idx // W).float()
    pc = torch.stack([(u - K[0, 2]) / K[0, 0] * z, (v - K[1, 2]) / K[1, 1] * z, z, torch.ones_like(z)], 0)
    pts = (_rigid_inv(cur) @ pc)[:3].T
    pts = torch.where(valid[:, None], pts, torch.full_like(pts, float("nan")))   # NaN projects inside no image
    frac = KF.overlap_fractions(pts, kw, K, W, H) * (cfg["points"] / valid.sum().clamp(min=1).float())
    score = torch.where(near & aligned, frac, torch.full_like(frac, -1.0))
    s = score.tolist()                                                    # the one host read
    order = sorted(range(len(ids)), key=lambda k: -s[k])
    keep = [k for k in order if s[k] >= cfg["min_overlap"]][:cfg["max_candidates"]]
    return [ids[k] for k in keep], [s[k] for k in keep]


def measure(keyframe, frame, t, rots, trans, intrinsics, cfg):
    """The loop measurement of frame t against `keyframe` by icp.align: the model is the keyframe's own sensor depth
    (silhouette 1) at its column pose, the data frame t's depth, the guess frame t's column.  Returns (record, Z):
    record = dict(frame, keyframe, accepted, inlier_frac, rms, correction_m, correction_deg), where `accepted` is
    sb_icp_align's acceptance and the loop tests (inlier fraction, RMS, the correction implied at frame t); Z [4,4]
    float64 device tensor, the measured w2c_t w2c_j^-1."""
    j = int(keyframe["id"])
    w2c = w2c_columns(rots, trans, [j, t])
    d = keyframe["depth"].reshape(keyframe["depth"].shape[-2:]).float()
    model = torch.stack([d, torch.ones_like(d)])
    out, st = icp.align(model, frame["depth"], intrinsics, w2c[0], w2c[1])
    Z = out.double() @ _rigid_inv(w2c[0].double())
    D = out.double() @ _rigid_inv(w2c[1].double())
    shift = (_centres(out.double()) - _centres(w2c[1].double())).norm()
    host = torch.cat([st[:3], shift.reshape(1), D[:3, :3].reshape(-1)]).cpu().numpy()
    ang = math.degrees(math.acos(min(1.0, max(-1.0, 0.5 * (host[4] + host[8] + host[12] - 1.0)))))
    ok = (host[0] == 1.0 and host[1] >= cfg["min_inlier_frac"] and host[2] <= cfg["max_rms"]
          and host[3] <= cfg["max_correction"][0] and ang <= cfg["max_correction"][1])
    rec = dict(frame=int(t), keyframe=j, accepted=bool(ok), inlier_frac=float(host[1]), rms=float(host[2]),
               correction_m=float(host[3]), correction_deg=float(ang))
    return rec, Z


def deform_gaussians(means3D, unnorm_rotations, timestep, table, apply_flag):
    """sb_deform_gaussians in place: means3D [P,3] and unnorm_rotations [P,4] float32 (views of one buffer are fine),
    timestep [P] float32, table [T,12] float32, apply_flag [1] int32, all on one device."""
    _need_cuda("loop.deform_gaussians", means3D, unnorm_rotations, timestep, table, apply_flag)
    P = means3D.shape[0]
    if (means3D.dtype != torch.float32 or unnorm_rotations.dtype != torch.float32 or timestep.dtype != torch.float32
            or table.dtype != torch.float32 or apply_flag.dtype != torch.int32):
        raise ValueError("deform_gaussians takes float32 maps, timestep and table and an int32 flag")
    if (tuple(means3D.shape) != (P, 3) or tuple(unnorm_rotations.shape) != (P, 4) or timestep.numel() != P
            or table.dim() != 2 or table.shape[1] != 12 or apply_flag.numel() != 1):
        raise ValueError("deform_gaussians: shapes %s %s %s %s %s" % tuple(
            tuple(x.shape) for x in (means3D, unnorm_rotations, timestep, table, apply_flag)))
    for x in (means3D, unnorm_rotations, timestep, table):
        if not x.is_contiguous():
            raise ValueError("deform_gaussians needs contiguous tensors")
    _lib.call("sb_deform_gaussians", P, means3D, unnorm_rotations, timestep, table.shape[0], table, apply_flag,
              device=means3D.device)


def _quaternions(R):
    """Batched matrix_to_quaternion: (w, x, y, z) [n,4] of rotations [n,3,3], up to sign."""
    m = R.reshape(-1, 9)
    m00, m01, m02, m10, m11, m12, m20, m21, m22 = m.unbind(1)
    four = torch.stack([1 + m00 + m11 + m22, 1 + m00 - m11 - m22, 1 - m00 + m11 - m22, 1 - m00 - m11 + m22], 1)
    cand = torch.stack([torch.stack([four[:, 0], m21 - m12, m02 - m20, m10 - m01], 1),
                        torch.stack([m21 - m12, four[:, 1], m10 + m01, m02 + m20], 1),
                        torch.stack([m02 - m20, m10 + m01, four[:, 2], m12 + m21], 1),
                        torch.stack([m10 - m01, m02 + m20, m12 + m21, four[:, 3]], 1)], 1)
    k = four.argmax(1)
    rows = cand[torch.arange(len(k), device=R.device), k]
    return rows / (2 * torch.sqrt(four.gather(1, k[:, None]).clamp(min=0)))


def _table_matrices(table):
    C = torch.zeros(table.shape[0], 4, 4, device=table.device, dtype=table.dtype)
    C[:, :3] = table.reshape(-1, 3, 4)
    C[:, 3, 3] = 1.0
    return C


def correct_cameras(rots, trans, table, t):
    """Columns 0..t move as w2c_s <- w2c_s C_s^-1, in place (the tensors' versions change, so fused_pose_cached sees
    it): the quaternion by the Hamilton product with C_s's conjugate, which keeps its norm and sign."""
    with torch.no_grad():
        C = table[:t + 1]
        R = C.reshape(-1, 3, 4)[:, :, :3]
        qc = F.normalize(_quaternions(R), dim=1)
        qc_conj = qc * torch.tensor([1.0, -1.0, -1.0, -1.0], device=qc.device)
        q = rots[0, :, :t + 1].T
        w2c = w2c_columns(rots, trans, range(t + 1))
        new = w2c @ _rigid_inv(_table_matrices(C))
        rots[0, :, :t + 1] = M.quat_mult(q, qc_conj).T
        trans[0, :, :t + 1] = new[:, :3, 3].T


class PoseGraph:
    """The keyframe pose graph.  Nodes are the frames that became keyframes, in order (the first node, frame
    `first`, is fixed); an odometry edge joins each node to the previous one, loop edges join a node to an old one.
    An edge is (i, j, Z, kind) with frame ids i, j and the measurement Z = w2c_j w2c_i^-1 ([4,4] float64)."""

    def __init__(self, first=0):
        self.first = int(first)
        self.edges = []

    def nodes(self):
        return [self.first] + [j for i, j, _, k in self.edges if k == ODOMETRY]

    def add_odometry(self, i, j, Z):
        if i != self.nodes()[-1]:
            raise ValueError("an odometry edge continues the chain from node %d, got %d" % (self.nodes()[-1], i))
        self.edges.append((int(i), int(j), Z, ODOMETRY))

    def add_loop(self, i, j, Z):
        nodes = self.nodes()
        if i not in nodes or j not in nodes or i == j:
            raise ValueError("a loop edge joins two different nodes, got %d, %d" % (i, j))
        self.edges.append((int(i), int(j), Z, LOOP))

    def odometry_from(self, rots, trans, t):
        """The odometry edge measurement to a new node t from the camera columns: w2c_t w2c_prev^-1 (device)."""
        w2c = w2c_columns(rots, trans, [self.nodes()[-1], t]).double()
        return w2c[1] @ _rigid_inv(w2c[0])

    def frame_nodes(self, T, t):
        """Node index of every frame s < T: the first node at or after s for s <= t, -1 (no correction) after t."""
        nodes = self.nodes()
        out, k = [], 0
        for s in range(T):
            while k < len(nodes) and nodes[k] < s:
                k += 1
            out.append(k if s <= t and k < len(nodes) else -1)
        return out

    def solve(self, w2c, T, t, cfg, extra=None):
        """Gauss-Newton over the nodes from their poses w2c [N,4,4] (device, node order), with the edges and `extra`
        (one more (i, j, Z, kind) edge, not kept).  Returns dict(poses [N,4,4] float64, correction_table [T,12] float32,
        flag [1] int32 (1: every edge within max_residual), edge_err [E,2] (m, rad), steps) on the device."""
        edges = self.edges + ([extra] if extra is not None else [])
        nodes = self.nodes()
        pos = {f: n for n, f in enumerate(nodes)}
        N, E, dev = len(nodes), len(edges), w2c.device
        e_idx = torch.tensor([[pos[i], pos[j]] for i, j, _, _ in edges], dtype=torch.int32, device=dev)
        Z = torch.stack([torch.as_tensor(z, dtype=torch.float64).to(dev)[:3].reshape(12) for _, _, z, _ in edges])
        wts = [cfg["loop_weights"] if k == LOOP else cfg["odometry_weights"] for _, _, _, k in edges]
        W = torch.tensor(wts, dtype=torch.float64, device=dev)
        poses = w2c[:, :3].double().reshape(N, 12).contiguous()
        old = poses.clone()
        n = 6 * (N - 1)
        H = torch.empty(n, n, dtype=torch.float64, device=dev)
        b = torch.empty(n, dtype=torch.float64, device=dev)
        res = torch.empty(E, 6, dtype=torch.float64, device=dev)
        jac = torch.empty(E, 72, dtype=torch.float64, device=dev)
        fn = torch.tensor(self.frame_nodes(T, t), dtype=torch.int32, device=dev)
        table = torch.empty(T, 12, dtype=torch.float32, device=dev)
        flag = torch.zeros(1, dtype=torch.int32, device=dev)
        err = torch.empty(E, 2, dtype=torch.float64, device=dev)
        steps = 0
        for _ in range(cfg["iters"]):
            _lib.call("sb_pose_graph_normal_equations", N, E, poses, e_idx, Z, W, res, jac, H, b, device=dev)
            L, info = torch.linalg.cholesky_ex(H)
            xi = torch.cholesky_solve(-b[:, None], L)[:, 0].contiguous()
            stop = int(info) != 0 or not float(xi.norm()) >= STEP_TOL
            if stop:
                xi.zero_()
            _lib.call("sb_pose_graph_update", N, E, T, poses, old, xi, e_idx, Z, fn, cfg["max_residual"][0],
                      math.radians(cfg["max_residual"][1]), table, flag, err, device=dev)
            if int(info) != 0:
                flag.zero_()                     # not positive definite: nothing is applied
            if stop:
                break
            steps += 1
        out = torch.zeros(N, 4, 4, dtype=torch.float64, device=dev)
        out[:, :3] = poses.reshape(N, 3, 4)
        out[:, 3, 3] = 1.0
        return dict(poses=out, correction_table=table, flag=flag, edge_err=err, steps=steps)

    def state(self):
        """The sidecar arrays of a checkpoint: loop_graph_edges int64 [E,3] (i, j, kind), loop_graph_z float64
        [E,4,4] and loop_graph_first."""
        z = [torch.as_tensor(e[2], dtype=torch.float64).cpu().numpy() for e in self.edges]
        return dict(loop_graph_edges=np.array([[i, j, k] for i, j, _, k in self.edges], dtype=np.int64).reshape(-1, 3),
                    loop_graph_z=np.array(z, dtype=np.float64).reshape(-1, 4, 4),
                    loop_graph_first=np.array(self.first, dtype=np.int64))

    @classmethod
    def from_state(cls, st, device=None):
        g = cls(int(st["loop_graph_first"]))
        for (i, j, k), z in zip(np.asarray(st["loop_graph_edges"]).reshape(-1, 3), np.asarray(st["loop_graph_z"])):
            zt = torch.from_numpy(np.array(z, dtype=np.float64))
            (g.add_loop if int(k) == LOOP else g.add_odometry)(int(i), int(j), zt if device is None else zt.to(device))
        return g

    @classmethod
    def chain(cls, ids, rots, trans):
        """Odometry edges between consecutive keyframes `ids`, measured from the camera columns (a resumed run whose
        checkpoint holds no graph)."""
        g = cls(int(ids[0]))
        for k in ids[1:]:
            g.add_odometry(g.nodes()[-1], int(k), g.odometry_from(rots, trans, int(k)))
        return g


def close_loop(t, frame, keyframes, rots, trans, graph, intrinsics, cfg, seed=0, mapper=None):
    """run_slam's loop-closure step at keyframe frame t, whose node and odometry edge `graph` already holds.  Rank 0
    finds the candidates, measures them in order and solves the graph with the first loop that passes; if every edge
    fits, the loop edge is kept and rank 0 corrects its camera columns (`correct_cameras`, in place).  Then, on every
    rank, the cameras go out through mapper.sync_camera, the correction table and flag are broadcast beside them, and
    each rank moves its Gaussians (mapper.deform) and its keyframes' est_w2c.  Returns (records, index into
    `keyframes` of the loop keyframe or None); records: one dict per measured candidate (see `measure`), `accepted`
    also requiring the graph's residual test."""
    T = rots.shape[-1]
    dev = rots.device
    world = mapper.world if mapper is not None else 1
    rank = mapper.rank if mapper is not None else 0
    records, loop_kf, table, flag = [], None, None, None
    if rank == 0:
        cands, _ = candidates(frame, t, keyframes, rots, trans, intrinsics, cfg, seed)
        for i in cands:
            rec, Z = measure(keyframes[i], frame, t, rots, trans, intrinsics, cfg)
            records.append(rec)
            if not rec["accepted"]:
                continue
            edge = (rec["keyframe"], t, Z, LOOP)
            nodes = graph.nodes()
            sol = graph.solve(w2c_columns(rots, trans, nodes), T, t, cfg, extra=edge)
            rec["accepted"] = bool(int(sol["flag"]))
            if rec["accepted"]:
                graph.add_loop(*edge[:3])
                loop_kf, table, flag = i, sol["correction_table"], sol["flag"]
                correct_cameras(rots, trans, table, t)
            break
    if world > 1:
        buf = torch.zeros(T * 12 + 2, dtype=torch.float32, device=dev)
        if table is not None:
            buf[:T * 12] = table.reshape(-1)
            buf[-2] = 1.0
            buf[-1] = float(loop_kf)
        mapper.dist.broadcast(buf, src=0, group=mapper.group)
        host = buf[-2:].tolist()
        if host[0] == 0.0:
            return records, None
        table, flag, loop_kf = buf[:T * 12].reshape(T, 12), torch.ones(1, dtype=torch.int32, device=dev), int(host[1])
        mapper.sync_camera()
    if table is None:
        return records, None
    if mapper is not None:
        mapper.deform(table, flag)
    with torch.no_grad():
        est = torch.stack([kf["est_w2c"].float() for kf in keyframes])
        C = _table_matrices(table.index_select(0, torch.tensor([int(kf["id"]) for kf in keyframes], device=dev)))
        est = est @ _rigid_inv(C)
        for kf, e in zip(keyframes, est):
            kf["est_w2c"] = e
    return records, loop_kf
