"""world_size-2 gloo test (CPU) of run_slam with motion masks: only rank 0's tracking result is the pose of record,
each rank then computes the frame's masks from its own replica, and the masks gate the mapping loss (and, on CUDA,
map growth), so the replicas stay identical only if every rank computes the same masks.  Both ranks must end with the
same cameras, the same map and the same keyframe masks.  Rasterizer: the float32 brute-force composite from oracle/."""
import os
import socket

import numpy as np
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

import scenes
from util import cpu_render

T = 5


def _problem():
    import splatam_b200 as S
    from splatam_b200 import slam
    sc = scenes.config1(seed=8, P=1024, w=48, h=48)
    cam = sc.settings(S.GaussianRasterizationSettings, "cpu")
    gt = sc.splatam_params(opacity_clamp=(0.9, 0.99))
    rots, trans = slam.look_trajectory(T, "cpu", step=(0.004, -0.002, 0.003), rot_step=(0.001, -0.001, 0.0005))
    frames = [slam.render_frame(gt, rots, trans, t, cam, render=cpu_render) for t in range(T)]
    for t in range(2, T):         # a flat occluder 40 % nearer than the scene, moving right 4 px per frame
        frames[t]["depth"][:, 14:30, 4 * t:4 * t + 10] *= 0.6
        frames[t]["im"][:, 14:30, 4 * t:4 * t + 10] = 0.5
    K = torch.tensor([[sc.fx, 0, sc.cx], [0, sc.fy, sc.cy], [0, 0, 1]])
    kw = dict(render=cpu_render, fused=False, tracking_iters=6, mapping_iters=2, keyframe_every=2, window=3,
              intrinsics=K, dynamic=dict(radius=4))
    return cam, frames, dict(gt), kw


def _worker(rank, world, port, q):
    from splatam_b200 import slam
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    torch.set_num_threads(2)
    cam, frames, init, kw = _problem()
    torch.manual_seed(1); np.random.seed(1)
    out = slam.run_slam(init, frames, cam, **kw)
    q.put((rank, out["rots"].numpy().copy(), out["trans"].numpy().copy(),
           {k: v.numpy().copy() for k, v in out["gauss"].items()},
           [m.numpy().copy() for m in out["keyframe_dynamic"]], out["dynamic"]))
    dist.barrier()
    dist.destroy_process_group()


def test_both_ranks_end_with_the_same_map_and_keyframe_masks():
    s = socket.socket(); s.bind(("127.0.0.1", 0)); port = s.getsockname()[1]; s.close()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    [p.start() for p in procs]
    res = sorted([q.get(timeout=600) for _ in range(2)], key=lambda t: t[0])
    [p.join(60) for p in procs]
    (_, r0, t0, g0, m0, s0), (_, r1, t1, g1, m1, s1) = res
    assert (r0 == r1).all() and (t0 == t1).all()
    for k in g0:
        assert (g0[k] == g1[k]).all(), k
    assert len(m0) == len(m1) and all((a == b).all() for a, b in zip(m0, m1))
    assert s0 == s1
    assert any(m.any() for m in m0)                     # the occluder was flagged on some keyframe
