"""world_size-2 gloo test (CPU) of keyframe-pose refinement in the sharded mapping step: the [7, T] pose-gradient table
travels in the one all-reduce bucket, so two ranks equal one process accumulating the same two keyframes, and both
replicas' poses stay bit-identical through steps, a prune and a grow.  Rasterizer: the float32 brute-force composite
from oracle/, as test_mapping_gloo.py."""
import os
import socket

import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from splatam_b200 import mapping as M
from test_mapping_gloo import _problem
from util import cpu_render

LRS = dict(cam_unnorm_rots=0.0004, cam_trans=0.002)
PRUNE = dict(start_after=0, remove_big_after=100, stop_after=20, prune_every=1, removal_opacity_threshold=0.1,
             final_removal_opacity_threshold=0.1, reset_opacities=False, reset_opacities_every=500)


def _worker(rank, world, port, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    torch.set_num_threads(2)
    gauss, rots, trans, frames = _problem()
    mapper = M.ShardedMapper(gauss, rots, trans, render=cpu_render, seed=123, lrs=LRS)
    _, _, picks = mapper.step(frames)
    first = dict(picks=picks, pose_grad=mapper.g.pose_grad.numpy().copy(),
                 cams=[mapper.cam[k].detach().numpy().copy() for k in M.CAM_KEYS],
                 flat=mapper.g.flat.detach().numpy().copy())
    counts = [mapper.prune_gaussians(0, PRUNE, 1.0)]
    mapper.step(frames)
    counts.append(mapper.add_gaussians({k: v.detach()[:7].clone() + 0.01 for k, v in mapper.g.params.items()}))
    mapper.step(frames)
    last = [mapper.cam[k].detach().numpy().copy() for k in M.CAM_KEYS]
    q.put((rank, first, counts, last))
    dist.barrier()
    dist.destroy_process_group()


def test_two_ranks_equal_one_process_and_poses_stay_identical():
    s = socket.socket(); s.bind(("127.0.0.1", 0)); port = s.getsockname()[1]; s.close()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    [p.start() for p in procs]
    res = sorted([q.get(timeout=300) for _ in range(2)], key=lambda t: t[0])
    [p.join(60) for p in procs]
    (_, f0, c0, last0), (_, f1, c1, last1) = res
    assert f0["picks"] == f1["picks"] and len(set(f0["picks"])) == 2
    for a, b in zip(f0["cams"] + last0, f1["cams"] + last1):
        assert (a == b).all(), "replicas' poses bit-identical"
    assert c0 == c1 and c0[0] < 96
    g0 = torch.from_numpy(f0["pose_grad"]).view(7, -1)
    assert torch.equal(g0, torch.from_numpy(f1["pose_grad"]).view(7, -1))
    # both drawn columns carry gradient, the others none
    drawn = sorted(f0["picks"])
    assert all(float(g0[:, c].abs().sum()) > 0 for c in drawn)
    assert all(float(g0[:, c].abs().sum()) == 0 for c in range(g0.shape[1]) if c not in drawn)
    # one process accumulating the same two keyframes, one Adam step of map and poses
    gauss, rots, trans, frames = _problem()
    ref = M.ShardedMapper(gauss, rots, trans, render=cpu_render, seed=123, lrs=LRS)
    ref.g.zero_grad()
    for k in f0["picks"]:
        ref.accumulate(frames[k])
    assert torch.allclose(ref.g.pose_grad.view(7, -1), g0, rtol=1e-5, atol=1e-7)
    ref.opt.step()
    ref._cam_step()
    assert torch.allclose(ref.g.flat.detach(), torch.from_numpy(f0["flat"]), rtol=1e-5, atol=1e-7)
    for k, c in zip(M.CAM_KEYS, f0["cams"]):
        assert torch.allclose(ref.cam[k].detach(), torch.from_numpy(c), rtol=1e-6, atol=1e-7), k
