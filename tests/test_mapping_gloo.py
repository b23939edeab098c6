"""world_size-2 gloo test (CPU) of the keyframe-sharded mapping step's host logic: schedule, packed
gradient all-reduce == 1-process accumulation over the same keyframes, replicas stay identical.
The raster op on this CPU-only path is the float32 brute-force composite from oracle/ (the product
rasterizer has no CPU fallback); the GPU variant of this test lives in test_parity_gpu.py."""
import os
import socket

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

import scenes
from util import cpu_render
from splatam_b200 import mapping as M


def _problem():
    import splatam_b200 as S
    sc = scenes.config1(seed=4, P=96, w=48, h=32)
    cam = sc.settings(S.GaussianRasterizationSettings, "cpu")
    g = torch.Generator().manual_seed(0)
    gauss = dict(means3D=sc.means3D.clone(), rgb_colors=sc.colors.clone(),
                 unnorm_rotations=sc.rotations.clone() * 1.3, logit_opacities=torch.logit(sc.opacities.clamp(0.02, 0.98)),
                 log_scales=torch.log(sc.scales[:, :1].clone()))
    nframes = 4
    rots = torch.zeros(1, 4, nframes); rots[:, 0] = 1.0
    rots[:, 1:] = 0.01 * torch.randn(1, 3, nframes, generator=g)
    trans = 0.02 * torch.randn(1, 3, nframes, generator=g)
    frames = []
    for t in range(nframes):
        frames.append(dict(id=t, cam=cam, w2c=torch.eye(4), im=torch.rand(3, sc.h, sc.w, generator=g),
                           depth=1.0 + 2.0 * torch.rand(1, sc.h, sc.w, generator=g)))
    return gauss, rots, trans, frames


def _worker(rank, world, port, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    torch.set_num_threads(2)
    gauss, rots, trans, frames = _problem()
    mapper = M.ShardedMapper(gauss, rots, trans, render=cpu_render, seed=123)
    before = mapper.g.flat.detach().clone()
    loss, seen, picks = mapper.step(frames)
    q.put((rank, picks, mapper.g.flat_grad.numpy().copy(), mapper.g.flat.detach().numpy().copy(), before.numpy().copy(), loss))
    dist.barrier()
    dist.destroy_process_group()


def test_sharded_mapping_step_matches_single_process_accumulation():
    s = socket.socket(); s.bind(("127.0.0.1", 0)); port = s.getsockname()[1]; s.close()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    [p.start() for p in procs]
    res = sorted([q.get(timeout=300) for _ in range(2)], key=lambda t: t[0])
    [p.join(60) for p in procs]
    res = [(r, pk, torch.from_numpy(g), torch.from_numpy(p), torch.from_numpy(b), l) for r, pk, g, p, b, l in res]
    (r0, picks0, g0, p0, b0, l0), (r1, picks1, g1, p1, b1, l1) = res
    assert picks0 == picks1 and len(set(picks0)) == 2, "shared-seed schedule, distinct keyframes per rank"
    assert torch.equal(g0, g1), "all-reduced gradient bucket identical on both ranks"
    assert torch.equal(p0, p1) and not torch.equal(p0, b0), "replicas applied the same Adam update"
    assert abs(l0 - l1) < 1e-7
    # single-process reference: accumulate the same two keyframes into one bucket, one Adam step
    gauss, rots, trans, frames = _problem()
    ref = M.ShardedMapper(gauss, rots, trans, render=cpu_render, seed=123)
    ref.g.zero_grad()
    for k in picks0:
        ref.accumulate(frames[k])
    assert torch.allclose(ref.g.flat_grad, g0, rtol=1e-5, atol=1e-7), float((ref.g.flat_grad - g0).abs().max())
    ref.opt.step()
    assert torch.allclose(ref.g.flat.detach(), p0, rtol=1e-5, atol=1e-7)


def test_flat_bucket_layout_and_schedule():
    gauss, rots, trans, frames = _problem()
    m = M.ShardedMapper(gauss, rots, trans, render=cpu_render, seed=1)
    P = gauss["means3D"].shape[0]
    assert m.g.flat.numel() == P * (3 + 3 + 4 + 1 + 1) and m.g.flat_grad.numel() == m.g.flat.numel()
    for k in M.GAUSSIAN_KEYS:
        assert m.g.params[k].grad.data_ptr() >= m.g.flat_grad.data_ptr()
        assert torch.equal(m.g.params[k].detach(), gauss[k])
    loss, radius = M.mapping_loss(m.params(), frames[0], cpu_render)
    loss.backward()
    assert m.g.flat_grad.abs().sum() > 0 and torch.isfinite(m.g.flat_grad).all()
    assert m.schedule(5)[0] in range(5)


def _worker_edit(rank, world, port, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    torch.set_num_threads(2)
    gauss, rots, trans, frames = _problem()
    mapper = M.ShardedMapper(gauss, rots, trans, render=cpu_render, seed=123)
    mapper.step(frames)
    prune = dict(start_after=0, remove_big_after=0, stop_after=20, prune_every=1, removal_opacity_threshold=0.25,
                 final_removal_opacity_threshold=0.25, reset_opacities=False, reset_opacities_every=500)
    P1 = mapper.prune_gaussians(1, prune, scene_radius=50.0)          # every rank prunes its (identical) replica
    g = torch.Generator().manual_seed(9)
    new = dict(means3D=torch.randn(7, 3, generator=g) * 0.3 + torch.tensor([0.0, 0.0, 2.5]),
               rgb_colors=torch.rand(7, 3, generator=g), unnorm_rotations=torch.tensor([[1.0, 0, 0, 0]]).repeat(7, 1),
               logit_opacities=torch.zeros(7, 1), log_scales=torch.full((7, 1), -3.5))
    P2 = mapper.add_gaussians(new)
    loss, seen, picks = mapper.step(frames)                           # all-reduce over the RESIZED bucket
    q.put((rank, P1, P2, mapper.g.bucket.numel(), mapper.g.flat.detach().numpy().copy(), loss))
    dist.barrier()
    dist.destroy_process_group()


def test_prune_and_grow_keep_replicas_identical():
    s = socket.socket(); s.bind(("127.0.0.1", 0)); port = s.getsockname()[1]; s.close()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker_edit, args=(r, 2, port, q)) for r in range(2)]
    [p.start() for p in procs]
    res = sorted([q.get(timeout=300) for _ in range(2)], key=lambda t: t[0])
    [p.join(60) for p in procs]
    (_, P1a, P2a, nb_a, flat_a, la), (_, P1b, P2b, nb_b, flat_b, lb) = res
    assert P1a == P1b and 0 < P1a < 96 and P2a == P2b == P1a + 7
    assert nb_a == nb_b == P2a * 12 + P2a + 2                         # gradients | seen flags | loss | overflow flag
    assert (flat_a == flat_b).all() and abs(la - lb) < 1e-7


def _worker_sync(rank, world, port, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    gauss, rots, trans, frames = _problem()
    mapper = M.ShardedMapper(gauss, rots, trans, render=cpu_render, seed=5)
    mapper.cam = dict(cam_unnorm_rots=rots + 0.1 * rank, cam_trans=trans - 0.2 * rank)    # rank 1 "tracked" differently
    cam = mapper.sync_camera(src=0)
    fr = dict(frames[0], im=frames[0]["im"] + rank, depth=frames[0]["depth"] * (1 + rank), w2c=torch.eye(4) * (1 + rank))
    fr = mapper.broadcast_frame(fr, src=0)
    q.put((rank, cam["cam_unnorm_rots"].numpy().copy(), cam["cam_trans"].numpy().copy(), fr["im"].numpy().copy(),
           fr["depth"].numpy().copy(), fr["w2c"].numpy().copy()))
    dist.barrier()
    dist.destroy_process_group()


def test_single_rank_results_are_broadcast():
    """Tracking / data loading stay on one rank; poses and keyframe images reach the others by broadcast."""
    s = socket.socket(); s.bind(("127.0.0.1", 0)); port = s.getsockname()[1]; s.close()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker_sync, args=(r, 2, port, q)) for r in range(2)]
    [p.start() for p in procs]
    res = sorted([q.get(timeout=300) for _ in range(2)], key=lambda t: t[0])
    [p.join(60) for p in procs]
    gauss, rots, trans, frames = _problem()
    for a, b in zip(res[0][1:], res[1][1:]):
        assert (a == b).all()
    assert (res[1][1] == rots.numpy()).all() and (res[1][2] == trans.numpy()).all()
    assert (res[1][3] == frames[0]["im"].numpy()).all() and (res[1][5] == torch.eye(4).numpy()).all()


def _worker_densify(rank, world, port, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    torch.set_num_threads(2)
    gauss, rots, trans, frames = _problem()
    mapper = M.ShardedMapper(gauss, rots, trans, render=cpu_render, seed=77, track_means2D=True)
    dd = dict(start_after=0, remove_big_after=0, stop_after=10, densify_every=1, grad_thresh=1e-9, num_to_split_into=2,
              removal_opacity_threshold=0.05, final_removal_opacity_threshold=0.05, reset_opacities=False,
              reset_opacities_every=100)
    counts = []
    for it in range(2):
        mapper.step(frames)                                   # each rank renders a different keyframe
        counts.append(mapper.densify(it, dd, scene_radius=0.4))
    loss, _, _ = mapper.step(frames)                          # the resized replicas keep stepping together
    q.put((rank, counts, mapper.g.flat.detach().numpy().copy(), loss))
    dist.barrier()
    dist.destroy_process_group()


def test_densify_keeps_replicas_identical():
    """Gradient-based densification on two ranks: the statistic is summed over the ranks' keyframes and the split samples
    come from a shared-seed generator, so both replicas clone / split / prune identically."""
    s = socket.socket(); s.bind(("127.0.0.1", 0)); port = s.getsockname()[1]; s.close()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker_densify, args=(r, 2, port, q)) for r in range(2)]
    [p.start() for p in procs]
    res = sorted([q.get(timeout=300) for _ in range(2)], key=lambda t: t[0])
    [p.join(60) for p in procs]
    (_, ca, fa, la), (_, cb, fb, lb) = res
    assert ca == cb and ca[-1] != 96
    assert fa.shape == fb.shape and (fa == fb).all() and abs(la - lb) < 1e-7
