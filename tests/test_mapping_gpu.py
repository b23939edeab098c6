"""GPU tests of the keyframe-sharded mapping step: the product rasterizer inside SplaTAM's mapping loss,
1-GPU accumulation vs the sharded step (NCCL, when >= 2 GPUs are visible)."""
import os
import socket

import numpy as np
import pytest
import torch

import scenes

pytestmark = pytest.mark.gpu


def _problem(dev, P=20000, nframes=4):
    import splatam_b200 as S
    sc = scenes.room(seed=21, P=P, cam=dict(w=320, h=192, fx=160.0, fy=160.0, cx=159.5, cy=95.5))
    cam = sc.settings(S.GaussianRasterizationSettings, dev)
    g = torch.Generator().manual_seed(0)
    gauss = sc.splatam_params(dev)
    rots = torch.zeros(1, 4, nframes); rots[:, 0] = 1.0
    rots[:, 1:] = 0.01 * torch.randn(1, 3, nframes, generator=g)
    trans = 0.02 * torch.randn(1, 3, nframes, generator=g)
    frames = [dict(id=t, cam=cam, w2c=torch.eye(4, device=dev), im=torch.rand(3, sc.h, sc.w, generator=g).to(dev),
                   depth=(1.0 + 2.0 * torch.rand(1, sc.h, sc.w, generator=g)).to(dev)) for t in range(nframes)]
    return gauss, rots.to(dev), trans.to(dev), frames


def test_mapping_loss_backward_single_gpu(cuda_device):
    from splatam_b200 import mapping as M
    gauss, rots, trans, frames = _problem(cuda_device)
    m = M.ShardedMapper(gauss, rots, trans, seed=5)
    before = m.g.flat.detach().clone()
    loss, seen, picks = m.step(frames)
    assert np.isfinite(loss) and seen.any()
    assert torch.isfinite(m.g.flat_grad).all() and m.g.flat_grad.abs().sum() > 0
    assert not torch.equal(before, m.g.flat.detach())
    # a second mapper fed the same keyframe accumulates the same gradient (deterministic schedule);
    # float atomics in the blend backward make it equal only to ~1e-6 relative
    m2 = M.ShardedMapper(gauss, rots, trans, seed=5)
    m2.g.zero_grad()
    m2.accumulate(frames[picks[0]])
    rel = (m2.g.flat_grad - m.g.flat_grad).norm() / m.g.flat_grad.norm()
    assert rel < 1e-4, float(rel)


def _worker(rank, world, port, q):
    import torch.distributed as dist
    from splatam_b200 import mapping as M
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dev = torch.device("cuda", rank)
    torch.cuda.set_device(dev)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    gauss, rots, trans, frames = _problem(dev)
    m = M.ShardedMapper(gauss, rots, trans, seed=7)
    loss, seen, picks = m.step(frames)
    torch.cuda.synchronize()
    q.put((rank, picks, m.g.flat_grad.cpu().numpy(), m.g.flat.detach().cpu().numpy(), loss))
    dist.barrier()
    dist.destroy_process_group()


def test_sharded_step_nccl_two_gpus(cuda_device):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp
    from splatam_b200 import mapping as M
    s = socket.socket(); s.bind(("127.0.0.1", 0)); port = s.getsockname()[1]; s.close()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    [p.start() for p in procs]
    res = sorted([q.get(timeout=600) for _ in range(2)], key=lambda t: t[0])
    [p.join(120) for p in procs]
    (_, p0, g0, f0, l0), (_, p1, g1, f1, l1) = res
    assert p0 == p1 and len(set(p0)) == 2
    assert np.array_equal(g0, g1) and np.array_equal(f0, f1), "replicas must stay bit-identical"
    gauss, rots, trans, frames = _problem(cuda_device)
    ref = M.ShardedMapper(gauss, rots, trans, seed=7)
    ref.g.zero_grad()
    for k in p0:
        ref.accumulate(frames[k])
    a, b = ref.g.flat_grad.cpu().numpy(), g0
    assert np.linalg.norm(a - b) / np.linalg.norm(b) < 1e-4


def test_graph_mode_matches_eager(cuda_device):
    """CUDA-graph replay of the mapping step (sync-free rasterizer) == the eager fused step."""
    from splatam_b200 import mapping as M
    gauss, rots, trans, frames = _problem(cuda_device)
    eager = M.ShardedMapper(gauss, rots, trans, seed=9)
    graph = M.ShardedMapper(gauss, rots, trans, seed=9)
    cap = graph.enable_graph(frames)
    le, _, pe = eager.step(frames)
    lg, _, pg = graph.step(frames)
    assert pe == pg
    assert abs(le - float(lg)) < 1e-5 * max(1.0, abs(le)), (le, float(lg))
    ge, gg = eager.g.flat_grad, graph.g.flat_grad
    assert float((ge - gg).norm() / ge.norm()) < 1e-4
    # (parameters are not compared after the update: with eps = 1e-15 Adam moves an entry by ~lr whatever the
    # gradient's size, so entries whose gradient is float-atomics noise legitimately differ between two runs)
    for _ in range(3):
        lg, seen, _ = graph.step(frames)
    n, overflow = graph.check_capacity()
    assert not overflow and 0 < n <= cap and bool(torch.isfinite(lg)) and bool(seen.any())
