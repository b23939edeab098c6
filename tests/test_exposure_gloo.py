"""world_size-2 gloo test (CPU) of per-frame exposure in the sharded mapper: the rank that tracks holds the exposure
table, `sync_camera` broadcasts it beside the poses, and both replicas then map through the same corrections and end
with the same table and the same map.  Rasterizer: the float32 brute-force composite from oracle/, as
test_mapping_gloo.py."""
import os
import socket

import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from splatam_b200 import mapping as M
from test_mapping_gloo import _problem
from util import cpu_render


def _worker(rank, world, port, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    torch.set_num_threads(2)
    gauss, rots, trans, frames = _problem()
    T = rots.shape[-1]
    expo = torch.zeros(1, 6, T)
    mapper = M.ShardedMapper(gauss, rots, trans, render=cpu_render, seed=123, cam_exposure=expo)
    if rank == 0:               # only rank 0 tracks: its estimates are the table of record
        table = torch.linspace(-0.1, 0.1, 6 * T).reshape(1, 6, T)
        table[..., 0] = 0.0
        mapper.cam["cam_exposure"] = table
    cam = mapper.sync_camera()
    for _ in range(2):
        mapper.step(frames)
    q.put((rank, cam["cam_exposure"].numpy().copy(), mapper.cam["cam_exposure"].numpy().copy(),
           mapper.g.flat.detach().numpy().copy()))
    dist.barrier()
    dist.destroy_process_group()


def test_both_ranks_end_with_the_same_exposure_table_and_map():
    s = socket.socket(); s.bind(("127.0.0.1", 0)); port = s.getsockname()[1]; s.close()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    [p.start() for p in procs]
    res = sorted([q.get(timeout=300) for _ in range(2)], key=lambda t: t[0])
    [p.join(60) for p in procs]
    (_, synced0, end0, flat0), (_, synced1, end1, flat1) = res
    assert (synced0 == synced1).all() and (end0 == end1).all()
    assert abs(end1).max() > 0.05                       # rank 1 received rank 0's table
    assert (flat0 == flat1).all(), "replicas bit-identical"
